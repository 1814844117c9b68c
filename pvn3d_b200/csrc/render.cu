// render.cu -- a batched z-buffer rasteriser of vertex-coloured triangle meshes at given poses: the rgb, depth (metres)
// and label images of LineMOD's synthetic `render` and `fuse` frames (linemod_dataset.py:48-61,192-204), made on the
// stream instead of read from pickles.
//
// The raster contract (tests/render_ref.py restates it bit for bit in numpy):
//   vertex    every vertex p (float32 promoted to float64) of a drawn class c (1 <= c < n_cls, present[f,c] != 0) goes
//             to q_j = ((R_j0 x + R_j1 y) + R_j2 z) + t_j, then sx = fx q_0 / q_2 + cx, sy = fy q_1 / q_2 + cy (as
//             ((fx * q_0) / q_2) + cx), every product, sum and quotient rounded on its own (no FMA).  fx = K[0,0],
//             cx = K[0,2], fy = K[1,1], cy = K[1,2]; K's other entries are not read.  Pixel (row v, col u) samples the
//             ray ((u - cx) / fx, (v - cy) / fy, 1): centres at integer u, v, as dpt_2_cld back-projects (not
//             OpenGL's +0.5).  A vertex is usable when q_2 >= z_near and |sx|, |sy| <= 16384 (the guard band; NaN
//             fails), and then snaps to X = rint(256 sx), Y = rint(256 sy) (1/256 px, half to even) with
//             1/z = 1 / q_2.
//   triangle  skipped when a vertex is unusable or outside its class's vertex range, or when its snapped signed
//             area A = (X1-X0)(Y2-Y0) - (Y1-Y0)(X2-X0) (int64) is 0.  A < 0 swaps vertices 1 and 2 (no back-face
//             culling).  Candidate pixels: the bounding box of the snapped vertices cut to the frame.
//   coverage  at P = (256 u, 256 v): w0 = E(V1,V2), w1 = E(V2,V0), w2 = E(V0,V1) with E(a,b) = (bx-ax)(Py-ay) -
//             (by-ay)(Px-ax), exact in int64 (w0 + w1 + w2 = A).  Covered when every w_k > 0, or w_k = 0 on an edge
//             a -> b that owns its pixels (top-left rule: by - ay < 0, or by == ay and bx - ax > 0); a pixel centre on
//             an edge two triangles share is covered once.
//   depth     t_k = double(w_k) * (1/z_k), n = (t0 + t1) + t2, z = double(A) / n, rounded to float32.
//   visible   the smallest float32 depth; equal depths: the lower packed face index (faces are packed by class, then
//             by face index, so the lower class id wins first).  A total order: the result does not depend on thread
//             scheduling.
//   colour    ((t0 c0 + t1 c1) + t2 c2) / n per channel in float64, rint (half to even), clamped to [0, 255].
//   label     the visible face's class id.  Uncovered pixels: rgb 0, depth 0, label 0, or the background's rgb and
//             depth (label 0) when one is given (add_real_back's mask composite; it takes no part in the depth test).
//
// One memset and five launches, no host sync, no allocation:
//   render_vertex_kernel    one thread per (frame, vertex) of a drawn class: the snapped vertex record.
//   render_setup_kernel     one thread per (frame, face): the candidate-pixel count of the face's bounding box, and
//                           the inclusive scan of those counts over each 1024-face block.
//   render_scan_kernel      one CTA: the exclusive scan of the block totals, and the fragment total.
//   render_fragment_kernel  persistent, grid-stride over the fragments (a face's candidate pixels, in scan order): each
//                           finds its face by binary search of the scan, tests coverage and atomicMin's a 64-bit key
//                           (float32 depth bits << 32 | packed face index) into its pixel.  A large triangle is spread
//                           over many threads.
//   render_resolve_kernel   one thread per pixel: the winner's colour, depth and label, or the background.
#include <math.h>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kMaxSide = 4096;
constexpr int kMaxCls = 256;
constexpr double kGuard = 16384.0;            // px; snapped |X|, |Y| <= 2^22, edge products < 2^47
constexpr int kVtxThreads = 256;
constexpr int kScanBlock = 1024;              // faces per block of the two-level scan (one thread each)
constexpr int kFragThreads = 256;
constexpr int kFragPerThread = 4;
constexpr int kChunk = kFragThreads * kFragPerThread;
constexpr int kResolveThreads = 256;
constexpr int kUnusable = static_cast<int>(0x80000000u);   // X of a vertex that no triangle may use
constexpr unsigned long long kEmpty = ~0ull;

struct Vtx {
  int x, y;     // snapped screen position, 1/256 px
  double iz;    // 1 / camera z
};

struct Mesh {
  const float *vtx;        // [n_vtx,3]
  const uint8_t *col;      // [n_vtx,3]
  const int *faces;        // [n_faces,3] packed vertex indices
  const int *vtx_off;      // [n_cls+1]
  const int *face_off;     // [n_cls+1]
  int n_cls, n_vtx, n_faces;
};

struct Frames {
  const void *poses;       // [b,n_cls,3,4]
  int poses_f64;
  const uint8_t *present;  // [b,n_cls]
  const double *k;         // [b,3,3]
  double z_near;
  int b, h, w;
};

struct Tri {
  long long x[3], y[3];
  double iz[3];
  int v[3];                // packed vertex indices, in the (possibly swapped) order of x / y / iz
  long long area;
  int u0, v0, bw, bh;      // candidate pixels [u0, u0 + bw) x [v0, v0 + bh)
};

__device__ __forceinline__ double dot3(double x, double y, double z, double a, double b, double c) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, a), __dmul_rn(y, b)), __dmul_rn(z, c));
}

// the largest c in [0, n) with off[c] <= i: the class owning packed element i (empty classes are passed over)
__device__ __forceinline__ int owner(const int *off, int n, int i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void load_offsets(int *s, const int *g, int n_cls) {
  for (int i = threadIdx.x; i <= n_cls; i += blockDim.x) s[i] = g[i];
  __syncthreads();
}

__device__ __forceinline__ bool drawn(const Frames &f, int n_cls, int b, int c) {
  return c > 0 && f.present[static_cast<size_t>(b) * n_cls + c] != 0;
}

// face `face` of class c in frame b from the frame's vertex records; false = not drawn or no candidate pixel
__device__ bool tri_setup(const Mesh &m, const Frames &f, const Vtx *fv, const int *s_voff, int face, int c, Tri &t) {
  const int lo = s_voff[c], hi = s_voff[c + 1];
  for (int k = 0; k < 3; ++k) {
    const int v = __ldg(m.faces + static_cast<size_t>(face) * 3 + k);
    if (v < lo || v >= hi) return false;
    const Vtx r = fv[v];
    if (r.x == kUnusable) return false;
    t.v[k] = v;
    t.x[k] = r.x;
    t.y[k] = r.y;
    t.iz[k] = r.iz;
  }
  long long a = (t.x[1] - t.x[0]) * (t.y[2] - t.y[0]) - (t.y[1] - t.y[0]) * (t.x[2] - t.x[0]);
  if (a == 0) return false;
  if (a < 0) {
    long long s = t.x[1]; t.x[1] = t.x[2]; t.x[2] = s;
    s = t.y[1]; t.y[1] = t.y[2]; t.y[2] = s;
    const double d = t.iz[1]; t.iz[1] = t.iz[2]; t.iz[2] = d;
    const int v = t.v[1]; t.v[1] = t.v[2]; t.v[2] = v;
    a = -a;
  }
  t.area = a;
  const long long x0 = min(min(t.x[0], t.x[1]), t.x[2]), x1 = max(max(t.x[0], t.x[1]), t.x[2]);
  const long long y0 = min(min(t.y[0], t.y[1]), t.y[2]), y1 = max(max(t.y[0], t.y[1]), t.y[2]);
  // pixels u with 256 u in [x0, x1]: ceil(x0 / 256) .. floor(x1 / 256) (arithmetic shifts floor)
  const long long ua = max(-((-x0) >> 8), 0ll), ub = min(x1 >> 8, static_cast<long long>(f.w - 1));
  const long long va = max(-((-y0) >> 8), 0ll), vb = min(y1 >> 8, static_cast<long long>(f.h - 1));
  if (ua > ub || va > vb) return false;
  t.u0 = static_cast<int>(ua);
  t.v0 = static_cast<int>(va);
  t.bw = static_cast<int>(ub - ua + 1);
  t.bh = static_cast<int>(vb - va + 1);
  return true;
}

__device__ __forceinline__ long long edge(long long ax, long long ay, long long bx, long long by, long long px,
                                          long long py) {
  return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}
__device__ __forceinline__ bool covers(long long e, long long ax, long long ay, long long bx, long long by) {
  return e > 0 || (e == 0 && (by - ay < 0 || (by == ay && bx - ax > 0)));
}

// coverage of pixel (u, v); on true, w[] holds the edge functions
__device__ __forceinline__ bool inside(const Tri &t, int u, int v, long long w[3]) {
  const long long px = static_cast<long long>(u) << 8, py = static_cast<long long>(v) << 8;
  w[0] = edge(t.x[1], t.y[1], t.x[2], t.y[2], px, py);
  w[1] = edge(t.x[2], t.y[2], t.x[0], t.y[0], px, py);
  w[2] = edge(t.x[0], t.y[0], t.x[1], t.y[1], px, py);
  return covers(w[0], t.x[1], t.y[1], t.x[2], t.y[2]) && covers(w[1], t.x[2], t.y[2], t.x[0], t.y[0]) &&
         covers(w[2], t.x[0], t.y[0], t.x[1], t.y[1]);
}

// ---- 1. vertices ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kVtxThreads)
    render_vertex_kernel(const __grid_constant__ Mesh m, const __grid_constant__ Frames f, Vtx *__restrict__ out) {
  __shared__ int s_voff[kMaxCls + 1];
  load_offsets(s_voff, m.vtx_off, m.n_cls);
  const long long total = static_cast<long long>(f.b) * m.n_vtx;
  for (long long i = blockIdx.x * static_cast<long long>(kVtxThreads) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * kVtxThreads) {
    const int b = static_cast<int>(i / m.n_vtx), vi = static_cast<int>(i - static_cast<long long>(b) * m.n_vtx);
    const int c = owner(s_voff, m.n_cls, vi);
    if (!drawn(f, m.n_cls, b, c)) continue;   // no face of an undrawn class reads this record
    const float *p = m.vtx + static_cast<size_t>(vi) * 3;
    const double x = p[0], y = p[1], z = p[2];
    double rt[12];
    const size_t pe = (static_cast<size_t>(b) * m.n_cls + c) * 12;
    if (f.poses_f64) {
      for (int e = 0; e < 12; ++e) rt[e] = static_cast<const double *>(f.poses)[pe + e];
    } else {
      for (int e = 0; e < 12; ++e) rt[e] = static_cast<const float *>(f.poses)[pe + e];
    }
    double q[3];
    for (int j = 0; j < 3; ++j) q[j] = __dadd_rn(dot3(x, y, z, rt[j * 4], rt[j * 4 + 1], rt[j * 4 + 2]), rt[j * 4 + 3]);
    const double *k = f.k + static_cast<size_t>(b) * 9;
    const double sx = __dadd_rn(__ddiv_rn(__dmul_rn(k[0], q[0]), q[2]), k[2]);
    const double sy = __dadd_rn(__ddiv_rn(__dmul_rn(k[4], q[1]), q[2]), k[5]);
    Vtx r;
    if (q[2] >= f.z_near && fabs(sx) <= kGuard && fabs(sy) <= kGuard) {
      r.x = static_cast<int>(rint(__dmul_rn(sx, 256.0)));
      r.y = static_cast<int>(rint(__dmul_rn(sy, 256.0)));
      r.iz = __ddiv_rn(1.0, q[2]);
    } else {
      r.x = r.y = kUnusable;
      r.iz = 0.0;
    }
    out[i] = r;
  }
}

// ---- 2. per-face candidate counts and their scan within each 1024-face block ---------------------------------------
__global__ void __launch_bounds__(kScanBlock)
    render_setup_kernel(const __grid_constant__ Mesh m, const __grid_constant__ Frames f, const Vtx *__restrict__ vtx,
                        unsigned long long *__restrict__ incl, unsigned long long *__restrict__ blk_total) {
  __shared__ int s_voff[kMaxCls + 1], s_foff[kMaxCls + 1];
  __shared__ unsigned long long s_warp[kScanBlock / 32];
  for (int i = threadIdx.x; i <= m.n_cls; i += blockDim.x) s_foff[i] = m.face_off[i];
  load_offsets(s_voff, m.vtx_off, m.n_cls);
  const long long j = static_cast<long long>(blockIdx.x) * kScanBlock + threadIdx.x;
  unsigned long long cnt = 0;
  if (j < static_cast<long long>(f.b) * m.n_faces) {
    const int b = static_cast<int>(j / m.n_faces), face = static_cast<int>(j - static_cast<long long>(b) * m.n_faces);
    const int c = owner(s_foff, m.n_cls, face);
    Tri t;
    if (drawn(f, m.n_cls, b, c) &&
        tri_setup(m, f, vtx + static_cast<size_t>(b) * m.n_vtx, s_voff, face, c, t))
      cnt = static_cast<unsigned long long>(t.bw) * t.bh;
  }
  // inclusive block scan: warp shuffles, then the warp totals
  unsigned long long s = cnt;
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long o = __shfl_up_sync(0xffffffffu, s, d);
    if (static_cast<int>(lane_id()) >= d) s += o;
  }
  const int warp = threadIdx.x >> 5;
  if (lane_id() == 31) s_warp[warp] = s;
  __syncthreads();
  if (warp == 0) {
    unsigned long long ws = s_warp[lane_id()];
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long o = __shfl_up_sync(0xffffffffu, ws, d);
      if (static_cast<int>(lane_id()) >= d) ws += o;
    }
    s_warp[lane_id()] = ws;
  }
  __syncthreads();
  if (warp > 0) s += s_warp[warp - 1];
  incl[j] = s;
  if (threadIdx.x == kScanBlock - 1) blk_total[blockIdx.x] = s;
}

// ---- 3. exclusive scan of the block totals (one CTA); excl[nb] = the fragment total --------------------------------
__global__ void __launch_bounds__(kScanBlock)
    render_scan_kernel(const unsigned long long *__restrict__ blk_total, int nb, unsigned long long *__restrict__ excl) {
  __shared__ unsigned long long s_warp[kScanBlock / 32];
  __shared__ unsigned long long s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  for (int base = 0; base < nb; base += kScanBlock) {
    const int i = base + threadIdx.x;
    const unsigned long long v = i < nb ? blk_total[i] : 0ull;
    unsigned long long s = v;
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long o = __shfl_up_sync(0xffffffffu, s, d);
      if (static_cast<int>(lane_id()) >= d) s += o;
    }
    const int warp = threadIdx.x >> 5;
    if (lane_id() == 31) s_warp[warp] = s;
    __syncthreads();
    if (warp == 0) {
      unsigned long long ws = s_warp[lane_id()];
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long o = __shfl_up_sync(0xffffffffu, ws, d);
        if (static_cast<int>(lane_id()) >= d) ws += o;
      }
      s_warp[lane_id()] = ws;
    }
    __syncthreads();
    if (warp > 0) s += s_warp[warp - 1];
    const unsigned long long carry = s_carry;
    if (i < nb) excl[i] = carry + s - v;
    __syncthreads();
    if (threadIdx.x == kScanBlock - 1) s_carry = carry + s;
    __syncthreads();
  }
  if (threadIdx.x == 0) excl[nb] = s_carry;
}

// inclusive fragment count up to face slot j: the block-local scan plus the block's exclusive offset
__device__ __forceinline__ unsigned long long incl_at(const unsigned long long *incl, const unsigned long long *excl,
                                                      long long j) {
  return incl[j] + excl[j / kScanBlock];
}

// the face slot holding fragment i (< the total): the smallest j with incl_at(j) > i
__device__ long long find_slot(const unsigned long long *incl, const unsigned long long *excl, int nb,
                               unsigned long long i) {
  int lo = 0, hi = nb - 1;   // the last block whose exclusive offset is <= i (it holds fragment i)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (excl[mid] <= i) lo = mid; else hi = mid - 1;
  }
  const unsigned long long r = i - excl[lo];
  long long a = static_cast<long long>(lo) * kScanBlock, z = a + kScanBlock - 1;
  while (a < z) {
    const long long mid = (a + z) >> 1;
    if (incl[mid] > r) z = mid; else a = mid + 1;
  }
  return a;
}

// ---- 4. fragments -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kFragThreads)
    render_fragment_kernel(const __grid_constant__ Mesh m, const __grid_constant__ Frames f, const Vtx *__restrict__ vtx,
                           const unsigned long long *__restrict__ incl, const unsigned long long *__restrict__ excl,
                           int nb, unsigned long long *__restrict__ keys) {
  __shared__ int s_voff[kMaxCls + 1], s_foff[kMaxCls + 1];
  __shared__ long long s_lo, s_hi;
  for (int i = threadIdx.x; i <= m.n_cls; i += blockDim.x) s_foff[i] = m.face_off[i];
  load_offsets(s_voff, m.vtx_off, m.n_cls);
  const unsigned long long total = excl[nb];
  const size_t hw = static_cast<size_t>(f.h) * f.w;
  for (unsigned long long c0 = static_cast<unsigned long long>(blockIdx.x) * kChunk; c0 < total;
       c0 += static_cast<unsigned long long>(gridDim.x) * kChunk) {
    const unsigned long long c1 = min(c0 + kChunk, total);
    // the chunk's first and last face slots bound every thread's search
    if (threadIdx.x == 0) s_lo = find_slot(incl, excl, nb, c0);
    if (threadIdx.x == 32) s_hi = find_slot(incl, excl, nb, c1 - 1);
    __syncthreads();
    const long long lo0 = s_lo, hi0 = s_hi;
    __syncthreads();
    for (int r = 0; r < kFragPerThread; ++r) {
      const unsigned long long i = c0 + static_cast<unsigned long long>(r) * kFragThreads + threadIdx.x;
      if (i >= c1) break;
      long long lo = lo0, hi = hi0;
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (incl_at(incl, excl, mid) > i) hi = mid; else lo = mid + 1;
      }
      const unsigned long long first = lo == 0 ? 0ull : incl_at(incl, excl, lo - 1);
      const unsigned local = static_cast<unsigned>(i - first);
      const int b = static_cast<int>(lo / m.n_faces), face = static_cast<int>(lo - static_cast<long long>(b) * m.n_faces);
      const int c = owner(s_foff, m.n_cls, face);
      Tri t;
      if (!tri_setup(m, f, vtx + static_cast<size_t>(b) * m.n_vtx, s_voff, face, c, t)) continue;   // never: count > 0
      const int u = t.u0 + static_cast<int>(local % static_cast<unsigned>(t.bw));
      const int v = t.v0 + static_cast<int>(local / static_cast<unsigned>(t.bw));
      long long w[3];
      if (!inside(t, u, v, w)) continue;
      const double t0 = __dmul_rn(static_cast<double>(w[0]), t.iz[0]);
      const double t1 = __dmul_rn(static_cast<double>(w[1]), t.iz[1]);
      const double t2 = __dmul_rn(static_cast<double>(w[2]), t.iz[2]);
      const float d = __double2float_rn(__ddiv_rn(static_cast<double>(t.area), __dadd_rn(__dadd_rn(t0, t1), t2)));
      const unsigned long long key =
          (static_cast<unsigned long long>(__float_as_uint(d)) << 32) | static_cast<unsigned>(face);
      unsigned long long *px = keys + b * hw + static_cast<size_t>(v) * f.w + u;
      // keys only fall during the launch: a stale read can only be larger, so skipping on <= is safe
      if (*reinterpret_cast<volatile unsigned long long *>(px) > key) atomicMin(px, key);
    }
  }
}

// ---- 5. resolve -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kResolveThreads)
    render_resolve_kernel(const __grid_constant__ Mesh m, const __grid_constant__ Frames f, const Vtx *__restrict__ vtx,
                          const unsigned long long *__restrict__ keys, const uint8_t *__restrict__ back_rgb,
                          const float *__restrict__ back_depth, uint8_t *__restrict__ rgb, float *__restrict__ depth,
                          uint8_t *__restrict__ labels) {
  __shared__ int s_voff[kMaxCls + 1], s_foff[kMaxCls + 1];
  for (int i = threadIdx.x; i <= m.n_cls; i += blockDim.x) s_foff[i] = m.face_off[i];
  load_offsets(s_voff, m.vtx_off, m.n_cls);
  const long long hw = static_cast<long long>(f.h) * f.w, total = hw * f.b;
  for (long long p = blockIdx.x * static_cast<long long>(kResolveThreads) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * kResolveThreads) {
    const unsigned long long key = __ldcs(keys + p);
    uint8_t *o = rgb + p * 3;
    if (key == kEmpty) {
      if (back_rgb) {
        o[0] = back_rgb[p * 3];
        o[1] = back_rgb[p * 3 + 1];
        o[2] = back_rgb[p * 3 + 2];
        depth[p] = back_depth[p];
      } else {
        o[0] = o[1] = o[2] = 0;
        depth[p] = 0.0f;
      }
      labels[p] = 0;
      continue;
    }
    const int b = static_cast<int>(p / hw);
    const int rem = static_cast<int>(p - b * hw), v = rem / f.w, u = rem - v * f.w;
    const int face = static_cast<int>(key & 0xffffffffu);
    const int c = owner(s_foff, m.n_cls, face);
    Tri t;
    tri_setup(m, f, vtx + static_cast<size_t>(b) * m.n_vtx, s_voff, face, c, t);   // the winner: always set up
    long long w[3];
    inside(t, u, v, w);
    const double t0 = __dmul_rn(static_cast<double>(w[0]), t.iz[0]);
    const double t1 = __dmul_rn(static_cast<double>(w[1]), t.iz[1]);
    const double t2 = __dmul_rn(static_cast<double>(w[2]), t.iz[2]);
    const double n = __dadd_rn(__dadd_rn(t0, t1), t2);
    const uint8_t *c0 = m.col + static_cast<size_t>(t.v[0]) * 3, *c1 = m.col + static_cast<size_t>(t.v[1]) * 3,
                  *c2 = m.col + static_cast<size_t>(t.v[2]) * 3;
    for (int ch = 0; ch < 3; ++ch) {
      const double s = __dadd_rn(__dadd_rn(__dmul_rn(t0, static_cast<double>(c0[ch])),
                                           __dmul_rn(t1, static_cast<double>(c1[ch]))),
                                 __dmul_rn(t2, static_cast<double>(c2[ch])));
      o[ch] = static_cast<uint8_t>(fmin(fmax(rint(__ddiv_rn(s, n)), 0.0), 255.0));
    }
    depth[p] = __uint_as_float(static_cast<unsigned>(key >> 32));
    labels[p] = static_cast<uint8_t>(c);
  }
}

struct Layout {
  size_t keys, vtx, incl, blk, excl, total;
  int nb;
};

// 0 bytes = refused sizes
Layout layout(int b, int h, int w, int n_vtx, int n_faces) {
  Layout l{};
  if (b < 1 || h < 1 || w < 1 || n_vtx < 1 || n_faces < 1 || h > kMaxSide || w > kMaxSide) return l;
  const long long slots = static_cast<long long>(b) * n_faces;
  if (slots >= (1ll << 31) || static_cast<long long>(b) * n_vtx >= (1ll << 31) || b > 65535) return l;
  l.nb = static_cast<int>((slots + kScanBlock - 1) / kScanBlock);
  size_t off = 0;
  l.keys = off;
  off = align_up(off + static_cast<size_t>(b) * h * w * sizeof(unsigned long long), 256);
  l.vtx = off;
  off = align_up(off + static_cast<size_t>(b) * n_vtx * sizeof(Vtx), 256);
  l.incl = off;
  off = align_up(off + static_cast<size_t>(l.nb) * kScanBlock * sizeof(unsigned long long), 256);
  l.blk = off;
  off = align_up(off + static_cast<size_t>(l.nb) * sizeof(unsigned long long), 256);
  l.excl = off;
  off = align_up(off + static_cast<size_t>(l.nb + 1) * sizeof(unsigned long long), 256);
  l.total = off;
  return l;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_render_workspace_bytes(int b, int h, int w, int n_vtx, int n_faces) {
  return layout(b, h, w, n_vtx, n_faces).total;
}

extern "C" int pvn3d_render_meshes(const float *vtx, const uint8_t *colors, const int *faces, const int *vtx_off,
                                   const int *face_off, int n_cls, int n_vtx, int n_faces, const void *poses,
                                   int poses_f64, const uint8_t *present, const double *k, int b, int h, int w,
                                   double z_near, const uint8_t *back_rgb, const float *back_depth, uint8_t *rgb,
                                   float *depth, uint8_t *labels, void *workspace, size_t workspace_bytes,
                                   pvn3d_stream_t stream) {
  if (!vtx || !colors || !faces || !vtx_off || !face_off || !poses || !present || !k || !rgb || !depth || !labels ||
      (poses_f64 != 0 && poses_f64 != 1) || n_cls < 2 || n_vtx < 1 || n_faces < 1 || b < 1 || h < 1 || w < 1 ||
      !(z_near > 0.0) || isinf(z_near) || (!back_rgb != !back_depth))
    return PVN3D_ERR_INVALID_ARG;
  if (n_cls > kMaxCls || h > kMaxSide || w > kMaxSide) return PVN3D_ERR_UNSUPPORTED;
  const Layout l = layout(b, h, w, n_vtx, n_faces);
  if (l.total == 0) return PVN3D_ERR_UNSUPPORTED;
  if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255u)) return PVN3D_ERR_INVALID_ARG;
  if (workspace_bytes < l.total) return PVN3D_ERR_WORKSPACE;
  char *ws = static_cast<char *>(workspace);
  auto *keys = reinterpret_cast<unsigned long long *>(ws + l.keys);
  auto *vrec = reinterpret_cast<Vtx *>(ws + l.vtx);
  auto *incl = reinterpret_cast<unsigned long long *>(ws + l.incl);
  auto *blk = reinterpret_cast<unsigned long long *>(ws + l.blk);
  auto *excl = reinterpret_cast<unsigned long long *>(ws + l.excl);
  const Mesh m{vtx, colors, faces, vtx_off, face_off, n_cls, n_vtx, n_faces};
  const Frames fr{poses, poses_f64, present, k, z_near, b, h, w};
  const cudaStream_t st = as_stream(stream);
  const long long pixels = static_cast<long long>(b) * h * w;
  const long long persistent = static_cast<long long>(sm_count()) * 8;
  int rc;
  PVN3D_CUDA_TRY(cudaMemsetAsync(keys, 0xff, static_cast<size_t>(pixels) * sizeof(unsigned long long), st),
                 "render key memset");
  const long long vblocks = min((static_cast<long long>(b) * n_vtx + kVtxThreads - 1) / kVtxThreads, persistent * 2);
  render_vertex_kernel<<<static_cast<unsigned>(vblocks), kVtxThreads, 0, st>>>(m, fr, vrec);
  if ((rc = check_launch("render_vertex_kernel")) != PVN3D_OK) return rc;
  render_setup_kernel<<<static_cast<unsigned>(l.nb), kScanBlock, 0, st>>>(m, fr, vrec, incl, blk);
  if ((rc = check_launch("render_setup_kernel")) != PVN3D_OK) return rc;
  render_scan_kernel<<<1, kScanBlock, 0, st>>>(blk, l.nb, excl);
  if ((rc = check_launch("render_scan_kernel")) != PVN3D_OK) return rc;
  render_fragment_kernel<<<static_cast<unsigned>(persistent), kFragThreads, 0, st>>>(m, fr, vrec, incl, excl, l.nb,
                                                                                    keys);
  if ((rc = check_launch("render_fragment_kernel")) != PVN3D_OK) return rc;
  const long long rblocks = min((pixels + kResolveThreads - 1) / kResolveThreads, persistent * 2);
  render_resolve_kernel<<<static_cast<unsigned>(rblocks), kResolveThreads, 0, st>>>(m, fr, vrec, keys, back_rgb,
                                                                                   back_depth, rgb, depth, labels);
  return check_launch("render_resolve_kernel");
}
