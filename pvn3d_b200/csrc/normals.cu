// normals.cu -- the network input of an RGB-D frame, as the datasets' get_item builds it on the CPU
// (pvn3d/datasets/{ycb,linemod}/*_dataset.py): a seeded subset of the valid pixels (choose_2), the
// assembly of cld_rgb_nrm / pcld / choose, and point normals from the exact 50 nearest neighbours
// (PCL's NormalEstimation with setKSearch(50), get_normal).
//
// Sampling, one CTA per frame, no host round trip:
//   key(seed, b, p) = mix(mix(seed + (b + 1) * 0x9E3779B97F4A7C15) + p)   (uint64 wrap-around,
//   mix = the splitmix64 finaliser).  mix is a bijection, so the keys of one frame are distinct.
//   n_v valid pixels: n_v > N keeps the N smallest keys (an 8-pass radix select of the N-th key),
//   400 <= n_v <= N takes every valid pixel repeated cyclically (np.pad 'wrap'), n_v < 400 is not a
//   frame (ok = 0, zeros).  The chosen pixels are emitted in ascending raster order.
//
// Normals, one warp per query: the exact 50 nearest reference points by the float64 squared
// distance (dx*dx + dy*dy) + dz*dz of the float32 coordinates (no FMA), lowest index first on exact
// ties; the query is its own neighbour at distance 0.  The warp holds the sorted top 50 across its
// lanes (slot l and slot l + 32 in lane l).  C = (1/50) sum (p - mean)(p - mean)^T in float64, two
// passes; n = the unit eigenvector of C's smallest eigenvalue (cyclic Jacobi), flipped so that
// n . (0 - p) >= 0 (PCL's flipNormalTowardsViewpoint, viewpoint at the origin).  trace(C) == 0, or
// fewer than 50 usable reference points, gives n = (0, 0, 0) and curvature 0.
//
// Search structure (private to this file): per frame, a uniform grid over the bounding box of the
// usable (valid, finite) reference points with about two cells per point (at most 2 * n_ref + 64),
// a power-of-two cell edge on an origin that is a multiple of it (cell faces are exact), cell
// ranges, and the points sorted by cell as float4 (x, y, z, index bits).  It is built on the stream
// by five small kernels over all points of the batch.  The walk visits shells of cells around the
// query's cell and stops when a conservative lower bound on the distance to every unvisited cell
// exceeds the 50th best distance.
#include <cmath>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kK = 50;  // PCL's setKSearch(50) in get_normal
constexpr int kMinValid = 400;
constexpr int kSampleThreads = 1024;
constexpr int kAssembleThreads = 256;
constexpr int kGridThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kSearchThreads = 256;
constexpr unsigned kFull = 0xffffffffu;
// lower bounds are compared as lb * (1 - kRel) > best: the relative slack covers their own rounding
constexpr double kRel = 1e-9;

bool fits_int32(long long v) { return v < 0x80000000ll; }

// ------------------------------------------------------------------------------------------------
// sampling
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ unsigned long long frame_base(unsigned long long seed, int b) {
  return mix64(seed + static_cast<unsigned long long>(b + 1) * 0x9E3779B97F4A7C15ull);
}

struct SampleWs {
  size_t thresh, nv, total;
};
SampleWs sample_ws_layout(int b) {
  SampleWs L;
  L.thresh = 0;
  L.nv = align_up(static_cast<size_t>(b) * 8, 256);
  L.total = L.nv + align_up(static_cast<size_t>(b) * 4, 256);
  return L;
}

// per frame: n_v and the N-th smallest key among the valid pixels (all ones when n_v <= N)
__global__ void __launch_bounds__(kSampleThreads)
sample_select_kernel(const uint8_t *__restrict__ valid, int hw, int n, unsigned long long seed,
                     unsigned long long *__restrict__ thresh, int *__restrict__ nv_out) {
  __shared__ unsigned hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ unsigned s_rank, s_nv;
  const int b = blockIdx.x, t = threadIdx.x;
  const uint8_t *v = valid + static_cast<size_t>(b) * hw;
  const unsigned long long base = frame_base(seed, b);
  if (t == 0) {
    s_prefix = 0ull;
    s_rank = static_cast<unsigned>(n);
  }
  unsigned long long mask = 0ull;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = t; i < 256; i += kSampleThreads) hist[i] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    for (int p = t; p < hw; p += kSampleThreads) {
      if (!v[p]) continue;
      const unsigned long long key = mix64(base + static_cast<unsigned long long>(p));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (t == 0) {
      if (shift == 56) {
        unsigned tot = 0;
        for (int d = 0; d < 256; ++d) tot += hist[d];
        s_nv = tot;
      }
      unsigned rank = s_rank, d = 0;
      for (; d < 255 && hist[d] < rank; ++d) rank -= hist[d];
      s_rank = rank;
      s_prefix = prefix | (static_cast<unsigned long long>(d) << shift);
    }
    __syncthreads();
    if (s_nv <= static_cast<unsigned>(n)) break;  // nothing to select: every valid pixel is kept
    mask |= 255ull << shift;
  }
  if (t == 0) {
    nv_out[b] = static_cast<int>(s_nv);
    thresh[b] = s_nv > static_cast<unsigned>(n) ? s_prefix : ~0ull;
  }
}

// per frame: the chosen pixels in raster order (wrapped to N when n_v <= N), ok = n_v >= 400
__global__ void __launch_bounds__(kSampleThreads)
sample_compact_kernel(const uint8_t *__restrict__ valid, int hw, int n, unsigned long long seed,
                      const unsigned long long *__restrict__ thresh, const int *__restrict__ nv_in,
                      long long *__restrict__ choose, uint8_t *__restrict__ ok) {
  __shared__ int s_warp[kSampleThreads / 32];
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = t & 31u, warp = t >> 5;
  const int nv = nv_in[b];
  long long *out = choose + static_cast<size_t>(b) * n;
  if (nv < kMinValid) {
    for (int j = t; j < n; j += kSampleThreads) out[j] = 0;
    if (t == 0) ok[b] = 0;
    return;
  }
  const uint8_t *v = valid + static_cast<size_t>(b) * hw;
  const unsigned long long base = frame_base(seed, b), T = thresh[b];
  const int kept = nv < n ? nv : n;
  int run = 0;
  for (int p0 = 0; p0 < hw && run < kept; p0 += kSampleThreads) {
    const int p = p0 + t;
    const bool take = p < hw && v[p] && mix64(base + static_cast<unsigned long long>(p)) <= T;
    const unsigned bal = __ballot_sync(kFull, take);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < kSampleThreads / 32; ++w) {
      const int c = s_warp[w];
      before += w < static_cast<int>(warp) ? c : 0;
      total += c;
    }
    if (take) out[run + before + __popc(bal & lanemask_lt())] = p;
    run += total;
    __syncthreads();
  }
  // np.pad(choose_2, (0, N - n_v), 'wrap'); the stores above are visible to the block after the barrier
  for (int j = kept + t; j < n; j += kSampleThreads) out[j] = out[j % kept];
  if (t == 0) ok[b] = 1;
}

// cld_rgb_nrm[b, j, 0:6] = (cloud, rgb) at choose[b, j]; pcld; labels.  A frame with ok = 0 gets zeros.
__global__ void __launch_bounds__(kAssembleThreads)
assemble_kernel(const float *__restrict__ cloud, const void *__restrict__ rgb, int rgb_u8,
                const int *__restrict__ label_image, int hw, int n, int total, const long long *__restrict__ choose,
                const uint8_t *__restrict__ ok, float *__restrict__ cld_rgb_nrm, long long stride,
                float *__restrict__ pcld, int *__restrict__ labels) {
  const int g = blockIdx.x * kAssembleThreads + threadIdx.x;
  if (g >= total) return;
  const int b = g / n;
  float *row = cld_rgb_nrm + static_cast<size_t>(g) * stride;
  float *pc = pcld + static_cast<size_t>(g) * 3;
  if (!ok[b]) {
    for (int c = 0; c < 6; ++c) row[c] = 0.f;
    for (int c = 0; c < 3; ++c) pc[c] = 0.f;
    if (labels) labels[g] = 0;
    return;
  }
  const size_t p = static_cast<size_t>(choose[g]);
  const float *src = cloud + (static_cast<size_t>(b) * hw + p) * 3;
  for (int c = 0; c < 3; ++c) {
    const float x = src[c];
    row[c] = x;
    pc[c] = x;
  }
  const size_t px = static_cast<size_t>(b) * 3 * hw + p;
  for (int c = 0; c < 3; ++c)
    row[3 + c] = rgb_u8 ? static_cast<float>(static_cast<const uint8_t *>(rgb)[px + static_cast<size_t>(c) * hw])
                        : static_cast<const float *>(rgb)[px + static_cast<size_t>(c) * hw];
  if (labels) labels[g] = label_image[static_cast<size_t>(b) * hw + p];
}

// ------------------------------------------------------------------------------------------------
// the per-frame grid
// ------------------------------------------------------------------------------------------------
struct GridHdr {  // 64 bytes
  double lo[3];
  double h;       // cell edge
  double margin;  // absolute slack of every lower bound (covers cell-assignment rounding)
  int dims[3];
  int n_pts;      // usable points of the frame
};

// bounding box as order-preserving unsigned keys of the float coordinates, and the usable count
struct GridBox {
  unsigned mn[3], mx[3];
  unsigned count, pad;
};

int grid_cap(int n_ref) { return 2 * n_ref + 64; }

struct KnnWs {
  size_t hdr, box, cell_start, cursor, pts, total;
};
KnnWs knn_ws_layout(int b, int n_ref) {
  KnnWs L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t at = off;
    off = align_up(off + (bytes ? bytes : 1), 256);
    return at;
  };
  const size_t nb = static_cast<size_t>(b), cap = static_cast<size_t>(grid_cap(n_ref));
  L.hdr = take(nb * sizeof(GridHdr));
  L.box = take(nb * sizeof(GridBox));
  L.cell_start = take(nb * (cap + 1) * 4);
  L.cursor = take(nb * cap * 4);
  L.pts = take(nb * static_cast<size_t>(n_ref) * 16);
  L.total = off;
  return L;
}

__device__ __forceinline__ unsigned f2ord(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ bool usable(const float *ref, const uint8_t *valid, size_t i, float &x, float &y,
                                       float &z) {
  if (valid && !valid[i]) return false;
  x = ref[i * 3 + 0];
  y = ref[i * 3 + 1];
  z = ref[i * 3 + 2];
  return isfinite(x) && isfinite(y) && isfinite(z);
}

__device__ __forceinline__ int cell_coord(double v, double lo, double h, int dim) {
  const double f = floor((v - lo) / h);
  return f >= dim - 1 ? dim - 1 : (f > 0.0 ? static_cast<int>(f) : 0);
}

__device__ __forceinline__ int cell_of(const GridHdr &H, float x, float y, float z) {
  const int cx = cell_coord(x, H.lo[0], H.h, H.dims[0]);
  const int cy = cell_coord(y, H.lo[1], H.h, H.dims[1]);
  const int cz = cell_coord(z, H.lo[2], H.h, H.dims[2]);
  return (cz * H.dims[1] + cy) * H.dims[0] + cx;
}

__global__ void grid_init_kernel(int b, GridBox *__restrict__ box) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b) return;
  GridBox g;
  for (int d = 0; d < 3; ++d) {
    g.mn[d] = 0xffffffffu;
    g.mx[d] = 0u;
  }
  g.count = 0;
  g.pad = 0;
  box[f] = g;
}

// blockIdx.y = frame
__global__ void __launch_bounds__(kGridThreads)
grid_bbox_kernel(const float *__restrict__ ref, const uint8_t *__restrict__ valid, int n_ref,
                 GridBox *__restrict__ box) {
  const int b = blockIdx.y;
  unsigned mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u}, cnt = 0;
  for (int i = blockIdx.x * kGridThreads + threadIdx.x; i < n_ref; i += gridDim.x * kGridThreads) {
    float p[3];
    if (!usable(ref, valid, static_cast<size_t>(b) * n_ref + i, p[0], p[1], p[2])) continue;
    ++cnt;
    for (int d = 0; d < 3; ++d) {
      const unsigned k = f2ord(p[d]);
      mn[d] = min(mn[d], k);
      mx[d] = max(mx[d], k);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(kFull, cnt, o);
    for (int d = 0; d < 3; ++d) {
      mn[d] = min(mn[d], __shfl_xor_sync(kFull, mn[d], o));
      mx[d] = max(mx[d], __shfl_xor_sync(kFull, mx[d], o));
    }
  }
  if ((threadIdx.x & 31u) == 0 && cnt) {
    GridBox *g = box + b;
    atomicAdd(&g->count, cnt);
    for (int d = 0; d < 3; ++d) {
      atomicMin(&g->mn[d], mn[d]);
      atomicMax(&g->mx[d], mx[d]);
    }
  }
}

__global__ void grid_setup_kernel(int b, int cap, const GridBox *__restrict__ box, GridHdr *__restrict__ hdr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b) return;
  const GridBox g = box[f];
  GridHdr h{};
  h.n_pts = static_cast<int>(g.count);
  if (g.count == 0) {
    for (int d = 0; d < 3; ++d) {
      h.lo[d] = 0.0;
      h.dims[d] = 1;
    }
    h.h = 1.0;
    h.margin = 0.0;
    hdr[f] = h;
    return;
  }
  double lo[3], hi[3], e[3], emax = 0.0;
  for (int d = 0; d < 3; ++d) {
    lo[d] = ord2f(g.mn[d]);
    hi[d] = ord2f(g.mx[d]);
    emax = fmax(emax, hi[d] - lo[d]);
  }
  // flat and one-point clouds count zero-width axes as thin slabs
  const double floor_e = 1e-3 * emax + 1e-9;
  for (int d = 0; d < 3; ++d) e[d] = fmax(hi[d] - lo[d], floor_e);
  const double target = fmin(static_cast<double>(cap), 2.0 * g.count);
  // a power-of-two edge on an origin that is a multiple of it: every cell face lo + k*h is exact
  double cell = exp2(rint(log2(cbrt(e[0] * e[1] * e[2] / target))));
  double glo[3], gdim[3];
  for (;;) {
    double prod = 1.0;
    for (int d = 0; d < 3; ++d) {
      glo[d] = floor(lo[d] / cell) * cell;
      gdim[d] = floor((hi[d] - glo[d]) / cell) + 1.0;
      prod *= gdim[d];
    }
    if (prod <= cap) break;
    cell *= 2.0;
  }
  double cmax = 0.0;
  for (int d = 0; d < 3; ++d) {
    h.dims[d] = static_cast<int>(gdim[d]);
    h.lo[d] = glo[d];
    cmax = fmax(cmax, fmax(fabs(glo[d]), fabs(glo[d] + gdim[d] * cell)));
  }
  h.h = cell;
  h.margin = 1e-6 * cell + 1e-13 * cmax;
  hdr[f] = h;
}

__global__ void __launch_bounds__(kGridThreads)
grid_count_kernel(const float *__restrict__ ref, const uint8_t *__restrict__ valid, int n_ref, int cap,
                  const GridHdr *__restrict__ hdr, int *__restrict__ counts) {
  const int b = blockIdx.y;
  const GridHdr H = hdr[b];
  int *cnt = counts + static_cast<size_t>(b) * cap;
  for (int i = blockIdx.x * kGridThreads + threadIdx.x; i < n_ref; i += gridDim.x * kGridThreads) {
    float x, y, z;
    if (usable(ref, valid, static_cast<size_t>(b) * n_ref + i, x, y, z)) atomicAdd(&cnt[cell_of(H, x, y, z)], 1);
  }
}

// exclusive scan of the counts (in `cursor`) into cell_start, and cursor = cell_start: one CTA per frame
__global__ void __launch_bounds__(kScanThreads)
grid_scan_kernel(int cap, const GridHdr *__restrict__ hdr, int *__restrict__ cell_start, int *__restrict__ cursor) {
  __shared__ int s_scan[kScanThreads / 32];
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = t & 31u, warp = t >> 5;
  const GridHdr H = hdr[b];
  const int ncell = H.dims[0] * H.dims[1] * H.dims[2];
  int *cs = cell_start + static_cast<size_t>(b) * (cap + 1);
  int *cur = cursor + static_cast<size_t>(b) * cap;
  const int per = (ncell + kScanThreads - 1) / kScanThreads;
  const int c0 = min(t * per, ncell), c1 = min(c0 + per, ncell);
  int local = 0;
  for (int c = c0; c < c1; ++c) local += cur[c];
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(kFull, incl, o);
    if (lane >= static_cast<unsigned>(o)) incl += u;
  }
  if (lane == 31) s_scan[warp] = incl;
  __syncthreads();
  int before = 0;
  for (int w = 0; w < static_cast<int>(warp); ++w) before += s_scan[w];
  int run = before + incl - local;
  for (int c = c0; c < c1; ++c) {
    const int cnt = cur[c];
    cs[c] = run;
    cur[c] = run;
    run += cnt;
  }
  if (t == 0) cs[ncell] = H.n_pts;
}

// order inside a cell is irrelevant: the search ranks by (distance, index)
__global__ void __launch_bounds__(kGridThreads)
grid_scatter_kernel(const float *__restrict__ ref, const uint8_t *__restrict__ valid, int n_ref, int cap,
                    const GridHdr *__restrict__ hdr, int *__restrict__ cursor, float4 *__restrict__ pts) {
  const int b = blockIdx.y;
  const GridHdr H = hdr[b];
  int *cur = cursor + static_cast<size_t>(b) * cap;
  float4 *sp = pts + static_cast<size_t>(b) * n_ref;
  for (int i = blockIdx.x * kGridThreads + threadIdx.x; i < n_ref; i += gridDim.x * kGridThreads) {
    float x, y, z;
    if (!usable(ref, valid, static_cast<size_t>(b) * n_ref + i, x, y, z)) continue;
    const int pos = atomicAdd(&cur[cell_of(H, x, y, z)], 1);
    sp[pos] = make_float4(x, y, z, __int_as_float(i));
  }
}

// ------------------------------------------------------------------------------------------------
// exact 50 nearest neighbours and the normal, one warp per query
// ------------------------------------------------------------------------------------------------
// (dx*dx + dy*dy) + dz*dz in float64, no fused multiply-add
__device__ __forceinline__ double sqdist64(const double q[3], float x, float y, float z) {
  const double dx = __dsub_rn(q[0], static_cast<double>(x)), dy = __dsub_rn(q[1], static_cast<double>(y)),
               dz = __dsub_rn(q[2], static_cast<double>(z));
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ bool key_lt(double d, int i, double e, int j) { return d < e || (d == e && i < j); }

// the warp's sorted list: lane l holds slots l (da, ia) and l + 32 (db, ib); (d, i) is warp-uniform
__device__ __forceinline__ void topk_insert(double &da, int &ia, double &db, int &ib, double d, int i) {
  const unsigned lane = threadIdx.x & 31u;
  const int pos = __popc(__ballot_sync(kFull, key_lt(da, ia, d, i))) + __popc(__ballot_sync(kFull, key_lt(db, ib, d, i)));
  const double pa = __shfl_up_sync(kFull, da, 1), a31 = __shfl_sync(kFull, da, 31);
  const int pia = __shfl_up_sync(kFull, ia, 1), ia31 = __shfl_sync(kFull, ia, 31);
  double pb = __shfl_up_sync(kFull, db, 1);
  int pib = __shfl_up_sync(kFull, ib, 1);
  if (lane == 0) {
    pb = a31;
    pib = ia31;
  }
  const int sa = static_cast<int>(lane), sb = sa + 32;
  if (sa > pos) {
    da = pa;
    ia = pia;
  } else if (sa == pos) {
    da = d;
    ia = i;
  }
  if (sb > pos) {
    db = pb;
    ib = pib;
  } else if (sb == pos) {
    db = d;
    ib = i;
  }
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// one Jacobi rotation zeroing a[p][q] of the symmetric a, accumulated into the columns of v
template <int P, int Q, int R>
__device__ __forceinline__ void jacobi_rot(double (&a)[3][3], double (&v)[3][3]) {
  const double apq = a[P][Q];
  if (apq == 0.0) return;
  const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
  const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c), hh = t * apq;
  a[P][P] -= hh;
  a[Q][Q] += hh;
  a[P][Q] = a[Q][P] = 0.0;
  const double g = a[R][P], h = a[R][Q];
  a[R][P] = a[P][R] = g - s * (h + g * tau);
  a[R][Q] = a[Q][R] = h + s * (g - h * tau);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double vp = v[r][P], vq = v[r][Q];
    v[r][P] = vp - s * (vq + vp * tau);
    v[r][Q] = vq + s * (vp - vq * tau);
  }
}

// unit eigenvector n and eigenvalue of the smallest eigenvalue of the symmetric positive semi-definite c
__device__ __forceinline__ void smallest_eigvec(const double c[6], double n[3], double &lam) {
  double a[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 50; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    const double dia = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
    if (!(off > 1e-40 * dia)) break;
    jacobi_rot<0, 1, 2>(a, v);
    jacobi_rot<0, 2, 1>(a, v);
    jacobi_rot<1, 2, 0>(a, v);
  }
  // column of the smallest diagonal entry, selected without a dynamic index (keeps a and v in registers)
  lam = a[0][0];
  double w[3] = {v[0][0], v[1][0], v[2][0]};
  if (a[1][1] < lam) {
    lam = a[1][1];
    for (int r = 0; r < 3; ++r) w[r] = v[r][1];
  }
  if (a[2][2] < lam) {
    lam = a[2][2];
    for (int r = 0; r < 3; ++r) w[r] = v[r][2];
  }
  const double nn = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  for (int r = 0; r < 3; ++r) n[r] = w[r] / nn;
}

struct KnnParams {
  const float *ref;
  const uint8_t *ref_valid;
  const float *query;
  const uint8_t *frame_ok;
  const GridHdr *hdr;
  const int *cell_start;
  const float4 *pts;
  int n_ref, nq, b, cap;
  float *normals;
  long long stride;
  float *curv;
  double *normals64;
  int *nn;
};

__global__ void __launch_bounds__(kSearchThreads, 2) knn_normals_kernel(const KnnParams p) {
  const int gw = (blockIdx.x * kSearchThreads + static_cast<int>(threadIdx.x)) >> 5;
  const unsigned lane = threadIdx.x & 31u;
  if (gw >= p.b * p.nq) return;  // warp-uniform
  const int b = gw / p.nq;
  const float *qp = p.query + static_cast<size_t>(gw) * 3;
  const double q[3] = {qp[0], qp[1], qp[2]};
  const GridHdr H = p.hdr[b];
  const bool run = (!p.frame_ok || p.frame_ok[b]) && H.n_pts >= kK && isfinite(q[0]) && isfinite(q[1]) &&
                   isfinite(q[2]);
  double da = INFINITY, db = INFINITY;
  int ia = 0x7fffffff, ib = 0x7fffffff;
  if (run) {
    const int *cs = p.cell_start + static_cast<size_t>(b) * (p.cap + 1);
    const float4 *P = p.pts + static_cast<size_t>(b) * p.n_ref;
    const double scale = 1.0 - kRel;
    int c0[3];
    double g0[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      c0[d] = cell_coord(q[d], H.lo[d], H.h, H.dims[d]);
      const double slo = H.lo[d] + c0[d] * H.h;
      g0[d] = fmax(0.0, fmax(slo - q[d], q[d] - (slo + H.h)) - H.margin);
    }
    double kd = INFINITY;
    int ki = 0x7fffffff;
    const int dimx = H.dims[0], dimy = H.dims[1], dimz = H.dims[2];
    for (int r = 0;; ++r) {
      if (r > 0) {
        // every cell of shells >= r lies at index distance >= r along some axis
        double lb = INFINITY;
        bool any = false;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          double base = 0.0;
#pragma unroll
          for (int e = 0; e < 3; ++e)
            if (e != d) base += g0[e] * g0[e];
          if (c0[d] - r >= 0) {
            const double gap = fmax(0.0, q[d] - (H.lo[d] + (c0[d] - r + 1) * H.h) - H.margin);
            lb = fmin(lb, base + gap * gap);
            any = true;
          }
          if (c0[d] + r < H.dims[d]) {
            const double gap = fmax(0.0, (H.lo[d] + (c0[d] + r) * H.h) - q[d] - H.margin);
            lb = fmin(lb, base + gap * gap);
            any = true;
          }
        }
        if (!any || lb * scale > kd) break;
      }
      const int z0 = max(c0[2] - r, 0), z1 = min(c0[2] + r, dimz - 1);
      const int y0 = max(c0[1] - r, 0), y1 = min(c0[1] + r, dimy - 1);
      for (int z = z0; z <= z1; ++z) {
        const double gz = fmax(0.0, fmax(H.lo[2] + z * H.h - q[2], q[2] - (H.lo[2] + (z + 1) * H.h)) - H.margin);
        const bool ez = (z == c0[2] - r) || (z == c0[2] + r);
        for (int y = y0; y <= y1; ++y) {
          const double gy = fmax(0.0, fmax(H.lo[1] + y * H.h - q[1], q[1] - (H.lo[1] + (y + 1) * H.h)) - H.margin);
          const bool full = ez || (y == c0[1] - r) || (y == c0[1] + r);
          const int step = (full || r == 0) ? 1 : 2 * r;  // interior rows of the shell: only the two end cells
          for (int x = c0[0] - r; x <= c0[0] + r; x += step) {
            if (x < 0 || x >= dimx) continue;
            const double gx = fmax(0.0, fmax(H.lo[0] + x * H.h - q[0], q[0] - (H.lo[0] + (x + 1) * H.h)) - H.margin);
            if ((gx * gx + gy * gy + gz * gz) * scale > kd) continue;
            const int c = (z * dimy + y) * dimx + x;
            const int e = cs[c + 1];
            for (int k0 = cs[c]; k0 < e; k0 += 32) {
              const int k = k0 + static_cast<int>(lane);
              double d2 = INFINITY;
              int idx = 0x7fffffff;
              if (k < e) {
                const float4 v = P[k];
                d2 = sqdist64(q, v.x, v.y, v.z);
                idx = __float_as_int(v.w);
              }
              unsigned m = __ballot_sync(kFull, key_lt(d2, idx, kd, ki));
              while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                const double dd = __shfl_sync(kFull, d2, src);
                const int ii = __shfl_sync(kFull, idx, src);
                if (!key_lt(dd, ii, kd, ki)) continue;
                topk_insert(da, ia, db, ib, dd, ii);
                kd = __shfl_sync(kFull, db, kK - 33);
                ki = __shfl_sync(kFull, ib, kK - 33);
              }
            }
          }
        }
      }
    }
  }
  const size_t row = static_cast<size_t>(gw);
  if (p.nn) {
    int *o = p.nn + row * kK;
    o[lane] = da < INFINITY ? ia : -1;
    if (lane + 32 < kK) o[lane + 32] = db < INFINITY ? ib : -1;
  }
  double n[3] = {0.0, 0.0, 0.0}, curv = 0.0;
  if (run && __shfl_sync(kFull, db, kK - 33) < INFINITY) {
    const float *ref = p.ref + static_cast<size_t>(b) * p.n_ref * 3;
    const bool hb = lane + 32 < kK;
    double xa[3], xb[3] = {0.0, 0.0, 0.0}, mean[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      xa[d] = ref[static_cast<size_t>(ia) * 3 + d];
      if (hb) xb[d] = ref[static_cast<size_t>(ib) * 3 + d];
      mean[d] = warp_sum(xa[d] + xb[d]) / kK;
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      xa[d] -= mean[d];
      xb[d] = hb ? xb[d] - mean[d] : 0.0;
    }
    double c[6];
    c[0] = warp_sum(xa[0] * xa[0] + xb[0] * xb[0]) / kK;
    c[1] = warp_sum(xa[0] * xa[1] + xb[0] * xb[1]) / kK;
    c[2] = warp_sum(xa[0] * xa[2] + xb[0] * xb[2]) / kK;
    c[3] = warp_sum(xa[1] * xa[1] + xb[1] * xb[1]) / kK;
    c[4] = warp_sum(xa[1] * xa[2] + xb[1] * xb[2]) / kK;
    c[5] = warp_sum(xa[2] * xa[2] + xb[2] * xb[2]) / kK;
    const double tr = c[0] + c[3] + c[5];
    if (tr > 0.0) {
      double lam;
      smallest_eigvec(c, n, lam);
      if (n[0] * q[0] + n[1] * q[1] + n[2] * q[2] > 0.0)
        for (int d = 0; d < 3; ++d) n[d] = -n[d];
      curv = fmax(lam, 0.0) / tr;
    }
  }
  if (lane == 0) {
    float *o = p.normals + row * p.stride;
    for (int d = 0; d < 3; ++d) o[d] = static_cast<float>(n[d]);
    if (p.curv) p.curv[row] = static_cast<float>(curv);
    if (p.normals64)
      for (int d = 0; d < 3; ++d) p.normals64[row * 3 + d] = n[d];
  }
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_frame_sample_workspace_bytes(int b, int hw, int n) {
  if (b < 1 || hw < 1 || n < 1 || !fits_int32(static_cast<long long>(b) * hw) ||
      !fits_int32(static_cast<long long>(b) * n))
    return 0;
  return sample_ws_layout(b).total;
}

extern "C" int pvn3d_frame_sample(const float *cloud, const uint8_t *valid, const void *rgb, int rgb_u8,
                                  const int *label_image, int b, int hw, int n, unsigned long long seed,
                                  float *cld_rgb_nrm, long long row_stride, float *pcld, long long *choose,
                                  int *labels_out, uint8_t *ok, void *workspace, size_t workspace_bytes,
                                  pvn3d_stream_t stream) {
  if (!cloud || !valid || !rgb || !cld_rgb_nrm || !pcld || !choose || !ok || !workspace || b < 1 || hw < 1 ||
      n < 1 || row_stride < 6 || (labels_out && !label_image) || (rgb_u8 != 0 && rgb_u8 != 1))
    return PVN3D_ERR_INVALID_ARG;
  if (!fits_int32(static_cast<long long>(b) * hw) || !fits_int32(static_cast<long long>(b) * n))
    return PVN3D_ERR_UNSUPPORTED;
  const SampleWs L = sample_ws_layout(b);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  auto *thresh = reinterpret_cast<unsigned long long *>(ws + L.thresh);
  int *nv = reinterpret_cast<int *>(ws + L.nv);
  cudaStream_t st = as_stream(stream);
  sample_select_kernel<<<b, kSampleThreads, 0, st>>>(valid, hw, n, seed, thresh, nv);
  int rc = check_launch("sample_select_kernel");
  if (rc != PVN3D_OK) return rc;
  sample_compact_kernel<<<b, kSampleThreads, 0, st>>>(valid, hw, n, seed, thresh, nv, choose, ok);
  if ((rc = check_launch("sample_compact_kernel")) != PVN3D_OK) return rc;
  const int total = b * n;
  assemble_kernel<<<ceil_div(total, kAssembleThreads), kAssembleThreads, 0, st>>>(
      cloud, rgb, rgb_u8, label_image, hw, n, total, choose, ok, cld_rgb_nrm, row_stride, pcld, labels_out);
  return check_launch("assemble_kernel");
}

extern "C" size_t pvn3d_knn_normals_workspace_bytes(int b, int n_ref, int n_query) {
  if (b < 1 || n_ref < 1 || n_query < 1 || !fits_int32(static_cast<long long>(b) * (2ll * n_ref + 65)) ||
      !fits_int32(static_cast<long long>(b) * n_query * 32))
    return 0;
  return knn_ws_layout(b, n_ref).total;
}

extern "C" int pvn3d_knn_normals(const float *ref, const uint8_t *ref_valid, int n_ref, const float *query,
                                 int n_query, int b, const uint8_t *frame_ok, float *normals_out,
                                 long long row_stride, float *curv_out, double *normals64_out, int *nn_idx_out,
                                 void *workspace, size_t workspace_bytes, pvn3d_stream_t stream) {
  if (!ref || !query || !normals_out || !workspace || b < 1 || n_ref < 1 || n_query < 1 || row_stride < 3)
    return PVN3D_ERR_INVALID_ARG;
  // the search indexes warps as b * n_query * 32 threads, the grid as b * (2 * n_ref + 65) cells
  if (!fits_int32(static_cast<long long>(b) * (2ll * n_ref + 65)) ||
      !fits_int32(static_cast<long long>(b) * n_query * 32) || b > 65535)
    return PVN3D_ERR_UNSUPPORTED;
  const KnnWs L = knn_ws_layout(b, n_ref);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  auto *hdr = reinterpret_cast<GridHdr *>(ws + L.hdr);
  auto *box = reinterpret_cast<GridBox *>(ws + L.box);
  int *cell_start = reinterpret_cast<int *>(ws + L.cell_start), *cursor = reinterpret_cast<int *>(ws + L.cursor);
  auto *pts = reinterpret_cast<float4 *>(ws + L.pts);
  const int cap = grid_cap(n_ref);
  cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(cursor, 0, static_cast<size_t>(b) * cap * 4, st), "knn grid counts reset");
  grid_init_kernel<<<ceil_div(b, 128), 128, 0, st>>>(b, box);
  int rc = check_launch("grid_init_kernel");
  if (rc != PVN3D_OK) return rc;
  const dim3 pts_grid(static_cast<unsigned>(min(ceil_div(n_ref, kGridThreads), 1024)), static_cast<unsigned>(b));
  grid_bbox_kernel<<<pts_grid, kGridThreads, 0, st>>>(ref, ref_valid, n_ref, box);
  if ((rc = check_launch("grid_bbox_kernel")) != PVN3D_OK) return rc;
  grid_setup_kernel<<<ceil_div(b, 128), 128, 0, st>>>(b, cap, box, hdr);
  if ((rc = check_launch("grid_setup_kernel")) != PVN3D_OK) return rc;
  grid_count_kernel<<<pts_grid, kGridThreads, 0, st>>>(ref, ref_valid, n_ref, cap, hdr, cursor);
  if ((rc = check_launch("grid_count_kernel")) != PVN3D_OK) return rc;
  grid_scan_kernel<<<b, kScanThreads, 0, st>>>(cap, hdr, cell_start, cursor);
  if ((rc = check_launch("grid_scan_kernel")) != PVN3D_OK) return rc;
  grid_scatter_kernel<<<pts_grid, kGridThreads, 0, st>>>(ref, ref_valid, n_ref, cap, hdr, cursor, pts);
  if ((rc = check_launch("grid_scatter_kernel")) != PVN3D_OK) return rc;
  KnnParams p{};
  p.ref = ref;
  p.ref_valid = ref_valid;
  p.query = query;
  p.frame_ok = frame_ok;
  p.hdr = hdr;
  p.cell_start = cell_start;
  p.pts = pts;
  p.n_ref = n_ref;
  p.nq = n_query;
  p.b = b;
  p.cap = cap;
  p.normals = normals_out;
  p.stride = row_stride;
  p.curv = curv_out;
  p.normals64 = normals64_out;
  p.nn = nn_idx_out;
  const int warps = b * n_query;
  knn_normals_kernel<<<ceil_div(warps, kSearchThreads / 32), kSearchThreads, 0, st>>>(p);
  return check_launch("knn_normals_kernel");
}
