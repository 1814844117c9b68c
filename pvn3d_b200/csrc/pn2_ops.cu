// pn2_ops.cu -- the element-wise / search ops of lib.pointnet2_utils._ext for sm_90a:
// gather_points(+grad), ball_query, group_points(+grad), three_nn, three_interpolate(+grad),
// and the [B,C,N] <-> [B,N,C] staging transposes.
//
// The reference launches every one of these with grid = B (one CTA per cloud, e.g.
// ball_query_gpu.cu:50, group_points_gpu.cu:35, interpolate_gpu.cu:64,107): at B = 16..32 that
// leaves most of the 132 SMs of an H100 idle.  Here each op is tiled so that the grid covers the chip, the
// searched point set is staged through shared memory (bulk-copied by the TMA engine when
// alignment allows) and read back as broadcasts, and global accesses are coalesced.
#include "common.cuh"
#include "half_io.cuh"

namespace pvn3d {
namespace {

// ------------------------------------------------------------------------------------------------
// gather_points: out[b,c,j] = points[b,c,idx[b,j]]                (sampling_gpu.cu:8-20)
// ------------------------------------------------------------------------------------------------
__global__ void gather_points_kernel(const float *__restrict__ points, const int *__restrict__ idx,
                                     int c, int n, int m, float *__restrict__ out) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int a = idx[static_cast<size_t>(b) * m + j];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const size_t row = static_cast<size_t>(b) * c + l;
    out[row * m + j] = __ldg(points + row * n + a);
  }
}

__global__ void gather_points_grad_kernel(const float *__restrict__ grad_out,
                                          const int *__restrict__ idx, int c, int n, int m,
                                          float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int a = idx[static_cast<size_t>(b) * m + j];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const size_t row = static_cast<size_t>(b) * c + l;
    atomicAdd(grad_points + row * n + a, grad_out[row * m + j]);  // sampling_gpu.cu:42
  }
}

// ------------------------------------------------------------------------------------------------
// ball_query                                                    (ball_query_gpu.cu:9-44)
// One warp per query centre (CW centres per warp pass over the cloud): 32 lanes test 32
// consecutive points, a ballot + prefix-popcount appends the hits in index order, so the
// "first nsample in ascending k" rule holds by construction.  The cloud streams through shared
// memory in tiles; a CTA stops staging as soon as all of its balls are full.
// ------------------------------------------------------------------------------------------------
constexpr int kBqThreads = 256;
constexpr int kBqWarps = kBqThreads / 32;
constexpr int kBqCW = 4;                          // centres per warp
constexpr int kBqCentresPerCta = kBqWarps * kBqCW;  // 32
constexpr int kBqTile = 2048;                     // points per shared-memory tile (24 KB)

__global__ void __launch_bounds__(kBqThreads)
ball_query_kernel(const float *__restrict__ new_xyz, const float *__restrict__ xyz, int n, int m,
                  float radius, int nsample, int *__restrict__ idx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float *s_tile = reinterpret_cast<float *>(smem_raw);                       // kBqTile*3 floats
  int *s_rows = reinterpret_cast<int *>(smem_raw + kBqTile * 3 * sizeof(float));  // 32*nsample
  __shared__ uint64_t s_bar;

  const int b = blockIdx.y;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const float *cloud = xyz + static_cast<size_t>(b) * n * 3;
  const int j0 = blockIdx.x * kBqCentresPerCta + warp * kBqCW;
  const float r2 = __fmul_rn(radius, radius);  // ball_query_gpu.cu:22

  if (threadIdx.x == 0) {
    mbar_init(&s_bar, 1);
    mbar_fence_init();
  }
  float cx[kBqCW], cy[kBqCW], cz[kBqCW];
  int cnt[kBqCW], first[kBqCW];
#pragma unroll
  for (int c = 0; c < kBqCW; ++c) {
    const int j = j0 + c;
    const bool live = j < m;
    const float *p = new_xyz + (static_cast<size_t>(b) * m + (live ? j : 0)) * 3;
    cx[c] = p[0];
    cy[c] = p[1];
    cz[c] = p[2];
    cnt[c] = live ? 0 : nsample;  // dead centres count as full
    first[c] = 0;
  }
  __syncthreads();

  unsigned phase = 0;
  bool warp_open = true;
  for (int base = 0; base < n; base += kBqTile) {
    const int count = min(kBqTile, n - base);
    stage_xyz_tile(s_tile, cloud, base, count, &s_bar, phase, true);
    if (warp_open) {
      for (int off = 0; off < count; off += 32) {
        const int kk = off + static_cast<int>(lane);
        const bool in = kk < count;
        const float x = in ? s_tile[kk * 3 + 0] : 0.f;
        const float y = in ? s_tile[kk * 3 + 1] : 0.f;
        const float z = in ? s_tile[kk * 3 + 2] : 0.f;
        bool any_open = false;
#pragma unroll
        for (int c = 0; c < kBqCW; ++c) {
          if (cnt[c] < nsample) {  // warp-uniform
            const float d2 = ref_sqdist(cx[c] - x, cy[c] - y, cz[c] - z);
            const unsigned hits = __ballot_sync(0xffffffffu, in && d2 < r2);
            if (hits) {
              if (cnt[c] == 0) first[c] = base + off + __ffs(hits) - 1;
              const int slot = cnt[c] + __popc(hits & lanemask_lt());
              if (((hits >> lane) & 1u) && slot < nsample)
                s_rows[(warp * kBqCW + c) * nsample + slot] = base + kk;
              cnt[c] += __popc(hits);
            }
            any_open |= cnt[c] < nsample;
          }
        }
        if (!any_open) {
          warp_open = false;
          break;
        }
      }
    }
    // barrier: tile consumed by every warp before it is overwritten; the OR tells all threads the
    // same thing -- whether any ball of this CTA is still unfilled
    if (!__syncthreads_or(warp_open ? 1 : 0)) break;
  }

  // pad: slots >= cnt hold the first hit; empty ball -> zeros (torch::zeros, ball_query.cpp:19-21)
  __syncwarp();
#pragma unroll
  for (int c = 0; c < kBqCW; ++c) {
    const int j = j0 + c;
    if (j >= m) continue;
    int *dst = idx + (static_cast<size_t>(b) * m + j) * nsample;
    const int *row = s_rows + (warp * kBqCW + c) * nsample;
    const int filled = min(cnt[c], nsample);
    for (int s = lane; s < nsample; s += 32) dst[s] = s < filled ? row[s] : first[c];
  }
}

// ------------------------------------------------------------------------------------------------
// group_points: out[b,c,j,k] = points[b,c,idx[b,j,k]]            (group_points_gpu.cu:8-28)
// One thread per (j,k) slot (kVec = 1), or per two adjacent slots stored as one 4-byte pair (kVec = 2, 16-bit T, an
// even slot count), looping over a slice of channels: idx is read once per slice, the output is written coalesced
// along the slot axis.  T = float, __half or __nv_bfloat16: a copy, so every form is bit-exact.
// ------------------------------------------------------------------------------------------------
template <typename T, int kVec>
__global__ void group_points_kernel(const T *__restrict__ points, const int *__restrict__ idx,
                                    int c, int n, int slots, T *__restrict__ out) {
  const int b = blockIdx.z;
  if constexpr (kVec == 1) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots) return;
    const int ii = idx[static_cast<size_t>(b) * slots + s];
    for (int l = blockIdx.y; l < c; l += gridDim.y) {
      const size_t row = static_cast<size_t>(b) * c + l;
      stg_stream(out + row * slots + s, __ldg(points + row * n + ii));
    }
  } else {
    const int s = 2 * (blockIdx.x * blockDim.x + threadIdx.x);
    if (s >= slots) return;
    const int2 ii = *reinterpret_cast<const int2 *>(idx + static_cast<size_t>(b) * slots + s);
    for (int l = blockIdx.y; l < c; l += gridDim.y) {
      const size_t row = static_cast<size_t>(b) * c + l;
      stg_stream2(out + row * slots + s, __ldg(points + row * n + ii.x), __ldg(points + row * n + ii.y));
    }
  }
}

// grad_points[b,c,idx[b,s]] += grad_out[b,c,s] with float32 atomics; a 16-bit grad_out is widened on load and the
// float32 grad_points is the scratch that round_to16_kernel rounds once
template <typename T>
__global__ void group_points_grad_kernel(const T *__restrict__ grad_out,
                                         const int *__restrict__ idx, int c, int n, int slots,
                                         float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  const int ii = idx[static_cast<size_t>(b) * slots + s];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const size_t row = static_cast<size_t>(b) * c + l;
    atomicAdd(grad_points + row * n + ii, to_f32(grad_out[row * slots + s]));  // group_points_gpu.cu:60
  }
}

// ------------------------------------------------------------------------------------------------
// three_nn                                                      (interpolate_gpu.cu:9-59)
// One thread per unknown point; the known set streams through shared memory as float4 and is read
// as a broadcast.  The reference compares in double against bests seeded with 1e40; floats
// compared in double order exactly like floats, and 1e40 acts as +inf (it prints as +inf once
// narrowed to float, interpolate_gpu.cu:52-54), so a float cascade seeded with +inf is identical.
// ------------------------------------------------------------------------------------------------
constexpr int kNnThreads = 128;
constexpr int kNnTile = 1024;  // known points per tile (16 KB as float4)

struct Best3 {
  float d1, d2, d3;
  int i1, i2, i3;
};
__device__ __forceinline__ void best3_init(Best3 &b) {
  b.d1 = b.d2 = b.d3 = __int_as_float(0x7f800000);
  b.i1 = b.i2 = b.i3 = 0;
}
__device__ __forceinline__ void best3_push(Best3 &b, float d, int k) {
  if (d < b.d3) {  // d >= d3 fails all three strict tests of the reference cascade
    if (d < b.d1) {
      b.d3 = b.d2; b.i3 = b.i2;
      b.d2 = b.d1; b.i2 = b.i1;
      b.d1 = d;    b.i1 = k;
    } else if (d < b.d2) {
      b.d3 = b.d2; b.i3 = b.i2;
      b.d2 = d;    b.i2 = k;
    } else {
      b.d3 = d;    b.i3 = k;
    }
  }
}

// scans known[0..m) of cloud b for the calling thread's query point (ux,uy,uz); all threads of the
// CTA must call it (barriers inside).
// The tile holds NEGATED known points as pairs, s_known[2p] = (-x0,-x1,-y0,-y1), s_known[2p+1] = (-z0,-z1,.,.):
// u - q = u + (-q) exactly, so the distance of the query to two known points is, per component, the same
// IEEE operations in the same order as ref_sqdist
// (fma(dz,dz, fma(dx,dx, dy*dy))), pushed in index order: results stay bit-exact.  An odd tail is a point
// at infinity (d2 = inf never beats a finite or an initial inf candidate).
__device__ __forceinline__ void three_nn_scan(const float *__restrict__ known_cloud, int m,
                                              float4 *s_known, float ux, float uy, float uz,
                                              Best3 &best) {
  best3_init(best);
  const float2 ux2 = make_float2(ux, ux), uy2 = make_float2(uy, uy), uz2 = make_float2(uz, uz);
  const float ninf = -__int_as_float(0x7f800000);
  for (int base = 0; base < m; base += kNnTile) {
    const int count = min(kNnTile, m - base);
    const int npairs = (count + 1) >> 1;
    __syncthreads();
    for (int i = threadIdx.x; i < npairs; i += blockDim.x) {
      const float *p = known_cloud + static_cast<size_t>(base + 2 * i) * 3;
      const bool two = 2 * i + 1 < count;
      const float x0 = __ldg(p), y0 = __ldg(p + 1), z0 = __ldg(p + 2);
      const float x1 = two ? __ldg(p + 3) : -ninf, y1 = two ? __ldg(p + 4) : -ninf, z1 = two ? __ldg(p + 5) : -ninf;
      s_known[2 * i] = make_float4(-x0, -x1, -y0, -y1);
      s_known[2 * i + 1] = make_float4(-z0, -z1, 0.f, 0.f);
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < npairs; ++k) {
      const float4 a = s_known[2 * k], c = s_known[2 * k + 1];
      const float2 dx = f2_add(make_float2(a.x, a.y), ux2);
      const float2 dy = f2_add(make_float2(a.z, a.w), uy2);
      const float2 dz = f2_add(make_float2(c.x, c.y), uz2);
      const float2 d = f2_fma(dz, dz, f2_fma(dx, dx, f2_mul(dy, dy)));
      best3_push(best, d.x, base + 2 * k);
      best3_push(best, d.y, base + 2 * k + 1);
    }
  }
}

__global__ void __launch_bounds__(kNnThreads)
three_nn_kernel(const float *__restrict__ unknown, const float *__restrict__ known, int n, int m,
                float *__restrict__ dist2, int *__restrict__ idx) {
  __shared__ float4 s_known[kNnTile];
  const int b = blockIdx.y;
  const int j = blockIdx.x * kNnThreads + threadIdx.x;
  const bool live = j < n;
  const float *u = unknown + (static_cast<size_t>(b) * n + (live ? j : 0)) * 3;
  Best3 best;
  three_nn_scan(known + static_cast<size_t>(b) * m * 3, m, s_known, u[0], u[1], u[2], best);
  if (!live) return;
  float *d = dist2 + (static_cast<size_t>(b) * n + j) * 3;
  int *o = idx + (static_cast<size_t>(b) * n + j) * 3;
  d[0] = best.d1; d[1] = best.d2; d[2] = best.d3;
  o[0] = best.i1; o[1] = best.i2; o[2] = best.i3;
}

// ------------------------------------------------------------------------------------------------
// three_nn through an x-sorted copy of the known set.  The reference cascade (ascending k, strict '<') ends with
// the three smallest (d2, k) pairs in lexicographic order, so the scan order is free as long as ties are broken by
// the index.  With the known points of a frame sorted by x, a query walks outward from its own x in both
// directions and stops when the squared x-gap alone exceeds its third-best distance: d2 = fma(dz,dz, fma(dx,dx,
// dy*dy)) >= fl(dx*dx) by monotonicity of rounding, so nothing beyond can enter (gaps EQUAL to d3 are still
// examined: they could tie).  At the FP1 level (12288 queries x 2048 known) a query tests ~130 candidates instead
// of 2048.  d2 is evaluated by the same expression as the scan, indices / distances stay bit-exact.
constexpr int kNnSlabMaxM = 4096;

__global__ void __launch_bounds__(512) nn_sort_known_kernel(const float *__restrict__ known, int m, int m_pad,
                                                            float4 *__restrict__ sorted) {
  extern __shared__ float4 s_k[];
  known += static_cast<size_t>(blockIdx.x) * m * 3;
  sorted += static_cast<size_t>(blockIdx.x) * m_pad;
  const float inf = __int_as_float(0x7f800000);
  // a NaN x orders against nothing and would leave the copy unsorted for every other point: it is keyed (and stored)
  // as +inf.  Its distance is then inf or NaN instead of NaN -- never selected either way, as in the reference cascade
  for (int i = threadIdx.x; i < m_pad; i += blockDim.x) {
    float4 v = make_float4(inf, inf, inf, __int_as_float(0x7fffffff));
    if (i < m) {
      const float x = __ldg(known + i * 3);
      v = make_float4(x == x ? x : inf, __ldg(known + i * 3 + 1), __ldg(known + i * 3 + 2), __int_as_float(i));
    }
    s_k[i] = v;
  }
  __syncthreads();
  for (int k = 2; k <= m_pad; k <<= 1) {          // bitonic sort by (x, index)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < m_pad; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const float4 a = s_k[i], b = s_k[l];
          const bool a_gt_b = a.x > b.x || (a.x == b.x && __float_as_int(a.w) > __float_as_int(b.w));
          if (a_gt_b == ((i & k) == 0)) { s_k[i] = b; s_k[l] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < m_pad; i += blockDim.x) sorted[i] = s_k[i];
}

__device__ __forceinline__ void best3_push_lex(Best3 &b, float d, int k) {
  // insert (d, k) if it precedes the current third pair in (distance, index) order
  if (d < b.d3 || (d == b.d3 && k < b.i3)) {
    if (d < b.d1 || (d == b.d1 && k < b.i1)) {
      b.d3 = b.d2; b.i3 = b.i2;
      b.d2 = b.d1; b.i2 = b.i1;
      b.d1 = d;    b.i1 = k;
    } else if (d < b.d2 || (d == b.d2 && k < b.i2)) {
      b.d3 = b.d2; b.i3 = b.i2;
      b.d2 = d;    b.i2 = k;
    } else {
      b.d3 = d;    b.i3 = k;
    }
  }
}

__global__ void __launch_bounds__(kNnThreads)
three_nn_slab_kernel(const float *__restrict__ unknown, const float4 *__restrict__ sorted, int n, int m, int m_pad,
                     float *__restrict__ dist2, int *__restrict__ idx) {
  // the walk reads the frame's sorted copy (<= 64 KB) through the read-only cache: staged in shared memory, the same
  // walk lost the lower index of coincident known points on sm_90a (tests/test_pn2_gpu.py tie cases)
  const int b = blockIdx.y;
  const float4 *__restrict__ s_k = sorted + static_cast<size_t>(b) * m_pad;
  const int j = blockIdx.x * kNnThreads + threadIdx.x;
  if (j >= n) return;
  const float *u = unknown + (static_cast<size_t>(b) * n + j) * 3;
  const float ux = u[0], uy = u[1], uz = u[2];
  Best3 best;
  best3_init(best);
  best.i1 = best.i2 = best.i3 = 0x7fffffff;   // so that any real pair precedes an empty slot; restored to 0 at the end
  int lo = 0, hi = m;                          // first position with x >= ux
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s_k[mid].x < ux) lo = mid + 1; else hi = mid;
  }
  int l = lo - 1, r = lo;
  const float inf = __int_as_float(0x7f800000);
  float gl = inf, gr = inf;                    // squared x-gap of the next candidate on either side
  if (l >= 0) { const float dx = ux - s_k[l].x; gl = dx * dx; }
  if (r < m) { const float dx = ux - s_k[r].x; gr = dx * dx; }
  while (l >= 0 || r < m) {
    const bool left = gl <= gr;
    const float g = left ? gl : gr;
    if (g > best.d3) break;                    // both sides are farther in x alone than the third best
    const float4 q = s_k[left ? l : r];
    best3_push_lex(best, ref_sqdist(ux - q.x, uy - q.y, uz - q.z), __float_as_int(q.w));
    if (left) {
      --l;
      gl = inf;
      if (l >= 0) { const float dx = ux - s_k[l].x; gl = dx * dx; }
    } else {
      ++r;
      gr = inf;
      if (r < m) { const float dx = ux - s_k[r].x; gr = dx * dx; }
    }
  }
  float *d = dist2 + (static_cast<size_t>(b) * n + j) * 3;
  int *o = idx + (static_cast<size_t>(b) * n + j) * 3;
  d[0] = best.d1; d[1] = best.d2; d[2] = best.d3;
  o[0] = best.d1 < inf ? best.i1 : 0; o[1] = best.d2 < inf ? best.i2 : 0; o[2] = best.d3 < inf ? best.i3 : 0;
}

// dist = sqrt(dist2) (pointnet2_utils.py:126); 1/(dist+1e-8); normalise (modules.py:184-186) -- the IEEE operations of
// nn_weights_kernel (mlp_tc.cu), so both give the same bits
__device__ __forceinline__ void nn_inverse_distance_weights(float d1, float d2, float d3, float &w1, float &w2,
                                                            float &w3) {
  const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(d1), 1e-8f));
  const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(d2), 1e-8f));
  const float r3 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(d3), 1e-8f));
  const float norm = __fadd_rn(__fadd_rn(r1, r2), r3);
  w1 = __fdiv_rn(r1, norm);
  w2 = __fdiv_rn(r2, norm);
  w3 = __fdiv_rn(r3, norm);
}

// ------------------------------------------------------------------------------------------------
// three_nn + weights on per-frame cell grids (pvn3d_three_nn_weights_levels).
// The known set of every (level, frame) is counting-sorted into a uniform grid over its finite bounding box; a query
// visits the cells in rings of growing Chebyshev distance around its own cell and stops once every unvisited cell lies
// farther than its third-best distance.  The result is the reference cascade's by the same argument as the x-sorted
// walk: the three smallest (d2, k) pairs in lexicographic order, d2 by ref_sqdist, in any visiting order.
//   * Non-finite known points are left out of the grid: their d2 is NaN or inf, which never passes the cascade's
//     strict '<' against the 1e40 seed.
//   * The stop test is conservative.  A point binned into cell c lies within [lo + c h, lo + (c+1) h] up to the
//     rounding of (x - lo) * inv (below 1e-5 h at 64 cells per axis); `tol` covers that and the rounding of the face
//     coordinate lo + k h, and the factor (1 - 1e-5) the rounding of d2 itself.  Equality with d3 keeps searching.
//   * Cells are sized for ~kNnGridPts points per cell on a surface (depth clouds are surfaces; a volume cloud gets
//     smaller cells, which costs rings, not results), at most kNnGridAxis per axis and kNnGridCells in all: a far
//     outlier makes the cells coarse, never wrong.
// ------------------------------------------------------------------------------------------------
constexpr int kNnGridMaxLevels = 4;
constexpr int kNnGridMaxM = 8192;     // known points per frame the grid path takes
constexpr int kNnGridCells = 8192;    // cells per grid at most (the counting sort's table: 32 KB of shared memory)
constexpr int kNnGridAxis = 64;       // cells per axis at most
constexpr float kNnGridPts = 2.f;     // points per cell aimed at
constexpr int kNnGridBuildThreads = 512;

struct NnGridHdr {
  float lo[3];
  float h, inv, tol;
  int g[3];
  int pad;
};
struct NnGridLevel {
  const float *unknown, *known;
  float *dist2, *weight;
  int *idx;
  int n, m;
  int blk0;            // first blockIdx.x of this level in the search launch
  float hmin;          // smallest cell side (a ball query's larger radius; 0 for 3-NN)
  float4 *sorted;      // [B][m]: (x, y, z, index bits), grouped by cell
  int *cell_start;     // [B][kNnGridCells + 1]
  NnGridHdr *hdr;      // [B]
};
struct NnGridArgs {
  NnGridLevel lv[kNnGridMaxLevels];
  int nlev;
};

__device__ __forceinline__ bool finite3(float x, float y, float z) {
  return fabsf(x) <= 3.402823466e38f && fabsf(y) <= 3.402823466e38f && fabsf(z) <= 3.402823466e38f;
}
__device__ __forceinline__ int nn_cell_axis(const NnGridHdr &g, int d, float v) {
  const float c = floorf(__fmul_rn(__fsub_rn(v, g.lo[d]), g.inv));
  return static_cast<int>(fminf(fmaxf(c, 0.f), static_cast<float>(g.g[d] - 1)));   // NaN -> 0 (never queried so)
}
__device__ __forceinline__ int nn_cell_of(const NnGridHdr &g, float x, float y, float z) {
  return (nn_cell_axis(g, 2, z) * g.g[1] + nn_cell_axis(g, 1, y)) * g.g[0] + nn_cell_axis(g, 0, x);
}

// grid (B, levels): one CTA builds the grid of one frame of one level
__global__ void __launch_bounds__(kNnGridBuildThreads) nn_grid_build_kernel(NnGridArgs a) {
  __shared__ int s_cnt[kNnGridCells + 1];
  __shared__ float s_red[6][kNnGridBuildThreads / 32];
  __shared__ int s_wsum[kNnGridBuildThreads / 32];
  __shared__ NnGridHdr s_g;
  const NnGridLevel &L = a.lv[blockIdx.y];
  const int b = blockIdx.x, t = threadIdx.x, m = L.m;
  const unsigned lane = lane_id(), warp = t >> 5;
  const float *known = L.known + static_cast<size_t>(b) * m * 3;
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (int i = t; i < m; i += kNnGridBuildThreads) {
    const float x = __ldg(known + i * 3), y = __ldg(known + i * 3 + 1), z = __ldg(known + i * 3 + 2);
    if (finite3(x, y, z)) {
      lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
      hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if (lane == 0)
    for (int d = 0; d < 3; ++d) { s_red[d][warp] = lo[d]; s_red[3 + d][warp] = hi[d]; }
  for (int c = t; c <= kNnGridCells; c += kNnGridBuildThreads) s_cnt[c] = 0;
  __syncthreads();
  if (t == 0) {
    NnGridHdr g;
    float e[3];
    bool any = true;
    for (int d = 0; d < 3; ++d) {
      float l = s_red[d][0], h = s_red[3 + d][0];
      for (int w = 1; w < kNnGridBuildThreads / 32; ++w) { l = fminf(l, s_red[d][w]); h = fmaxf(h, s_red[3 + d][w]); }
      any = any && l <= h;
      g.lo[d] = l;
      e[d] = h - l;   // may round up; the binning clamps
    }
    if (!any) {       // no finite point: one empty cell
      for (int d = 0; d < 3; ++d) { g.lo[d] = 0.f; e[d] = 0.f; }
    }
    // the two largest extents span the surface
    const float e1 = fmaxf(e[0], fmaxf(e[1], e[2]));
    const float e3 = fminf(e[0], fminf(e[1], e[2]));
    const float e2 = e[0] + e[1] + e[2] - e1 - e3;
    const float per = kNnGridPts / static_cast<float>(m);
    float h = sqrtf(e1 * e2 * per);
    if (!(h > 0.f)) h = e1 * per;
    h = fmaxf(h, L.hmin);
    h = fmaxf(h, e1 / static_cast<float>(kNnGridAxis - 1));   // no axis needs more than kNnGridAxis cells
    if (!(h > 0.f)) h = 1.f;   // all finite points coincide
    if (!(e1 < 3.0e38f) || !(h < 3.0e38f)) {   // the extent itself overflows: one cell, every point binned into it
      g.g[0] = g.g[1] = g.g[2] = 1;
      h = 1.f;
      g.inv = 0.f;
    } else {
      for (;;) {
        int cells = 1;
        for (int d = 0; d < 3; ++d) {
          g.g[d] = static_cast<int>(fminf(floorf(e[d] / h), static_cast<float>(kNnGridAxis - 1))) + 1;
          cells *= g.g[d];
        }
        if (cells <= kNnGridCells) break;
        h *= 1.25f;
      }
      g.inv = 1.f / h;
    }
    g.h = h;
    float mag = 0.f;
    for (int d = 0; d < 3; ++d) mag = fmaxf(mag, fmaxf(fabsf(g.lo[d]), fabsf(g.lo[d] + g.g[d] * h)));
    g.tol = 1e-4f * h + 4e-6f * mag;
    g.pad = 0;
    s_g = g;
    L.hdr[b] = g;
  }
  __syncthreads();
  const NnGridHdr g = s_g;
  const int ncell = g.g[0] * g.g[1] * g.g[2];
  for (int i = t; i < m; i += kNnGridBuildThreads) {
    const float x = __ldg(known + i * 3), y = __ldg(known + i * 3 + 1), z = __ldg(known + i * 3 + 2);
    if (finite3(x, y, z)) atomicAdd(&s_cnt[nn_cell_of(g, x, y, z)], 1);
  }
  __syncthreads();
  // exclusive scan of the ncell + 1 counts: thread t owns the run [t*per_t, (t+1)*per_t)
  constexpr int per_t = (kNnGridCells + kNnGridBuildThreads) / kNnGridBuildThreads;   // 17: covers kNnGridCells + 1
  int run = 0;
  const int c0 = t * per_t;
  for (int c = c0; c < c0 + per_t && c <= ncell; ++c) run += s_cnt[c];
  int incl = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (static_cast<int>(lane) >= o) incl += v;
  }
  if (lane == 31) s_wsum[warp] = incl;
  __syncthreads();
  int acc = incl - run;
  for (int w = 0; w < static_cast<int>(warp); ++w) acc += s_wsum[w];
  int *starts = L.cell_start + static_cast<size_t>(b) * (kNnGridCells + 1);
  for (int c = c0; c < c0 + per_t && c <= ncell; ++c) {
    const int v = s_cnt[c];
    s_cnt[c] = acc;
    starts[c] = acc;
    acc += v;
  }
  __syncthreads();
  float4 *sorted = L.sorted + static_cast<size_t>(b) * m;
  for (int i = t; i < m; i += kNnGridBuildThreads) {
    const float x = __ldg(known + i * 3), y = __ldg(known + i * 3 + 1), z = __ldg(known + i * 3 + 2);
    if (finite3(x, y, z)) sorted[atomicAdd(&s_cnt[nn_cell_of(g, x, y, z)], 1)] = make_float4(x, y, z, __int_as_float(i));
  }
}

// grid (sum over levels of ceil(n / kNnThreads), B): one thread per query point
__global__ void __launch_bounds__(kNnThreads) three_nn_grid_kernel(NnGridArgs a) {
  int l = 0;
  while (l + 1 < a.nlev && static_cast<int>(blockIdx.x) >= a.lv[l + 1].blk0) ++l;
  const NnGridLevel &L = a.lv[l];
  const int b = blockIdx.y;
  const int j = (blockIdx.x - L.blk0) * kNnThreads + threadIdx.x;
  if (j >= L.n) return;
  const float *u = L.unknown + (static_cast<size_t>(b) * L.n + j) * 3;
  const float ux = u[0], uy = u[1], uz = u[2];
  const NnGridHdr g = L.hdr[b];
  const float4 *__restrict__ pts = L.sorted + static_cast<size_t>(b) * L.m;
  const int *__restrict__ start = L.cell_start + static_cast<size_t>(b) * (kNnGridCells + 1);
  const float inf = __int_as_float(0x7f800000);
  Best3 best;
  best3_init(best);
  best.i1 = best.i2 = best.i3 = 0x7fffffff;   // so that any real pair precedes an empty slot; restored to 0 at the end
  if (finite3(ux, uy, uz)) {   // a non-finite query has d2 NaN or inf to every point: nothing passes
    const int cx = nn_cell_axis(g, 0, ux), cy = nn_cell_axis(g, 1, uy), cz = nn_cell_axis(g, 2, uz);
    const float q[3] = {ux, uy, uz};
    const int cq[3] = {cx, cy, cz};
    for (int r = 0;; ++r) {
      const int y0 = max(cy - r, 0), y1 = min(cy + r, g.g[1] - 1);
      const int z0 = max(cz - r, 0), z1 = min(cz + r, g.g[2] - 1);
      const int x0 = max(cx - r, 0), x1 = min(cx + r, g.g[0] - 1);
      for (int z = z0; z <= z1; ++z) {
        for (int y = y0; y <= y1; ++y) {
          const int row = (z * g.g[1] + y) * g.g[0];
          auto visit = [&](int c_first, int c_last) {   // the points of cells c_first..c_last of this row: one run
            const int p1 = start[row + c_last + 1];
            for (int p = start[row + c_first]; p < p1; ++p) {
              const float4 k = pts[p];
              best3_push_lex(best, ref_sqdist(ux - k.x, uy - k.y, uz - k.z), __float_as_int(k.w));
            }
          };
          if (abs(z - cz) == r || abs(y - cy) == r) {   // the whole x-run of the row is on ring r
            visit(x0, x1);
          } else {                                       // an inner row: its two end cells
            if (cx - r >= 0) visit(cx - r, cx - r);
            if (cx + r < g.g[0]) visit(cx + r, cx + r);
          }
        }
      }
      // every cell within Chebyshev distance r is done; the rest lies beyond the nearest face of that box that has
      // cells behind it
      float gap = inf;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        if (cq[d] - r > 0) gap = fminf(gap, q[d] - (g.lo[d] + static_cast<float>(cq[d] - r) * g.h));
        if (cq[d] + r < g.g[d] - 1) gap = fminf(gap, (g.lo[d] + static_cast<float>(cq[d] + r + 1) * g.h) - q[d]);
      }
      if (gap == inf) break;   // the box covers the grid
      gap -= g.tol;
      if (gap > 0.f && gap * gap * (1.f - 1e-5f) > best.d3) break;
    }
  }
  const size_t o = (static_cast<size_t>(b) * L.n + j) * 3;
  L.dist2[o] = best.d1; L.dist2[o + 1] = best.d2; L.dist2[o + 2] = best.d3;
  L.idx[o] = best.d1 < inf ? best.i1 : 0;
  L.idx[o + 1] = best.d2 < inf ? best.i2 : 0;
  L.idx[o + 2] = best.d3 < inf ? best.i3 : 0;
  float w1, w2, w3;
  nn_inverse_distance_weights(best.d1, best.d2, best.d3, w1, w2, w3);
  L.weight[o] = w1; L.weight[o + 1] = w2; L.weight[o + 2] = w3;
}

// ------------------------------------------------------------------------------------------------
// ball query of both radii of an MSG level on per-frame cell grids (pvn3d_ball_query2_levels).
// The searched cloud of every (level, frame) is binned by nn_grid_build_kernel with cells at least as wide as the larger
// radius.  A warp per centre visits the cells that can hold a hit, tests every point with ref_sqdist and the strict
// '<' of both radii, and collects all hits in a per-warp buffer.  Each point sits in exactly one cell, so ranking the
// buffered hits by index gives the reference's "first ns in index order" for any visiting order.
//   * Reach: a hit has fl(dx*dx) <= d2 < r2 (monotone rounding), so |c - p| < r (1 + 2^-22) on every axis; the range
//     c -/+ R with R = 1.001 r + 1e-6 |c| contains it after rounding, and the binning is monotone in the coordinate,
//     so every hit's cell lies in [cell(c - R), cell(c + R)] -- clamped and misrounded binning included.
//   * Non-finite points are not binned: their d2 is NaN or inf and never passes '<'.  A non-finite centre has no hit.
//   * A centre with more than kBgCap hits runs the index-order scan of the whole cloud instead (ball_scan_kernel
//     without its boxes), so the buffer never decides a result.
// ------------------------------------------------------------------------------------------------
constexpr int kBgWarps = 8;
constexpr int kBgCap = 512;          // buffered hits per centre
constexpr int kBgMaxNs = 256;        // nsample of either radius the grid path takes

struct BallGridLevel {
  const float *xyz, *centres;        // searched cloud [B][n][3], centres [B][m][3]
  int n, m;
  float r0, r1;
  int ns0, ns1;
  int *idx0, *idx1;                  // [B][m][ns0], [B][m][ns1]
  int blk0;                          // first blockIdx.x of this level
};
struct BallGridArgs {
  BallGridLevel lv[kNnGridMaxLevels];
  float4 *sorted[kNnGridMaxLevels];
  int *cell_start[kNnGridMaxLevels];
  NnGridHdr *hdr[kNnGridMaxLevels];
  int nlev;
};

__global__ void __launch_bounds__(kBgWarps * 32) ball_grid_kernel(BallGridArgs a) {
  __shared__ int s_hit[kBgWarps][kBgCap];
  int l = 0;
  while (l + 1 < a.nlev && static_cast<int>(blockIdx.x) >= a.lv[l + 1].blk0) ++l;
  const BallGridLevel &L = a.lv[l];
  const int b = blockIdx.y;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const int j = (blockIdx.x - L.blk0) * kBgWarps + static_cast<int>(warp);
  if (j >= L.m) return;   // warp-uniform; no CTA barrier below
  const float *cp = L.centres + (static_cast<size_t>(b) * L.m + j) * 3;
  const float cx = cp[0], cy = cp[1], cz = cp[2];
  const float r2a = __fmul_rn(L.r0, L.r0), r2b = __fmul_rn(L.r1, L.r1);   // ball_query_gpu.cu:22
  int *hits = s_hit[warp];
  int cnt = 0;
  if (finite3(cx, cy, cz)) {
    const NnGridHdr g = a.hdr[l][b];
    const float4 *__restrict__ pts = a.sorted[l] + static_cast<size_t>(b) * L.n;
    const int *__restrict__ start = a.cell_start[l] + static_cast<size_t>(b) * (kNnGridCells + 1);
    const float r = fmaxf(L.r0, L.r1);
    const float c[3] = {cx, cy, cz};
    int lo[3], hi[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float reach = r * 1.001f + 1e-6f * fabsf(c[d]) + 1e-30f;
      lo[d] = nn_cell_axis(g, d, c[d] - reach);
      hi[d] = nn_cell_axis(g, d, c[d] + reach);
    }
    for (int z = lo[2]; z <= hi[2]; ++z)
      for (int y = lo[1]; y <= hi[1]; ++y) {
        const int row = (z * g.g[1] + y) * g.g[0];
        const int p1 = start[row + hi[0] + 1];
        for (int p0 = start[row + lo[0]]; p0 < p1; p0 += 32) {
          const int p = p0 + static_cast<int>(lane);
          bool ha = false, hb = false;
          int k = 0;
          if (p < p1) {
            const float4 q = pts[p];
            const float d2 = ref_sqdist(cx - q.x, cy - q.y, cz - q.z);
            ha = d2 < r2a;
            hb = d2 < r2b;
            k = __float_as_int(q.w);
          }
          const unsigned any = __ballot_sync(0xffffffffu, ha || hb);
          if ((ha || hb)) {
            const int slot = cnt + __popc(any & lanemask_lt());
            if (slot < kBgCap) hits[slot] = k | (ha ? 0x40000000 : 0) | (hb ? static_cast<int>(0x80000000u) : 0);
          }
          cnt += __popc(any);
        }
      }
  }
  const size_t cent = static_cast<size_t>(b) * L.m + j;
  int *out_a = L.idx0 + cent * L.ns0, *out_b = L.idx1 + cent * L.ns1;
  if (cnt > kBgCap) {
    // the index-order scan: hits appended in ascending k, the first ns of each radius kept
    const float *cloud = L.xyz + static_cast<size_t>(b) * L.n * 3;
    int ca = 0, cb = 0, fa = 0, fb = 0;
    for (int off = 0; off < L.n && (ca < L.ns0 || cb < L.ns1); off += 32) {
      const int k = off + static_cast<int>(lane);
      bool ha = false, hb = false;
      if (k < L.n) {
        const float *q = cloud + static_cast<size_t>(k) * 3;
        const float d2 = ref_sqdist(cx - __ldg(q), cy - __ldg(q + 1), cz - __ldg(q + 2));
        ha = d2 < r2a;
        hb = d2 < r2b;
      }
      const unsigned ma = __ballot_sync(0xffffffffu, ha), mb = __ballot_sync(0xffffffffu, hb);
      if (ma) {
        if (ca == 0) fa = off + __ffs(ma) - 1;
        const int slot = ca + __popc(ma & lanemask_lt());
        if (ha && slot < L.ns0) out_a[slot] = k;
        ca += __popc(ma);
      }
      if (mb) {
        if (cb == 0) fb = off + __ffs(mb) - 1;
        const int slot = cb + __popc(mb & lanemask_lt());
        if (hb && slot < L.ns1) out_b[slot] = k;
        cb += __popc(mb);
      }
    }
    for (int s = static_cast<int>(lane) + min(ca, L.ns0); s < L.ns0; s += 32) out_a[s] = fa;
    for (int s = static_cast<int>(lane) + min(cb, L.ns1); s < L.ns1; s += 32) out_b[s] = fb;
    return;
  }
  __syncwarp();
  // rank every buffered hit among the hits of its radius: rank < ns -> slot rank; rank 0 is the first hit
  int ca = 0, cb = 0, fa = 0x7fffffff, fb = 0x7fffffff;
  for (int i = static_cast<int>(lane); i < cnt; i += 32) {
    const int h = hits[i], k = h & 0x3fffffff;
    const bool ia = (h & 0x40000000) != 0, ib = h < 0;
    int ra = 0, rb = 0;
    for (int e = 0; e < cnt; ++e) {
      const int o = hits[e], ko = o & 0x3fffffff;
      ra += (ko < k && (o & 0x40000000)) ? 1 : 0;
      rb += (ko < k && o < 0) ? 1 : 0;
    }
    if (ia) {
      ++ca;
      fa = min(fa, k);
      if (ra < L.ns0) out_a[ra] = k;
    }
    if (ib) {
      ++cb;
      fb = min(fb, k);
      if (rb < L.ns1) out_b[rb] = k;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ca += __shfl_xor_sync(0xffffffffu, ca, o);
    cb += __shfl_xor_sync(0xffffffffu, cb, o);
    fa = min(fa, __shfl_xor_sync(0xffffffffu, fa, o));
    fb = min(fb, __shfl_xor_sync(0xffffffffu, fb, o));
  }
  // pad: slots >= cnt hold the first hit; an empty ball is zeros (torch::zeros, ball_query.cpp:19-21)
  if (ca == 0) fa = 0;
  if (cb == 0) fb = 0;
  for (int s = static_cast<int>(lane) + min(ca, L.ns0); s < L.ns0; s += 32) out_a[s] = fa;
  for (int s = static_cast<int>(lane) + min(cb, L.ns1); s < L.ns1; s += 32) out_b[s] = fb;
}

// ------------------------------------------------------------------------------------------------
// three_interpolate: out[b,c,j] = sum_t points[b,c,idx[b,j,t]] * w[b,j,t]   (interpolate_gpu.cu:72-101)
// contraction as in the reference SASS (oracle/_ref build, interpolate_gpu.o):
//   t = p2*w2 (FMUL); t = fma(p1,w1,t); out = fma(p3,w3,t)  -- the MIDDLE product is the bare multiply
// T = __half / __nv_bfloat16: the same float32 sum of the widened features, rounded once; kVec = 2 gives a thread two
// adjacent points (an even n) and one 4-byte store per channel.
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float interp3(const T *row, int i1, int i2, int i3, float w1, float w2, float w3) {
  return __fmaf_rn(to_f32(__ldg(row + i3)), w3,
                   __fmaf_rn(to_f32(__ldg(row + i1)), w1, __fmul_rn(to_f32(__ldg(row + i2)), w2)));
}

template <typename T, int kVec>
__global__ void three_interpolate_kernel(const T *__restrict__ points,
                                         const int *__restrict__ idx,
                                         const float *__restrict__ weight, int c, int m, int n,
                                         T *__restrict__ out) {
  const int b = blockIdx.z;
  const int j = kVec * (blockIdx.x * blockDim.x + threadIdx.x);
  if (j >= n) return;
  const size_t q = (static_cast<size_t>(b) * n + j) * 3;
  const float w1 = weight[q], w2 = weight[q + 1], w3 = weight[q + 2];
  const int i1 = idx[q], i2 = idx[q + 1], i3 = idx[q + 2];
  if constexpr (kVec == 1) {
    for (int l = blockIdx.y; l < c; l += gridDim.y) {
      const T *row = points + (static_cast<size_t>(b) * c + l) * m;
      out[(static_cast<size_t>(b) * c + l) * n + j] = from_f32<T>(interp3(row, i1, i2, i3, w1, w2, w3));
    }
  } else {
    const float v1 = weight[q + 3], v2 = weight[q + 4], v3 = weight[q + 5];
    const int k1 = idx[q + 3], k2 = idx[q + 4], k3 = idx[q + 5];
    for (int l = blockIdx.y; l < c; l += gridDim.y) {
      const T *row = points + (static_cast<size_t>(b) * c + l) * m;
      st_pair(out + (static_cast<size_t>(b) * c + l) * n + j, from_f32<T>(interp3(row, i1, i2, i3, w1, w2, w3)),
              from_f32<T>(interp3(row, k1, k2, k3, v1, v2, v3)));
    }
  }
}

// float32 atomics of fl(g * w) into grad_points (a float32 scratch for a 16-bit grad_out, rounded afterwards)
template <typename T>
__global__ void three_interpolate_grad_kernel(const T *__restrict__ grad_out,
                                              const int *__restrict__ idx,
                                              const float *__restrict__ weight, int c, int n, int m,
                                              float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t q = (static_cast<size_t>(b) * n + j) * 3;
  const float w1 = weight[q], w2 = weight[q + 1], w3 = weight[q + 2];
  const int i1 = idx[q], i2 = idx[q + 1], i3 = idx[q + 2];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const float g = to_f32(grad_out[(static_cast<size_t>(b) * c + l) * n + j]);
    float *row = grad_points + (static_cast<size_t>(b) * c + l) * m;
    atomicAdd(row + i1, g * w1);  // interpolate_gpu.cu:139-141
    atomicAdd(row + i2, g * w2);
    atomicAdd(row + i3, g * w3);
  }
}

// ------------------------------------------------------------------------------------------------
// [B,R,Cc] -> [B,Cc,R] tiled transpose (both staging directions)
// ------------------------------------------------------------------------------------------------
__global__ void transpose_kernel(const float *__restrict__ src, int rows, int cols,
                                 float *__restrict__ dst) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  src += static_cast<size_t>(b) * rows * cols;
  dst += static_cast<size_t>(b) * rows * cols;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, cc = c0 + threadIdx.x;
    if (r < rows && cc < cols) tile[i][threadIdx.x] = src[static_cast<size_t>(r) * cols + cc];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int cc = c0 + i, r = r0 + threadIdx.x;
    if (r < rows && cc < cols) dst[static_cast<size_t>(cc) * rows + r] = tile[threadIdx.x][i];
  }
}

// ------------------------------------------------------------------------------------------------
// three_nn + inverse-distance weights + three_interpolate on point-major descriptors: the geometric
// half of PointnetFPModule.forward (pointnet2_modules.py:183-190) in one kernel.  Each unknown
// point reads three full descriptor rows (coalesced) instead of 3*C strided scalars.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kNnThreads)
three_nn_interp_kernel(const float *__restrict__ unknown, const float *__restrict__ known,
                       const float *__restrict__ known_feat_pm, int n, int m, int c,
                       float *__restrict__ out_pm, int ldo, int col0, float *__restrict__ dist2,
                       int *__restrict__ idx) {
  __shared__ float4 s_known[kNnTile];
  __shared__ int s_i[kNnThreads][3];
  __shared__ float s_w[kNnThreads][3];
  const int b = blockIdx.y;
  const int j0 = blockIdx.x * kNnThreads;
  const int j = j0 + threadIdx.x;
  const bool live = j < n;
  const float *u = unknown + (static_cast<size_t>(b) * n + (live ? j : 0)) * 3;
  Best3 best;
  three_nn_scan(known + static_cast<size_t>(b) * m * 3, m, s_known, u[0], u[1], u[2], best);
  {
    nn_inverse_distance_weights(best.d1, best.d2, best.d3, s_w[threadIdx.x][0], s_w[threadIdx.x][1],
                                s_w[threadIdx.x][2]);
    s_i[threadIdx.x][0] = best.i1;
    s_i[threadIdx.x][1] = best.i2;
    s_i[threadIdx.x][2] = best.i3;
    if (live) {
      const size_t q = (static_cast<size_t>(b) * n + j) * 3;
      if (dist2) { dist2[q] = best.d1; dist2[q + 1] = best.d2; dist2[q + 2] = best.d3; }
      if (idx) { idx[q] = best.i1; idx[q + 1] = best.i2; idx[q + 2] = best.i3; }
    }
  }
  __syncthreads();
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const float *feat_b = known_feat_pm + static_cast<size_t>(b) * m * c;
  const int jn = min(kNnThreads, n - j0);
  for (int lj = warp; lj < jn; lj += kNnThreads / 32) {
    const float w1 = s_w[lj][0], w2 = s_w[lj][1], w3 = s_w[lj][2];
    const float *p1 = feat_b + static_cast<size_t>(s_i[lj][0]) * c;
    const float *p2 = feat_b + static_cast<size_t>(s_i[lj][1]) * c;
    const float *p3 = feat_b + static_cast<size_t>(s_i[lj][2]) * c;
    float *o = out_pm + (static_cast<size_t>(b) * n + j0 + lj) * ldo + col0;
    for (int ch = lane; ch < c; ch += 32)
      o[ch] = __fmaf_rn(__ldg(p3 + ch), w3, __fmaf_rn(__ldg(p1 + ch), w1, __fmul_rn(__ldg(p2 + ch), w2)));
  }
}

int channel_slices(int c, int other_ctas) {
  // enough CTAs to fill the chip (~4 waves), but never more slices than channels
  int want = ceil_div(4 * sm_count(), other_ctas > 0 ? other_ctas : 1);
  if (want < 1) want = 1;
  if (want > c) want = c;
  if (want > 65535) want = 65535;
  return want;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

// new_xyz[b, j, :] = xyz[b, idx[b, j], :] -- what the reference spells
// gather_operation(xyz.transpose(1,2).contiguous(), idx).transpose(1,2).contiguous() (pointnet2_modules.py:47-53)
__global__ void gather_xyz_kernel(const float *__restrict__ xyz, const int *__restrict__ idx, int n, long long total,
                                  int m, float *__restrict__ out) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const long long b = p / m;
  const float *src = xyz + (b * n + idx[p]) * 3;
  out[p * 3 + 0] = __ldg(src + 0);
  out[p * 3 + 1] = __ldg(src + 1);
  out[p * 3 + 2] = __ldg(src + 2);
}

extern "C" int pvn3d_gather_xyz(const float *xyz, const int *idx, int b, int n, int m, float *out,
                                pvn3d_stream_t stream) {
  if (!xyz || !idx || !out || b < 0 || n <= 0 || m < 0) return PVN3D_ERR_INVALID_ARG;
  const long long total = static_cast<long long>(b) * m;
  if (total == 0) return PVN3D_OK;
  gather_xyz_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, as_stream(stream)>>>(xyz, idx, n, total, m,
                                                                                               out);
  return check_launch("gather_xyz_kernel");
}

extern "C" int pvn3d_gather_points(const float *points, const int *idx, int b, int c, int n, int m,
                                   float *out, pvn3d_stream_t stream) {
  if (!points || !idx || !out || b < 0 || c < 0 || n <= 0 || m < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0 || m == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  const int gx = ceil_div(m, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  gather_points_kernel<<<grid, 256, 0, as_stream(stream)>>>(points, idx, c, n, m, out);
  return check_launch("gather_points_kernel");
}

extern "C" int pvn3d_gather_points_grad(const float *grad_out, const int *idx, int b, int c, int n,
                                        int m, float *grad_points, pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || n <= 0 || m < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  // an input with no elements may be null: torch hands out null data pointers for empty tensors
  if (!grad_points || (m > 0 && (!grad_out || !idx))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)n,
                                 as_stream(stream)),
                 "memset");
  if (m == 0) return PVN3D_OK;
  const int gx = ceil_div(m, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  gather_points_grad_kernel<<<grid, 256, 0, as_stream(stream)>>>(grad_out, idx, c, n, m,
                                                                 grad_points);
  return check_launch("gather_points_grad_kernel");
}

extern "C" int pvn3d_ball_query(const float *new_xyz, const float *xyz, int b, int n, int m,
                                float radius, int nsample, int *idx, pvn3d_stream_t stream) {
  if (!new_xyz || !xyz || !idx || b < 0 || n <= 0 || m < 0 || nsample < 0)
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || m == 0 || nsample == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  const size_t smem = kBqTile * 3 * sizeof(float) + sizeof(int) * kBqCentresPerCta * (size_t)nsample;
  if (smem > 200 * 1024) return PVN3D_ERR_UNSUPPORTED;  // nsample <= ~1400
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once,
                        cudaFuncSetAttribute(ball_query_kernel,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024),
                        "ball_query smem attr");
  dim3 grid(ceil_div(m, kBqCentresPerCta), b);
  ball_query_kernel<<<grid, kBqThreads, smem, as_stream(stream)>>>(new_xyz, xyz, n, m, radius,
                                                                   nsample, idx);
  return check_launch("ball_query_kernel");
}

extern "C" int pvn3d_group_points(const float *points, const int *idx, int b, int c, int n,
                                  int npoints, int nsample, float *out, pvn3d_stream_t stream) {
  if (!points || !idx || !out || b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0)
    return PVN3D_ERR_INVALID_ARG;
  const long long slots_ll = static_cast<long long>(npoints) * nsample;
  if (b == 0 || c == 0 || slots_ll == 0) return PVN3D_OK;
  if (b > 65535 || slots_ll > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  const int slots = static_cast<int>(slots_ll);
  const int gx = ceil_div(slots, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  group_points_kernel<float, 1><<<grid, 256, 0, as_stream(stream)>>>(points, idx, c, n, slots, out);
  return check_launch("group_points_kernel");
}

extern "C" int pvn3d_group_points_grad(const float *grad_out, const int *idx, int b, int c, int n,
                                       int npoints, int nsample, float *grad_points,
                                       pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  const long long slots_ll = static_cast<long long>(npoints) * nsample;
  if (!grad_points || (slots_ll > 0 && (!grad_out || !idx))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535 || slots_ll > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)n,
                                 as_stream(stream)),
                 "memset");
  if (slots_ll == 0) return PVN3D_OK;
  const int slots = static_cast<int>(slots_ll);
  const int gx = ceil_div(slots, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  group_points_grad_kernel<float><<<grid, 256, 0, as_stream(stream)>>>(grad_out, idx, c, n, slots,
                                                                grad_points);
  return check_launch("group_points_grad_kernel");
}

extern "C" int pvn3d_three_nn(const float *unknown, const float *known, int b, int n, int m,
                              float *dist2, int *idx, pvn3d_stream_t stream) {
  if (!unknown || !known || !dist2 || !idx || b < 0 || n < 0 || m < 0)
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || n == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  dim3 grid(ceil_div(n, kNnThreads), b);
  if (m >= 512 && m <= kNnSlabMaxM && n >= 2 * m) {
    // x-sorted copy of the known set (stream-ordered scratch), then the outward walk
    int m_pad = 1;
    while (m_pad < m) m_pad <<= 1;
    const size_t smem = static_cast<size_t>(m_pad) * sizeof(float4);
    static PerDeviceOnce once;
    if (once.pending()) {
      PVN3D_CUDA_TRY(cudaFuncSetAttribute(nn_sort_known_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          kNnSlabMaxM * (int)sizeof(float4)), "nn sort smem attr");
      once.mark();
    }
    int rc = keep_async_pool_warm();
    if (rc != PVN3D_OK) return rc;
    float4 *sorted = nullptr;
    PVN3D_CUDA_TRY(cudaMallocAsync(&sorted, static_cast<size_t>(b) * m_pad * sizeof(float4), as_stream(stream)),
                   "three_nn scratch alloc");
    nn_sort_known_kernel<<<b, 512, smem, as_stream(stream)>>>(known, m, m_pad, sorted);
    rc = check_launch("nn_sort_known_kernel");
    if (rc == PVN3D_OK) {
      three_nn_slab_kernel<<<grid, kNnThreads, 0, as_stream(stream)>>>(
          unknown, sorted, n, m, m_pad, dist2, idx);
      rc = check_launch("three_nn_slab_kernel");
    }
    cudaFreeAsync(sorted, as_stream(stream));
    return rc;
  }
  three_nn_kernel<<<grid, kNnThreads, 0, as_stream(stream)>>>(unknown, known, n, m, dist2, idx);
  return check_launch("three_nn_kernel");
}

extern "C" int pvn3d_three_nn_grid_supported(int n, int m) { return n >= 1 && m >= 1 && m <= kNnGridMaxM; }

extern "C" int pvn3d_three_nn_weights_levels(int nlev, const float *const *unknown, const float *const *known,
                                             const int *n, const int *m, int b, float *const *dist2, int *const *idx,
                                             float *const *weight, pvn3d_stream_t stream) {
  if (nlev < 0 || nlev > kNnGridMaxLevels || b < 0 || (nlev > 0 && (!unknown || !known || !n || !m || !dist2 || !idx ||
                                                                     !weight)))
    return PVN3D_ERR_INVALID_ARG;
  for (int l = 0; l < nlev; ++l)
    if (!unknown[l] || !known[l] || !dist2[l] || !idx[l] || !weight[l] || n[l] < 0 || m[l] < 0)
      return PVN3D_ERR_INVALID_ARG;
  if (b == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  // levels outside the grid's shape rule: today's 3-NN, then the weights
  NnGridArgs a{};
  size_t bytes = 0;
  long long blocks = 0;
  for (int l = 0; l < nlev; ++l) {
    if (!pvn3d_three_nn_grid_supported(n[l], m[l])) {
      int rc = pvn3d_three_nn(unknown[l], known[l], b, n[l], m[l], dist2[l], idx[l], stream);
      if (rc == PVN3D_OK) rc = pvn3d_three_nn_weights(dist2[l], static_cast<long long>(b) * n[l], weight[l], stream);
      if (rc != PVN3D_OK) return rc;
      continue;
    }
    NnGridLevel &L = a.lv[a.nlev++];
    L.unknown = unknown[l]; L.known = known[l]; L.dist2 = dist2[l]; L.idx = idx[l]; L.weight = weight[l];
    L.n = n[l]; L.m = m[l];
    L.blk0 = static_cast<int>(blocks);
    blocks += ceil_div(n[l], kNnThreads);
    bytes += align_up(sizeof(float4) * b * m[l], 256) + align_up(sizeof(int) * b * (kNnGridCells + 1), 256) +
             align_up(sizeof(NnGridHdr) * b, 256);
  }
  if (a.nlev == 0) return PVN3D_OK;
  if (blocks > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  int rc = keep_async_pool_warm();
  if (rc != PVN3D_OK) return rc;
  unsigned char *scratch = nullptr;
  PVN3D_CUDA_TRY(cudaMallocAsync(&scratch, bytes, st), "three_nn grid scratch");
  unsigned char *p = scratch;
  for (int l = 0; l < a.nlev; ++l) {
    NnGridLevel &L = a.lv[l];
    L.sorted = reinterpret_cast<float4 *>(p);
    p += align_up(sizeof(float4) * b * L.m, 256);
    L.cell_start = reinterpret_cast<int *>(p);
    p += align_up(sizeof(int) * b * (kNnGridCells + 1), 256);
    L.hdr = reinterpret_cast<NnGridHdr *>(p);
    p += align_up(sizeof(NnGridHdr) * b, 256);
  }
  nn_grid_build_kernel<<<dim3(b, a.nlev), kNnGridBuildThreads, 0, st>>>(a);
  rc = check_launch("nn_grid_build_kernel");
  if (rc == PVN3D_OK) {
    three_nn_grid_kernel<<<dim3(static_cast<unsigned>(blocks), b), kNnThreads, 0, st>>>(a);
    rc = check_launch("three_nn_grid_kernel");
  }
  cudaFreeAsync(scratch, st);
  return rc;
}

extern "C" int pvn3d_ball_grid_supported(int n, int m, int ns0, int ns1) {
  return n >= 1 && n < (1 << 30) && m >= 1 && ns0 >= 1 && ns1 >= 1 && ns0 <= kBgMaxNs && ns1 <= kBgMaxNs;
}

extern "C" int pvn3d_ball_query2_levels(int nlev, const float *const *xyz, const float *const *new_xyz, const int *n,
                                        const int *m, int b, const float *radius0, const int *ns0, int *const *idx0,
                                        const float *radius1, const int *ns1, int *const *idx1,
                                        pvn3d_stream_t stream) {
  if (nlev < 0 || nlev > kNnGridMaxLevels || b < 0 ||
      (nlev > 0 && (!xyz || !new_xyz || !n || !m || !radius0 || !ns0 || !idx0 || !radius1 || !ns1 || !idx1)))
    return PVN3D_ERR_INVALID_ARG;
  for (int l = 0; l < nlev; ++l)
    if (!xyz[l] || !new_xyz[l] || !idx0[l] || !idx1[l] || n[l] <= 0 || m[l] < 0 || ns0[l] <= 0 || ns1[l] <= 0)
      return PVN3D_ERR_INVALID_ARG;
  if (b == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  NnGridArgs grids{};
  BallGridArgs a{};
  size_t bytes = 0;
  long long blocks = 0;
  for (int l = 0; l < nlev; ++l) {
    if (m[l] == 0) continue;
    if (!pvn3d_ball_grid_supported(n[l], m[l], ns0[l], ns1[l])) {   // levels outside the rule: today's scan
      const int rc = pvn3d_query_and_group2(xyz[l], new_xyz[l], nullptr, 0, b, n[l], m[l], 0, radius0[l], ns0[l],
                                            idx0[l], nullptr, radius1[l], ns1[l], idx1[l], nullptr, stream);
      if (rc != PVN3D_OK) return rc;
      continue;
    }
    NnGridLevel &G = grids.lv[grids.nlev++];
    G.known = xyz[l];
    G.m = n[l];
    G.hmin = fmaxf(radius0[l], radius1[l]);
    BallGridLevel &L = a.lv[a.nlev++];
    L.xyz = xyz[l]; L.centres = new_xyz[l]; L.n = n[l]; L.m = m[l];
    L.r0 = radius0[l]; L.r1 = radius1[l]; L.ns0 = ns0[l]; L.ns1 = ns1[l]; L.idx0 = idx0[l]; L.idx1 = idx1[l];
    L.blk0 = static_cast<int>(blocks);
    blocks += ceil_div(m[l], kBgWarps);
    bytes += align_up(sizeof(float4) * b * (size_t)n[l], 256) + align_up(sizeof(int) * b * (kNnGridCells + 1), 256) +
             align_up(sizeof(NnGridHdr) * b, 256);
  }
  if (a.nlev == 0) return PVN3D_OK;
  if (blocks > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  int rc = keep_async_pool_warm();
  if (rc != PVN3D_OK) return rc;
  unsigned char *scratch = nullptr;
  PVN3D_CUDA_TRY(cudaMallocAsync(&scratch, bytes, st), "ball grid scratch");
  unsigned char *p = scratch;
  for (int l = 0; l < grids.nlev; ++l) {
    NnGridLevel &G = grids.lv[l];
    a.sorted[l] = G.sorted = reinterpret_cast<float4 *>(p);
    p += align_up(sizeof(float4) * b * (size_t)G.m, 256);
    a.cell_start[l] = G.cell_start = reinterpret_cast<int *>(p);
    p += align_up(sizeof(int) * b * (kNnGridCells + 1), 256);
    a.hdr[l] = G.hdr = reinterpret_cast<NnGridHdr *>(p);
    p += align_up(sizeof(NnGridHdr) * b, 256);
  }
  nn_grid_build_kernel<<<dim3(b, grids.nlev), kNnGridBuildThreads, 0, st>>>(grids);
  rc = check_launch("nn_grid_build_kernel");
  if (rc == PVN3D_OK) {
    ball_grid_kernel<<<dim3(static_cast<unsigned>(blocks), b), kBgWarps * 32, 0, st>>>(a);
    rc = check_launch("ball_grid_kernel");
  }
  cudaFreeAsync(scratch, st);
  return rc;
}

extern "C" int pvn3d_three_interpolate(const float *points, const int *idx, const float *weight,
                                       int b, int c, int m, int n, float *out,
                                       pvn3d_stream_t stream) {
  if (!points || !idx || !weight || !out || b < 0 || c < 0 || m <= 0 || n < 0)
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0 || n == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  const int gx = ceil_div(n, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  three_interpolate_kernel<float, 1><<<grid, 256, 0, as_stream(stream)>>>(points, idx, weight, c, m, n, out);
  return check_launch("three_interpolate_kernel");
}

extern "C" int pvn3d_three_interpolate_grad(const float *grad_out, const int *idx,
                                            const float *weight, int b, int c, int n, int m,
                                            float *grad_points, pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || m <= 0 || n < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  if (!grad_points || (n > 0 && (!grad_out || !idx || !weight))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)m,
                                 as_stream(stream)),
                 "memset");
  if (n == 0) return PVN3D_OK;
  const int gx = ceil_div(n, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  three_interpolate_grad_kernel<float><<<grid, 256, 0, as_stream(stream)>>>(grad_out, idx, weight, c, n, m,
                                                                     grad_points);
  return check_launch("three_interpolate_grad_kernel");
}

// ---- 16-bit forms (torch.autocast): the kernels above on __half / __nv_bfloat16 --------------------------------------
// the one rounding of a 16-bit atomic grad: scratch [count] f32 -> out [count] 16-bit
template <typename T>
static int round_scratch(const float *scratch, long long count, T *out, cudaStream_t st) {
  const bool pairs = aligned_to(scratch, 8) && aligned_to(out, 4);
  const long long work = pairs ? (count + 1) / 2 : count;
  const long long want = (work + 255) / 256, cap = 16ll * sm_count();
  const unsigned grid = static_cast<unsigned>(want < cap ? want : cap);
  if (pairs)
    round_to16_kernel<T, 2><<<grid, 256, 0, st>>>(scratch, count, out);
  else
    round_to16_kernel<T, 1><<<grid, 256, 0, st>>>(scratch, count, out);
  return check_launch("round_to16_kernel");
}

extern "C" int pvn3d_group_points_16(int dtype, const void *points, const int *idx, int b, int c, int n, int npoints,
                                     int nsample, void *out, pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (!points || !idx || !out || b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0)
      return PVN3D_ERR_INVALID_ARG;
    const long long slots_ll = static_cast<long long>(npoints) * nsample;
    if (b == 0 || c == 0 || slots_ll == 0) return PVN3D_OK;
    if (b > 65535 || slots_ll > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
    const int slots = static_cast<int>(slots_ll);
    const T *src = static_cast<const T *>(points);
    T *dst = static_cast<T *>(out);
    if (slots % 2 == 0 && aligned_to(idx, 8) && aligned_to(out, 4)) {
      const int gx = ceil_div(slots / 2, 256);
      dim3 grid(gx, channel_slices(c, gx * b), b);
      group_points_kernel<T, 2><<<grid, 256, 0, as_stream(stream)>>>(src, idx, c, n, slots, dst);
    } else {
      const int gx = ceil_div(slots, 256);
      dim3 grid(gx, channel_slices(c, gx * b), b);
      group_points_kernel<T, 1><<<grid, 256, 0, as_stream(stream)>>>(src, idx, c, n, slots, dst);
    }
    return check_launch("group_points_kernel");
  });
}

extern "C" int pvn3d_group_points_grad_16(int dtype, const void *grad_out, const int *idx, int b, int c, int n,
                                          int npoints, int nsample, float *scratch, void *grad_points,
                                          pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0) return PVN3D_ERR_INVALID_ARG;
    if (b == 0 || c == 0) return PVN3D_OK;
    const long long slots_ll = static_cast<long long>(npoints) * nsample;
    if (!grad_points || (slots_ll > 0 && (!grad_out || !idx || !scratch))) return PVN3D_ERR_INVALID_ARG;
    if (b > 65535 || slots_ll > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
    const size_t count = static_cast<size_t>(b) * c * n;
    cudaStream_t st = as_stream(stream);
    if (slots_ll == 0) {
      PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(T) * count, st), "memset");   // +0.0 in both formats
      return PVN3D_OK;
    }
    PVN3D_CUDA_TRY(cudaMemsetAsync(scratch, 0, sizeof(float) * count, st), "memset");
    const int slots = static_cast<int>(slots_ll);
    const int gx = ceil_div(slots, 256);
    dim3 grid(gx, channel_slices(c, gx * b), b);
    group_points_grad_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T *>(grad_out), idx, c, n, slots, scratch);
    const int rc = check_launch("group_points_grad_kernel");
    return rc != PVN3D_OK ? rc : round_scratch(scratch, static_cast<long long>(count), static_cast<T *>(grad_points), st);
  });
}

extern "C" int pvn3d_three_interpolate_16(int dtype, const void *points, const int *idx, const float *weight, int b,
                                          int c, int m, int n, void *out, pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (!points || !idx || !weight || !out || b < 0 || c < 0 || m <= 0 || n < 0) return PVN3D_ERR_INVALID_ARG;
    if (b == 0 || c == 0 || n == 0) return PVN3D_OK;
    if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
    const T *src = static_cast<const T *>(points);
    T *dst = static_cast<T *>(out);
    if (n % 2 == 0 && aligned_to(out, 4)) {
      const int gx = ceil_div(n / 2, 256);
      dim3 grid(gx, channel_slices(c, gx * b), b);
      three_interpolate_kernel<T, 2><<<grid, 256, 0, as_stream(stream)>>>(src, idx, weight, c, m, n, dst);
    } else {
      const int gx = ceil_div(n, 256);
      dim3 grid(gx, channel_slices(c, gx * b), b);
      three_interpolate_kernel<T, 1><<<grid, 256, 0, as_stream(stream)>>>(src, idx, weight, c, m, n, dst);
    }
    return check_launch("three_interpolate_kernel");
  });
}

extern "C" int pvn3d_three_interpolate_grad_16(int dtype, const void *grad_out, const int *idx, const float *weight,
                                               int b, int c, int n, int m, float *scratch, void *grad_points,
                                               pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (b < 0 || c < 0 || m <= 0 || n < 0) return PVN3D_ERR_INVALID_ARG;
    if (b == 0 || c == 0) return PVN3D_OK;
    if (!grad_points || (n > 0 && (!grad_out || !idx || !weight || !scratch))) return PVN3D_ERR_INVALID_ARG;
    if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
    const size_t count = static_cast<size_t>(b) * c * m;
    cudaStream_t st = as_stream(stream);
    if (n == 0) {
      PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(T) * count, st), "memset");
      return PVN3D_OK;
    }
    PVN3D_CUDA_TRY(cudaMemsetAsync(scratch, 0, sizeof(float) * count, st), "memset");
    const int gx = ceil_div(n, 256);
    dim3 grid(gx, channel_slices(c, gx * b), b);
    three_interpolate_grad_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T *>(grad_out), idx, weight, c, n, m,
                                                           scratch);
    const int rc = check_launch("three_interpolate_grad_kernel");
    return rc != PVN3D_OK ? rc : round_scratch(scratch, static_cast<long long>(count), static_cast<T *>(grad_points), st);
  });
}

static int launch_transpose(const float *src, int b, int rows, int cols, float *dst,
                            pvn3d_stream_t stream) {
  if (!src || !dst || b < 0 || rows < 0 || cols < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || rows == 0 || cols == 0) return PVN3D_OK;
  if (b > 65535 || ceil_div(rows, 32) > 65535) return PVN3D_ERR_UNSUPPORTED;
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32), b), block(32, 8);
  transpose_kernel<<<grid, block, 0, as_stream(stream)>>>(src, rows, cols, dst);
  return check_launch("transpose_kernel");
}

extern "C" int pvn3d_transpose_cn_to_nc(const float *src_bcn, int b, int c, int n, float *dst_bnc,
                                        pvn3d_stream_t stream) {
  return launch_transpose(src_bcn, b, c, n, dst_bnc, stream);
}
extern "C" int pvn3d_transpose_nc_to_cn(const float *src_bnc, int b, int n, int c, float *dst_bcn,
                                        pvn3d_stream_t stream) {
  return launch_transpose(src_bnc, b, n, c, dst_bcn, stream);
}

extern "C" int pvn3d_three_nn_interpolate(const float *unknown, const float *known,
                                          const float *known_feat_pm, int b, int n, int m, int c,
                                          float *out_pm, int ldo, int col0, float *dist2, int *idx,
                                          pvn3d_stream_t stream) {
  if (!unknown || !known || !known_feat_pm || !out_pm || b < 0 || n < 0 || m <= 0 || c < 0 ||
      col0 < 0 || ldo < col0 + c)
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || n == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  dim3 grid(ceil_div(n, kNnThreads), b);
  three_nn_interp_kernel<<<grid, kNnThreads, 0, as_stream(stream)>>>(
      unknown, known, known_feat_pm, n, m, c, out_pm, ldo, col0, dist2, idx);
  return check_launch("three_nn_interp_kernel");
}
