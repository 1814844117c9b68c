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
// One thread per (j,k) slot, looping over a slice of channels: idx is read once per slice, the
// output is written coalesced along the slot axis.
// ------------------------------------------------------------------------------------------------
__global__ void group_points_kernel(const float *__restrict__ points, const int *__restrict__ idx,
                                    int c, int n, int slots, float *__restrict__ out) {
  const int b = blockIdx.z;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  const int ii = idx[static_cast<size_t>(b) * slots + s];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const size_t row = static_cast<size_t>(b) * c + l;
    stg_stream(out + row * slots + s, __ldg(points + row * n + ii));
  }
}

__global__ void group_points_grad_kernel(const float *__restrict__ grad_out,
                                         const int *__restrict__ idx, int c, int n, int slots,
                                         float *__restrict__ grad_points) {
  const int b = blockIdx.z;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= slots) return;
  const int ii = idx[static_cast<size_t>(b) * slots + s];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const size_t row = static_cast<size_t>(b) * c + l;
    atomicAdd(grad_points + row * n + ii, grad_out[row * slots + s]);  // group_points_gpu.cu:60
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

// ------------------------------------------------------------------------------------------------
// three_interpolate: out[b,c,j] = sum_t points[b,c,idx[b,j,t]] * w[b,j,t]   (interpolate_gpu.cu:72-101)
// contraction as in the reference SASS (oracle/_ref build, interpolate_gpu.o):
//   t = p2*w2 (FMUL); t = fma(p1,w1,t); out = fma(p3,w3,t)  -- the MIDDLE product is the bare multiply
// ------------------------------------------------------------------------------------------------
__global__ void three_interpolate_kernel(const float *__restrict__ points,
                                         const int *__restrict__ idx,
                                         const float *__restrict__ weight, int c, int m, int n,
                                         float *__restrict__ out) {
  const int b = blockIdx.z;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t q = (static_cast<size_t>(b) * n + j) * 3;
  const float w1 = weight[q], w2 = weight[q + 1], w3 = weight[q + 2];
  const int i1 = idx[q], i2 = idx[q + 1], i3 = idx[q + 2];
  for (int l = blockIdx.y; l < c; l += gridDim.y) {
    const float *row = points + (static_cast<size_t>(b) * c + l) * m;
    const float v = __fmaf_rn(__ldg(row + i3), w3,
                              __fmaf_rn(__ldg(row + i1), w1, __fmul_rn(__ldg(row + i2), w2)));
    out[(static_cast<size_t>(b) * c + l) * n + j] = v;
  }
}

__global__ void three_interpolate_grad_kernel(const float *__restrict__ grad_out,
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
    const float g = grad_out[(static_cast<size_t>(b) * c + l) * n + j];
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
    // dist = sqrt(dist2) (pointnet2_utils.py:126); 1/(dist+1e-8); normalise (modules.py:184-186)
    const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(best.d1), 1e-8f));
    const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(best.d2), 1e-8f));
    const float r3 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(best.d3), 1e-8f));
    const float norm = __fadd_rn(__fadd_rn(r1, r2), r3);
    s_w[threadIdx.x][0] = __fdiv_rn(r1, norm);
    s_w[threadIdx.x][1] = __fdiv_rn(r2, norm);
    s_w[threadIdx.x][2] = __fdiv_rn(r3, norm);
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
  group_points_kernel<<<grid, 256, 0, as_stream(stream)>>>(points, idx, c, n, slots, out);
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
  group_points_grad_kernel<<<grid, 256, 0, as_stream(stream)>>>(grad_out, idx, c, n, slots,
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

extern "C" int pvn3d_three_interpolate(const float *points, const int *idx, const float *weight,
                                       int b, int c, int m, int n, float *out,
                                       pvn3d_stream_t stream) {
  if (!points || !idx || !weight || !out || b < 0 || c < 0 || m <= 0 || n < 0)
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0 || n == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  const int gx = ceil_div(n, 256);
  dim3 grid(gx, channel_slices(c, gx * b), b);
  three_interpolate_kernel<<<grid, 256, 0, as_stream(stream)>>>(points, idx, weight, c, m, n, out);
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
  three_interpolate_grad_kernel<<<grid, 256, 0, as_stream(stream)>>>(grad_out, idx, weight, c, n, m,
                                                                     grad_points);
  return check_launch("three_interpolate_grad_kernel");
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
