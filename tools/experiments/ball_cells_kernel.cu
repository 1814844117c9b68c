// PROTOTYPE (NOT linked into libpvn3d_b200.so), driven by tools/experiments/ball_cells_test.cu at level-1
// geometry (B=32, N=12288, M=2048, radii 0.0175/0.025): its first version was bit-exact against the CPU
//   restatement but slower than the shipped ball_scan_kernel (speed on the H100 not measured):
//   on a surface scene ~8 points fall into a voxel and most of the 27 neighbour buckets are empty, so the
//   warp spends 27 dependent bucket look-ups on steps that fill 0-8 of its 32 lanes.  The kernel below is
//   already v2 (prefix-summed ranges, lanes walk the CONCATENATED candidate list: ~200 candidates = 7 full
//   steps) -- it compiles and passes the same harness build, but the GPU budget ran out before it could run:
//   FIRST thing to do in round 2: `tools/experiments/ball_cells_test` (prints mismatches and both timings).
//
// ball query by cell list with the reference's exact first-nsample-in-index-order semantics.
// Algorithm + exactness argument: tools/experiments/ball_cells.py (checked against the oracle on CPU by
// tests/test_oracle_cpu.py::test_cell_list_ball_query_prototype_matches_oracle).
//
//   cells_build_kernel   one CTA per cloud: bounding box, voxel (edge = 1.001 r_max) -> bucket hash,
//                        histogram, exclusive scan, scatter of (x, y, z, index) into bucket order.
//   ball_cells_kernel    one warp per centre: the <= 27 distinct buckets around the centre's voxel, 32
//                        candidates per step tested with the reference's d2 (ref_sqdist), hits of both
//                        radii appended to per-warp shared-memory lists, bitonic sort by index, first
//                        nsample out, padding with the smallest index.  A ball with more hits than the
//                        list (dense cloud) is left to the index-order scan, which exits early there:
//                        overflow[b*m + j] = 1 tells the caller to run ball_scan_kernel for that centre.
//
// Compile check:  nvcc -gencode arch=compute_90a,code=sm_90a -I pvn3d_b200/csrc -I include -c \
//                      tools/experiments/ball_cells_kernel.cu -o /dev/null
#include "common.cuh"

namespace pvn3d {
namespace experiment {

constexpr int kCellBuckets = 4096;
constexpr int kCellListCap = 256;  // hits per (centre, radius) the sorted path can take
constexpr int kCellWarps = 8;

struct CellArgs {
  const float *xyz;      // [B][N][3]
  const float *new_xyz;  // [B][M][3]
  int n, m;
  float cell;            // 1.001 * r_max
  float4 *sorted;        // [B][N]  (x, y, z, index as int bits) in bucket order
  int *start;            // [B][kCellBuckets + 1]
  float *lo;             // [B][3]   bounding-box corner the voxel grid hangs on
  float r2[2];
  int ns[2];
  int *idx[2];           // [B][M][ns]
  unsigned char *overflow;  // [B][M]
};

__device__ __forceinline__ int cell_coord(float p, float lo, float inv_cell) {
  const float q = (p - lo) * inv_cell;  // monotone in p: a neighbour is within +-1 of the centre's voxel
  // NaN -> 0, +-inf / huge -> clamped: such points can never pass the distance test anyway
  return !(q == q) ? 0 : static_cast<int>(fminf(fmaxf(floorf(q), -1.0e6f), 1.0e6f));
}
__device__ __forceinline__ unsigned cell_hash(int i, int j, int k) {
  return (static_cast<unsigned>(i) * 73856093u ^ static_cast<unsigned>(j) * 19349663u ^
          static_cast<unsigned>(k) * 83492791u) & (kCellBuckets - 1);
}

__global__ void __launch_bounds__(1024) cells_build_kernel(CellArgs a) {
  __shared__ int s_cnt[kCellBuckets];
  __shared__ float s_red[3][32];
  __shared__ int s_warp[32];
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = lane_id(), warp = t >> 5;
  const float *cloud = a.xyz + static_cast<size_t>(b) * a.n * 3;
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f};
  for (int k = t; k < a.n; k += 1024)
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float v = cloud[static_cast<size_t>(k) * 3 + d];
      if (fabsf(v) < 3.0e38f) lo[d] = fminf(lo[d], v);
    }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
    if (lane == 0) s_red[d][warp] = lo[d];
  }
  for (int i = t; i < kCellBuckets; i += 1024) s_cnt[i] = 0;
  __syncthreads();
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float v = s_red[d][0];
    for (int w = 1; w < 32; ++w) v = fminf(v, s_red[d][w]);
    lo[d] = v;
  }
  if (t < 3) a.lo[b * 3 + t] = lo[t];
  const float inv = 1.0f / a.cell;
  auto bucket_of = [&](int k) {
    const float *p = cloud + static_cast<size_t>(k) * 3;
    return cell_hash(cell_coord(p[0], lo[0], inv), cell_coord(p[1], lo[1], inv), cell_coord(p[2], lo[2], inv));
  };
  for (int k = t; k < a.n; k += 1024) atomicAdd(&s_cnt[bucket_of(k)], 1);
  __syncthreads();
  // exclusive scan of the 4096 counts: 4 per thread
  int c[4], sum = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) { c[i] = s_cnt[4 * t + i]; sum += c[i]; }
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (static_cast<int>(lane) >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int base = 0;
  for (int w = 0; w < static_cast<int>(warp); ++w) base += s_warp[w];
  int run = base + incl - sum;
  __syncthreads();
  int *start = a.start + static_cast<size_t>(b) * (kCellBuckets + 1);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    s_cnt[4 * t + i] = run;  // becomes the scatter cursor
    start[4 * t + i] = run;
    run += c[i];
  }
  if (t == 1023) start[kCellBuckets] = run;
  __syncthreads();
  float4 *sorted = a.sorted + static_cast<size_t>(b) * a.n;
  for (int k = t; k < a.n; k += 1024) {
    const float *p = cloud + static_cast<size_t>(k) * 3;
    const int pos = atomicAdd(&s_cnt[bucket_of(k)], 1);
    sorted[pos] = make_float4(p[0], p[1], p[2], __int_as_float(k));
  }
}

// ascending bitonic sort of `p2` (power of two, <= kCellListCap) ints in shared memory by one warp
__device__ __forceinline__ void warp_bitonic(int *v, int p2, unsigned lane) {
  for (int k = 2; k <= p2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < p2; i += 32) {
        const int l = i ^ j;
        if (l > i) {
          const int x = v[i], y = v[l];
          if ((x > y) == ((i & k) == 0)) { v[i] = y; v[l] = x; }
        }
      }
      __syncwarp();
    }
}

__global__ void __launch_bounds__(kCellWarps * 32) ball_cells_kernel(CellArgs a) {
  __shared__ int s_list[kCellWarps][2][kCellListCap];
  __shared__ int s_pre[kCellWarps][32], s_beg[kCellWarps][32];
  const int b = blockIdx.y;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const int j = blockIdx.x * kCellWarps + static_cast<int>(warp);
  if (j >= a.m) return;
  const float *c = a.new_xyz + (static_cast<size_t>(b) * a.m + j) * 3;
  const float cx = c[0], cy = c[1], cz = c[2];
  const float inv = 1.0f / a.cell;
  const float *lo = a.lo + b * 3;
  const int ci = cell_coord(cx, lo[0], inv), cj = cell_coord(cy, lo[1], inv), ck = cell_coord(cz, lo[2], inv);
  // lane l < 27: bucket of neighbour voxel l; only the lowest lane of equal buckets keeps it
  unsigned bucket = 0xffffffffu;
  if (lane < 27) bucket = cell_hash(ci + static_cast<int>(lane % 3) - 1, cj + static_cast<int>(lane / 3 % 3) - 1,
                                    ck + static_cast<int>(lane / 9) - 1);
  const unsigned same = __match_any_sync(0xffffffffu, bucket);
  const bool leader = lane < 27 && (__ffs(same) - 1) == static_cast<int>(lane);
  const int *start = a.start + static_cast<size_t>(b) * (kCellBuckets + 1);
  const float4 *sorted = a.sorted + static_cast<size_t>(b) * a.n;
  // v2 (not yet run): the <= 27 bucket ranges are CONCATENATED -- lane l owns range l, an exclusive
  // prefix sum of the lengths gives every candidate a rank, and the warp walks the ranks 32 at a time
  // (v1 walked bucket by bucket: 27 dependent look-ups for steps that filled 0-8 lanes on surface scenes)
  const int rs = leader ? start[bucket] : 0;
  const int rl = leader ? start[bucket + 1] - rs : 0;
  int incl = rl;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (static_cast<int>(lane) >= o) incl += v;
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  s_pre[warp][lane] = incl - rl;  // rank of the first candidate of range `lane`
  s_beg[warp][lane] = rs;
  __syncwarp();
  int cnt[2] = {0, 0};
  for (int base = 0; base < total; base += 32) {
    const int g = base + static_cast<int>(lane);
    const bool in = g < total;
    // owner = last range whose first rank is <= g (empty ranges share a rank with their successor and lose)
    int lo_r = 0, hi_r = 31;
    while (lo_r < hi_r) {
      const int mid = (lo_r + hi_r + 1) >> 1;
      if (s_pre[warp][mid] <= (in ? g : 0)) lo_r = mid; else hi_r = mid - 1;
    }
    const int q = s_beg[warp][lo_r] + ((in ? g : 0) - s_pre[warp][lo_r]);
    const float4 p = sorted[in ? q : 0];
    const float d2 = ref_sqdist(cx - p.x, cy - p.y, cz - p.z);  // ball_query_gpu.cu:31-33
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const unsigned hits = __ballot_sync(0xffffffffu, in && d2 < a.r2[r]);
      const int slot = cnt[r] + __popc(hits & lanemask_lt());
      if (((hits >> lane) & 1u) && slot < kCellListCap) s_list[warp][r][slot] = __float_as_int(p.w);
      cnt[r] += __popc(hits);
    }
  }
  __syncwarp();
  bool over = false;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    int *out = a.idx[r] + (static_cast<size_t>(b) * a.m + j) * a.ns[r];
    if (cnt[r] > kCellListCap) { over = true; continue; }  // dense ball: the index-order scan takes it
    int p2 = 1;
    while (p2 < cnt[r]) p2 <<= 1;
    for (int i = cnt[r] + static_cast<int>(lane); i < p2; i += 32) s_list[warp][r][i] = 0x7fffffff;
    __syncwarp();
    warp_bitonic(s_list[warp][r], p2, lane);
    const int first = cnt[r] ? s_list[warp][r][0] : 0;  // empty ball: zeros (torch::zeros, ball_query.cpp:19)
    for (int sl = static_cast<int>(lane); sl < a.ns[r]; sl += 32) out[sl] = sl < cnt[r] ? s_list[warp][r][sl] : first;
  }
  if (lane == 0) a.overflow[static_cast<size_t>(b) * a.m + j] = over ? 1 : 0;
}

}  // namespace experiment
}  // namespace pvn3d
