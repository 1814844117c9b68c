// fps.cu -- furthest point sampling for sm_90a.
//
// Replaces furthest_point_sampling (reference pvn3d/_ext-src/src/sampling.cpp:65-86 and
// sampling_gpu.cu:69-229).  Same result bit for bit, different machine mapping:
//
//   reference : one 512-thread CTA per cloud; per iteration every thread re-reads its points
//               AND the running min-distance array `temp` from global memory, then a 10-level
//               shared-memory tree with 10 __syncthreads picks the arg-max.
//   here      : one CTA per cloud with the cloud resident on chip for the whole run: each thread
//               keeps its points (x,y,z) and their running min-distance in REGISTERS, the
//               per-iteration arg-max is two REDUX.MAX per warp + one shared-memory hop + ONE
//               barrier, and the winner's coordinates come from a shared-memory copy of the cloud.
//               HBM traffic = the cloud once + the index list (the algorithmic minimum).
//
// Tie-break (SURVEY App. A.1, re-derived from sampling_gpu.cu:59-65,108-168): the reference thread
// `tid = k mod bs` (bs = opt_n_threads(n)) keeps the lowest k among its equal maxima (strict '>'),
// and every tree level keeps the LOWER slot on ties, the last level being (0,1).  Among equal
// values the winner is therefore the candidate with the smallest bit-reversed tid, then the
// smallest k/bs.  We fold that order into a 32-bit priority and reduce the pair
// (value bits, ~priority) with integer max, which reproduces the reference exactly for any mapping
// of points to threads.
#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kFpsThreads = 512;  // multiple of every reference block size (<= 512)

__device__ __forceinline__ uint32_t fps_prio(int k, int log2_bs) {
  const uint32_t tid_ref = static_cast<uint32_t>(k) & ((1u << log2_bs) - 1u);
  const uint32_t rev = log2_bs ? (__brev(tid_ref) >> (32 - log2_bs)) : 0u;
  return (rev << 22) | (static_cast<uint32_t>(k) >> log2_bs);
}
__device__ __forceinline__ int fps_decode(uint32_t prio, int log2_bs) {
  const uint32_t q = prio & 0x3FFFFFu;
  const uint32_t rev = prio >> 22;
  const uint32_t tid_ref = log2_bs ? (__brev(rev) >> (32 - log2_bs)) : 0u;
  return static_cast<int>((q << log2_bs) | tid_ref);
}

// value key: -1 (thread saw no eligible point) -> 0 ; v >= +0 -> bits(v)+1 (monotone for v >= 0)
__device__ __forceinline__ uint32_t fps_value_key(float best) {
  return best < 0.0f ? 0u : (__float_as_uint(best) + 1u);
}

// Block-wide arg-max of (hi, lo) pairs; returns the winning index (0 when nobody was eligible).
template <int NT>
__device__ __forceinline__ int fps_block_argmax(uint32_t hi, uint32_t lo, uint32_t (*s_hi)[32],
                                                uint32_t (*s_lo)[32], int parity, int log2_bs) {
  constexpr int NW = NT / 32;
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t whi = __reduce_max_sync(0xffffffffu, hi);
  uint32_t wlo = __reduce_max_sync(0xffffffffu, hi == whi ? lo : 0u);
  if (lane == 0) {
    s_hi[parity][warp] = whi;
    s_lo[parity][warp] = wlo;
  }
  __syncthreads();
  uint32_t vhi = lane < NW ? s_hi[parity][lane] : 0u;
  uint32_t vlo = lane < NW ? s_lo[parity][lane] : 0u;
  uint32_t ghi = __reduce_max_sync(0xffffffffu, vhi);
  uint32_t glo = __reduce_max_sync(0xffffffffu, vhi == ghi ? vlo : 0u);
  return ghi == 0u ? 0 : fps_decode(~glo, log2_bs);
}

// Register-resident variant: n <= NT*PPT, cloud also mirrored in shared memory (3*n floats).
template <int NT, int PPT>
__global__ void __launch_bounds__(NT, 1)
fps_regs_kernel(const float *__restrict__ xyz, int n, int m, int log2_bs, int *__restrict__ out) {
  extern __shared__ float s_xyz[];
  __shared__ uint32_t s_hi[2][32];
  __shared__ uint32_t s_lo[2][32];
  if (m <= 0) return;

  const int t = threadIdx.x;
  xyz += static_cast<size_t>(blockIdx.x) * n * 3;
  out += static_cast<size_t>(blockIdx.x) * m;

  for (int i = t; i < n * 3; i += NT) s_xyz[i] = __ldg(xyz + i);
  __syncthreads();

  float px[PPT], py[PPT], pz[PPT], md[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) {
    const int k = t + i * NT;
    px[i] = py[i] = pz[i] = 0.0f;
    md[i] = -1.0f;  // ineligible: min(d, -1) = -1 can never beat the thread-local best of -1
    if (k < n) {
      const float x = s_xyz[k * 3 + 0], y = s_xyz[k * 3 + 1], z = s_xyz[k * 3 + 2];
      // reference: mag = x*x + y*y + z*z contracted fmul(y,y), fma(x,x), fma(z,z); skip when
      // (double)mag <= 1e-3 (sampling_gpu.cu:100-101, the literal is a double)
      const float mag = __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
      if (!(static_cast<double>(mag) <= 1e-3)) {
        px[i] = x;
        py[i] = y;
        pz[i] = z;
        md[i] = 1e10f;  // sampling.cpp:73-75
      }
    }
  }

  int old = 0;
  if (t == 0) out[0] = 0;
  float ox = s_xyz[0], oy = s_xyz[1], oz = s_xyz[2];

  for (int j = 1; j < m; ++j) {
    float best = -1.0f;
    int bi = 0;
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
      const float d = ref_sqdist(px[i] - ox, py[i] - oy, pz[i] - oz);
      const float d2 = fminf(d, md[i]);
      md[i] = d2;
      if (d2 > best) {  // strict: lowest k of this thread wins its ties (sampling_gpu.cu:108-109)
        best = d2;
        bi = i;
      }
    }
    const uint32_t hi = fps_value_key(best);
    const uint32_t lo = ~fps_prio(t + bi * NT, log2_bs);
    old = fps_block_argmax<NT>(hi, lo, s_hi, s_lo, j & 1, log2_bs);
    ox = s_xyz[old * 3 + 0];
    oy = s_xyz[old * 3 + 1];
    oz = s_xyz[old * 3 + 2];
    if (t == 0) out[j] = old;
  }
}

// Generic variant for clouds too large for registers: min-distances in a global scratch array.
template <int NT>
__global__ void __launch_bounds__(NT, 1)
fps_generic_kernel(const float *__restrict__ xyz, int n, int m, int log2_bs,
                   float *__restrict__ temp, int *__restrict__ out) {
  __shared__ uint32_t s_hi[2][32];
  __shared__ uint32_t s_lo[2][32];
  if (m <= 0) return;
  const int t = threadIdx.x;
  xyz += static_cast<size_t>(blockIdx.x) * n * 3;
  temp += static_cast<size_t>(blockIdx.x) * n;
  out += static_cast<size_t>(blockIdx.x) * m;

  for (int k = t; k < n; k += NT) {
    const float x = xyz[k * 3 + 0], y = xyz[k * 3 + 1], z = xyz[k * 3 + 2];
    const float mag = __fmaf_rn(z, z, __fmaf_rn(x, x, __fmul_rn(y, y)));
    temp[k] = (static_cast<double>(mag) <= 1e-3) ? -1.0f : 1e10f;
  }
  int old = 0;
  if (t == 0) out[0] = 0;
  __syncthreads();
  for (int j = 1; j < m; ++j) {
    const float ox = xyz[old * 3 + 0], oy = xyz[old * 3 + 1], oz = xyz[old * 3 + 2];
    float best = -1.0f;
    int bk = 0;
    for (int k = t; k < n; k += NT) {
      const float tk = temp[k];
      const float d = ref_sqdist(xyz[k * 3 + 0] - ox, xyz[k * 3 + 1] - oy, xyz[k * 3 + 2] - oz);
      const float d2 = fminf(d, tk);
      temp[k] = d2;
      if (d2 > best) {
        best = d2;
        bk = k;
      }
    }
    old = fps_block_argmax<NT>(fps_value_key(best), ~fps_prio(bk, log2_bs), s_hi, s_lo, j & 1,
                               log2_bs);
    if (t == 0) out[j] = old;
  }
}

template <int PPT>
int launch_regs(const float *xyz, int b, int n, int m, int log2_bs, int *idx, cudaStream_t st) {
  auto kern = fps_regs_kernel<kFpsThreads, PPT>;
  const size_t smem = static_cast<size_t>(n) * 3 * sizeof(float);
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once,
                        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kFpsThreads * PPT * 3 * (int)sizeof(float)),
                        "fps smem attr");
  kern<<<b, kFpsThreads, smem, st>>>(xyz, n, m, log2_bs, idx);
  return check_launch("fps_regs_kernel");
}

}  // namespace
}  // namespace pvn3d

extern "C" int pvn3d_furthest_point_sampling(const float *xyz, int b, int n, int m, int *idx,
                                             pvn3d_stream_t stream) {
  using namespace pvn3d;
  if (!xyz || !idx || b < 0 || n <= 0 || m < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || m == 0) return PVN3D_OK;
  cudaStream_t st = as_stream(stream);
  const int bs_ref = ref_opt_n_threads(n);
  int log2_bs = 0;
  while ((1 << (log2_bs + 1)) <= bs_ref) ++log2_bs;
  if ((static_cast<long long>(n) >> log2_bs) >= (1ll << 22)) return PVN3D_ERR_UNSUPPORTED;

  const int ppt = ceil_div(n, kFpsThreads);
  if (ppt <= 1) return launch_regs<1>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 2) return launch_regs<2>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 4) return launch_regs<4>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 8) return launch_regs<8>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 12) return launch_regs<12>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 16) return launch_regs<16>(xyz, b, n, m, log2_bs, idx, st);
  if (ppt <= 24) return launch_regs<24>(xyz, b, n, m, log2_bs, idx, st);

  // large clouds: stream-ordered scratch for the running min-distances
  int rc0 = keep_async_pool_warm();
  if (rc0 != PVN3D_OK) return rc0;
  float *temp = nullptr;
  PVN3D_CUDA_TRY(cudaMallocAsync(&temp, static_cast<size_t>(b) * n * sizeof(float), st),
                 "fps scratch alloc");
  fps_generic_kernel<kFpsThreads><<<b, kFpsThreads, 0, st>>>(xyz, n, m, log2_bs, temp, idx);
  int rc = check_launch("fps_generic_kernel");
  cudaFreeAsync(temp, st);
  return rc;
}
