// runtime.cu -- error plumbing and device queries behind the C ABI.
#include <cmath>
#include <cstring>

#include "common.cuh"

namespace pvn3d {

static thread_local char g_last_err[256] = "";
static unsigned long long g_launches = 0ull;

void count_launch() { __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED); }

void note_cuda_error(cudaError_t e, const char *where) {
  snprintf(g_last_err, sizeof(g_last_err), "%s: %s (%s)", where, cudaGetErrorString(e),
           cudaGetErrorName(e));
}

int sm_count() {
  static int cached = 0;
  if (cached > 0) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;
  cached = n;
  return n;
}

int keep_async_pool_warm() {
  // cudaMallocAsync scratch (query_group box tables, FPS fallback): by default the device pool hands
  // memory back to the OS at every synchronisation, which makes the next allocation slow.  Keep it.
  static PerDeviceOnce once;
  if (!once.pending()) return PVN3D_OK;
  int dev = 0;
  PVN3D_CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
  cudaMemPool_t pool;
  PVN3D_CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, dev), "default mempool");
  unsigned long long keep = ~0ull;
  PVN3D_CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep), "mempool threshold");
  once.mark();
  return PVN3D_OK;
}

int ref_opt_n_threads(int work_size) {
  // reference: cuda_utils.h:15-19 -- pow_2 = log(work)/log(2) truncated; clamp(1<<pow_2, 1, 512)
  const int pow_2 = static_cast<int>(std::log(static_cast<double>(work_size)) / std::log(2.0));
  int v = 1 << pow_2;
  if (v > 512) v = 512;
  if (v < 1) v = 1;
  return v;
}

}  // namespace pvn3d

extern "C" {

int pvn3d_version(void) { return 1; }

unsigned long long pvn3d_launch_count(void) {
  return __atomic_load_n(&pvn3d::g_launches, __ATOMIC_RELAXED);
}

const char *pvn3d_strerror(int code) {
  switch (code) {
    case PVN3D_OK: return "ok";
    case PVN3D_ERR_INVALID_ARG: return "invalid argument";
    case PVN3D_ERR_UNSUPPORTED: return "unsupported size";
    case PVN3D_ERR_CUDA: return "CUDA error";
    case PVN3D_ERR_WORKSPACE: return "workspace too small";
    default: return "unknown error";
  }
}

const char *pvn3d_last_cuda_error(void) { return pvn3d::g_last_err; }

int pvn3d_device_sm_count(int *sm, int *major, int *minor) {
  int dev = 0;
  PVN3D_CUDA_TRY(cudaGetDevice(&dev), "cudaGetDevice");
  int v = 0;
  if (sm) {
    PVN3D_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev), "attr");
    *sm = v;
  }
  if (major) {
    PVN3D_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev), "attr");
    *major = v;
  }
  if (minor) {
    PVN3D_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev), "attr");
    *minor = v;
  }
  return PVN3D_OK;
}

}  // extern "C"
