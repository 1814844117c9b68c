// flat_meanshift.cu -- batched flat-kernel mean shift (sklearn MeanShift(bandwidth, bin_seeding=True))
// over float64 point segments, one CTA per segment; the algorithm is in flat_meanshift.cuh.
#include "flat_meanshift.cuh"

namespace pvn3d {
namespace {

__global__ void __launch_bounds__(kFlatMsThreads, 1)
flat_ms_segments_kernel(const double *__restrict__ X, const int *__restrict__ fit_off, int cap, double bw,
                        int max_iter, int *labels, double *centres, int *counts, int *n_clusters, int *n_iter) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int f = blockIdx.x, t = threadIdx.x;
  const int p0 = fit_off[f], n = fit_off[f + 1] - p0;
  if (n < 1 || n > cap) {  // empty, or larger than the launch's max_fit_pts: nothing is clustered
    for (int i = t; i < n; i += kFlatMsThreads) labels[p0 + i] = -1;
    if (t == 0) {
      n_clusters[f] = n < 1 ? 0 : -1;
      n_iter[f] = 0;
    }
    return;
  }
  const FlatMsSmem s = flat_ms_smem(smem, cap);
  for (int i = t; i < n; i += kFlatMsThreads) {
    const double *p = X + static_cast<size_t>(p0 + i) * 3;
    s.x[i] = p[0];
    s.y[i] = p[1];
    s.z[i] = p[2];
  }
  __syncthreads();
  FlatMsOut o{};
  o.centres = centres + static_cast<size_t>(p0) * 3;
  o.counts = counts ? counts + p0 : nullptr;
  o.labels = labels + p0;
  o.n_clusters = n_clusters + f;
  o.n_iter = n_iter + f;
  flat_ms_cta(s, n, bw, max_iter, o);
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_flat_ms_fit_batch(const double *X, const int *fit_off, int n_fits, int max_fit_pts,
                                       double bandwidth, int max_iter, int *labels_out, double *centres_out,
                                       int *counts_out, int *n_clusters_out, int *n_iter_out,
                                       pvn3d_stream_t stream) {
  if (!fit_off || !labels_out || !centres_out || !n_clusters_out || !n_iter_out || n_fits < 0 ||
      max_fit_pts < 0 || !(bandwidth > 0.0) || !(bandwidth < INFINITY) || max_iter < 0 || (max_fit_pts > 0 && !X))
    return PVN3D_ERR_INVALID_ARG;
  if (max_fit_pts > kFlatMsMaxPts) return PVN3D_ERR_UNSUPPORTED;
  if (n_fits == 0) return PVN3D_OK;
  const size_t smem = flat_ms_smem_bytes(max_fit_pts);
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once,
                        cudaFuncSetAttribute(flat_ms_segments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(flat_ms_smem_bytes(kFlatMsMaxPts))),
                        "flat_ms_segments_kernel smem");
  flat_ms_segments_kernel<<<n_fits, kFlatMsThreads, smem, as_stream(stream)>>>(
      X, fit_off, max_fit_pts < 1 ? 1 : max_fit_pts, bandwidth, max_iter, labels_out, centres_out, counts_out,
      n_clusters_out, n_iter_out);
  return check_launch("flat_ms_segments_kernel");
}
