// metrics.cu -- the callers either side of the hot path, on device (SURVEY section 8 f4):
//
//   seg_argmax   per-point class id = argmax over the segmentation logits -- `_, classes_rgbd =
//                torch.max(pred_rgbd_seg, -1)` (reference pvn3d/demo.py:108, train_*_pvn3d.py eval path) --
//                written as the int32 mask pvn3d_frame_poses_batch consumes, so the pipeline input is the
//                network output and no int64 label tensor is materialised.
//   add / add-s  the two pose-error metrics of the evaluation loop, Basic_Utils.cal_add_cuda /
//                cal_adds_cuda (reference pvn3d/lib/utils/basic_utils.py:617-635).  ADD-S is an N x N
//                nearest-neighbour search like the mean-shift density pass; the reference materialises two
//                [N,N,3] tensors per object for it.  pvn3d_pose_add_adds scores F pose pairs over one mesh;
//                pvn3d_frame_add_adds scores every ground-truth slot of a batch of frames against the pose
//                table of the pose solver, each slot over its own class's mesh (TorchEval's eval_metric /
//                eval_metric_lm, pvn3d_eval_utils.py:113-137,204-220).  Both are the same two launches.
#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kMetThreads = 256;
constexpr int kMetTile = 2048;  // transformed mesh points per shared-memory tile (24 KB)
constexpr int kMetMaxPoints = 0x7fffffff / 3;  // mesh coordinates are indexed with int
__device__ __forceinline__ int ceil_div_dev(int a, int b) { return (a + b - 1) / b; }

// first maximal index, like torch.max(dim=-1) (ascending scan, strict '>'; NaN never wins)
__global__ void seg_argmax_kernel(const float *__restrict__ logits, long long rows, int n_cls,
                                  int *__restrict__ labels) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= rows) return;
  const float *row = logits + p * n_cls;
  float best = row[0];
  int bi = 0;
  for (int c = 1; c < n_cls; ++c) {
    const float v = row[c];
    if (v > best || (best != best && v == v)) {  // a leading NaN is replaced by the first number
      best = v;
      bi = c;
    }
  }
  labels[p] = bi;
}

__device__ __forceinline__ float3 rt_apply(const float *rt, float x, float y, float z) {
  // p @ R^T + t  (basic_utils.py:620-621): row-vector times transposed rotation = R p + t
  float3 o;
  o.x = __fmaf_rn(rt[2], z, __fmaf_rn(rt[1], y, rt[0] * x)) + rt[3];
  o.y = __fmaf_rn(rt[6], z, __fmaf_rn(rt[5], y, rt[4] * x)) + rt[7];
  o.z = __fmaf_rn(rt[10], z, __fmaf_rn(rt[9], y, rt[8] * x)) + rt[11];
  return o;
}

// Where each fit of add_adds_kernel takes its poses and its mesh from.  Pair form (cls_ids == NULL, one mesh):
// fit f scores pred[f] against gt[f] over mesh 0.  Frame form: fit f = (frame b, slot i) of a [B, slots] table
// scores poses[b, cls_ids[b,i]] -- or zeros / the identity when present[b, cls] == 0 -- against gt[f] over the mesh
// of that class.  A slot is scored only when no earlier slot of its frame holds class 0 and its class lies in
// [1, n_cls) (pvn3d_eval_utils.py:117-119); the rest are written as NaN.  Passed by value (__grid_constant__): the
// offsets are indexed straight out of the parameter bank.
struct FitTable {
  const float *pred;        // pair: [F,12]; frame: poses [B,n_cls,12]
  const float *gt;          // [F,12]
  const uint8_t *present;   // frame: [B,n_cls]
  const int *cls_ids;       // frame: [B,slots]; NULL selects the pair form
  const float *meshes;      // [off[n_mesh],3]
  int slots, n_cls, absent;
  int off[PVN3D_ADD_MAX_CLASSES + 1];
};

// mesh of fit f, or -1 when the slot is not scored
__device__ __forceinline__ int fit_mesh(const FitTable &tab, int f) {
  if (!tab.cls_ids) return 0;
  const int *ids = tab.cls_ids + static_cast<size_t>(f / tab.slots) * tab.slots;
  for (int j = 0; j < f % tab.slots; ++j)
    if (ids[j] == 0) return -1;                          // the `break` at the first class 0
  const int c = ids[f % tab.slots];
  return (c >= 1 && c < tab.n_cls) ? c : -1;
}

// grid (ceil(max P/256), F).  Thread i owns mesh point i under the GROUND-TRUTH pose; the mesh under the
// PREDICTED pose streams through shared memory.  partial[f][blk] = (sum_i |pd_i - gt_i|, sum_i min_j |pd_j - gt_i|).
// Blocks past the end of a fit's mesh (and every block of an unscored slot) write nothing.
__global__ void __launch_bounds__(kMetThreads) add_adds_kernel(const __grid_constant__ FitTable tab,
                                                               float2 *__restrict__ partial) {
  __shared__ float4 s_pd[kMetTile];
  __shared__ float s_rt[24];
  __shared__ float2 s_red[kMetThreads / 32];
  const int f = blockIdx.y, t = threadIdx.x;
  const int m = fit_mesh(tab, f);
  if (m < 0) return;
  const int p = tab.off[m + 1] - tab.off[m];
  if (static_cast<int>(blockIdx.x) * kMetThreads >= p) return;
  const float *__restrict__ p3ds = tab.meshes + static_cast<size_t>(tab.off[m]) * 3;
  if (t < 12) {
    float v;
    if (!tab.cls_ids) {
      v = tab.pred[f * 12 + t];
    } else {
      const size_t pc = static_cast<size_t>(f / tab.slots) * tab.n_cls + m;
      if (tab.present[pc]) v = tab.pred[pc * 12 + t];
      else v = (tab.absent == PVN3D_ADD_ABSENT_IDENTITY && t % 5 == 0) ? 1.f : 0.f;   // rows of [I | 0]
    }
    s_rt[t] = v;
  } else if (t < 24) {
    s_rt[t] = tab.gt[f * 12 + t - 12];
  }
  __syncthreads();
  const int i = blockIdx.x * kMetThreads + t;
  const bool live = i < p;
  float3 g = make_float3(0.f, 0.f, 0.f), own = g;
  if (live) {
    const float x = p3ds[i * 3 + 0], y = p3ds[i * 3 + 1], z = p3ds[i * 3 + 2];
    g = rt_apply(s_rt + 12, x, y, z);
    own = rt_apply(s_rt, x, y, z);
  }
  float best = __int_as_float(0x7f800000);
  for (int base = 0; base < p; base += kMetTile) {
    const int n = min(kMetTile, p - base);
    __syncthreads();
    for (int q = t; q < n; q += kMetThreads) {
      const float3 v = rt_apply(s_rt, p3ds[(base + q) * 3 + 0], p3ds[(base + q) * 3 + 1], p3ds[(base + q) * 3 + 2]);
      s_pd[q] = make_float4(v.x, v.y, v.z, 0.f);
    }
    __syncthreads();
#pragma unroll 8
    for (int j = 0; j < n; ++j) {
      const float4 v = s_pd[j];
      best = fminf(best, torch_sqnorm(v.x - g.x, v.y - g.y, v.z - g.z));
    }
  }
  float2 acc = make_float2(0.f, 0.f);
  if (live) {
    acc.x = __fsqrt_rn(torch_sqnorm(own.x - g.x, own.y - g.y, own.z - g.z));  // ADD term
    acc.y = __fsqrt_rn(best);                                                  // ADD-S term
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
    acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
  }
  if ((t & 31) == 0) s_red[t >> 5] = acc;
  __syncthreads();
  if (t == 0) {
    float2 s = s_red[0];
    for (int w = 1; w < kMetThreads / 32; ++w) { s.x += s_red[w].x; s.y += s_red[w].y; }
    partial[static_cast<size_t>(f) * gridDim.x + blockIdx.x] = s;
  }
}

// fixed-order sum of the per-block partials (bitwise reproducible) and the mean; NaN for an unscored slot.
// stride = the x extent of add_adds_kernel's grid.
__global__ void add_adds_finish_kernel(const __grid_constant__ FitTable tab, const float2 *__restrict__ partial,
                                       int stride, int nfit, float *__restrict__ add, float *__restrict__ adds) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nfit) return;
  const int m = fit_mesh(tab, f);
  if (m < 0) {
    if (add) add[f] = __int_as_float(0x7fc00000);
    if (adds) adds[f] = __int_as_float(0x7fc00000);
    return;
  }
  const int p = tab.off[m + 1] - tab.off[m];
  const int blocks = ceil_div_dev(p, kMetThreads);
  double sa = 0.0, ss = 0.0;
  for (int b = 0; b < blocks; ++b) {
    sa += partial[static_cast<size_t>(f) * stride + b].x;
    ss += partial[static_cast<size_t>(f) * stride + b].y;
  }
  if (add) add[f] = static_cast<float>(sa / p);
  if (adds) adds[f] = static_cast<float>(ss / p);
}

// both launches of one scoring call; tab.off[] is filled and checked by the caller
int launch_add_adds(const FitTable &tab, int nfit, int max_points, float *add, float *adds, float2 *partial,
                    cudaStream_t stream) {
  const int blocks = ceil_div(max_points, kMetThreads);
  add_adds_kernel<<<dim3(blocks, nfit), kMetThreads, 0, stream>>>(tab, partial);
  int rc = check_launch("add_adds_kernel");
  if (rc != PVN3D_OK) return rc;
  add_adds_finish_kernel<<<ceil_div(nfit, 64), 64, 0, stream>>>(tab, partial, blocks, nfit, add, adds);
  return check_launch("add_adds_finish_kernel");
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_seg_argmax(const float *logits, long long rows, int n_cls, int *labels,
                                pvn3d_stream_t stream) {
  if (!logits || !labels || rows < 0 || n_cls < 1) return PVN3D_ERR_INVALID_ARG;
  if (rows == 0) return PVN3D_OK;
  if (rows > 0x7fffffffll * 256) return PVN3D_ERR_UNSUPPORTED;
  seg_argmax_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, as_stream(stream)>>>(logits, rows, n_cls,
                                                                                             labels);
  return check_launch("seg_argmax_kernel");
}

static size_t add_adds_workspace(int n_fit, int max_points) {
  return static_cast<size_t>(n_fit > 0 ? n_fit : 1) * ceil_div(max_points > 0 ? max_points : 1, kMetThreads) *
             sizeof(float2) + 256;
}

extern "C" size_t pvn3d_pose_add_adds_workspace_bytes(int n_poses, int n_points) {
  if (n_poses < 0 || n_points < 0) return 0;
  return add_adds_workspace(n_poses, n_points);
}

extern "C" int pvn3d_pose_add_adds(const float *pred_rt, const float *gt_rt, int n_poses, const float *p3ds,
                                   int n_points, float *add, float *adds, void *workspace,
                                   size_t workspace_bytes, pvn3d_stream_t stream) {
  if (!pred_rt || !gt_rt || !p3ds || (!add && !adds) || !workspace || n_poses < 0 || n_points <= 0)
    return PVN3D_ERR_INVALID_ARG;
  if (n_poses == 0) return PVN3D_OK;
  if (n_poses > 65535 || n_points > kMetMaxPoints) return PVN3D_ERR_UNSUPPORTED;
  if (workspace_bytes < pvn3d_pose_add_adds_workspace_bytes(n_poses, n_points)) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 7u) return PVN3D_ERR_INVALID_ARG;
  FitTable tab{};
  tab.pred = pred_rt;
  tab.gt = gt_rt;
  tab.meshes = p3ds;
  tab.slots = 1;
  tab.n_cls = 1;
  tab.off[0] = 0;
  tab.off[1] = n_points;
  return launch_add_adds(tab, n_poses, n_points, add, adds, static_cast<float2 *>(workspace), as_stream(stream));
}

extern "C" size_t pvn3d_frame_add_adds_workspace_bytes(int b, int slots, int max_points) {
  if (b < 0 || slots < 0 || max_points < 0 || (slots > 0 && b > 65535 / slots)) return 0;
  return add_adds_workspace(b * slots, max_points);
}

extern "C" int pvn3d_frame_add_adds(const float *poses, const uint8_t *present, int n_cls, const float *gt_rt,
                                    const int *cls_ids, int b, int slots, const float *meshes, const int *mesh_off,
                                    int absent, float *add, float *adds, void *workspace, size_t workspace_bytes,
                                    pvn3d_stream_t stream) {
  if (!poses || !present || !gt_rt || !cls_ids || !meshes || !mesh_off || (!add && !adds) || !workspace || b < 0 ||
      slots < 0 || n_cls < 2 || (absent != PVN3D_ADD_ABSENT_ZEROS && absent != PVN3D_ADD_ABSENT_IDENTITY))
    return PVN3D_ERR_INVALID_ARG;
  if (n_cls > PVN3D_ADD_MAX_CLASSES) return PVN3D_ERR_UNSUPPORTED;
  FitTable tab{};
  int max_points = 0;
  if (mesh_off[0] != 0 || mesh_off[1] < 0) return PVN3D_ERR_INVALID_ARG;
  for (int c = 0; c <= n_cls; ++c) tab.off[c] = mesh_off[c];
  for (int c = 1; c < n_cls; ++c) {
    if (tab.off[c + 1] <= tab.off[c]) return PVN3D_ERR_INVALID_ARG;   // every scorable class needs a mesh
    if (tab.off[c + 1] - tab.off[c] > max_points) max_points = tab.off[c + 1] - tab.off[c];
  }
  if (tab.off[n_cls] > kMetMaxPoints) return PVN3D_ERR_UNSUPPORTED;
  if (b == 0 || slots == 0) return PVN3D_OK;
  if (b > 65535 / slots) return PVN3D_ERR_UNSUPPORTED;
  if (workspace_bytes < pvn3d_frame_add_adds_workspace_bytes(b, slots, max_points)) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 7u) return PVN3D_ERR_INVALID_ARG;
  tab.pred = poses;
  tab.gt = gt_rt;
  tab.present = present;
  tab.cls_ids = cls_ids;
  tab.meshes = meshes;
  tab.slots = slots;
  tab.n_cls = n_cls;
  tab.absent = absent;
  return launch_add_adds(tab, b * slots, max_points, add, adds, static_cast<float2 *>(workspace), as_stream(stream));
}
