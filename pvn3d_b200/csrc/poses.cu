// poses.cu -- cal_frame_poses / cal_frame_poses_lm and best_fit_transform for a batch of frames,
// entirely on device (reference pvn3d/lib/utils/pvn3d_eval_utils.py:37-110,156-201 and
// pvn3d/lib/utils/basic_utils.py:47-80).
//
// The reference walks classes and keypoints in Python, calling MeanShiftTorch.fit 1+1+8 times per
// object with >= 3 device->host syncs per class, then runs np.linalg.svd on the host.  Here the
// whole batch is a fixed sequence of launches with no host sync:
//   class compaction (stable, per frame) -> centre votes -> [YCB: mean-shift per class ->
//   nearest-centre relabel -> compaction] -> mean-shift per class (centre + inlier labels) ->
//   stable label compaction -> keypoint votes -> mean-shift per (class, keypoint) -> Kabsch.
// Ragged per-class point sets are (start,count) segments of flat float4 buffers.
#include <cmath>

#include "common.cuh"
#include "kabsch.cuh"

namespace pvn3d {

int meanshift_launch(const float4 *pts, const int *fit_start, const int *fit_count, int n_fits,
                     int cap, double bandwidth, int max_iter, unsigned flags, float4 *ctr,
                     uint8_t *labels, int *max_idx, int *n_in, unsigned char *ws, cudaStream_t st,
                     bool density_only);
size_t meanshift_ws_bytes(int cap, int n_fits, int max_iter);

namespace {

constexpr int kMaxCls = 64;
constexpr int kCompactThreads = 1024;

// ------------------------------------------------------------------------------------------------
// Stable compaction of one frame's points by class id (classes 1..n_cls-1; 0 = background).
//   perm[b][cls_off[b][c] .. cls_off[b][c+1])  = ascending point indices with mask == c
// == the order of pred_ctr[cls_msk, :] in the reference (boolean-mask indexing keeps index order).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCompactThreads)
class_compact_kernel(const int *__restrict__ mask, int n, int n_cls, int *__restrict__ perm,
                     int *__restrict__ cls_off /*[B][n_cls+1]*/, uint8_t *__restrict__ present) {
  __shared__ int s_hist[kMaxCls];
  __shared__ int s_base[kMaxCls];
  __shared__ int s_wcnt[kCompactThreads / 32][kMaxCls];
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = t & 31u, warp = t >> 5;
  mask += static_cast<size_t>(b) * n;
  perm += static_cast<size_t>(b) * n;
  cls_off += static_cast<size_t>(b) * (n_cls + 1);
  if (t < kMaxCls) s_hist[t] = 0;
  __syncthreads();
  for (int i = t; i < n; i += kCompactThreads) {
    const int c = mask[i];
    if (c > 0 && c < n_cls) atomicAdd(&s_hist[c], 1);
  }
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int c = 0; c < n_cls; ++c) {
      cls_off[c] = run;
      s_base[c] = run;
      run += (c > 0) ? s_hist[c] : 0;
    }
    cls_off[n_cls] = run;
  }
  if (present && t < n_cls) present[static_cast<size_t>(b) * n_cls + t] = (t > 0 && s_hist[t] > 0);
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += kCompactThreads) {
    const int i = i0 + t;
    int c = 0;
    if (i < n) {
      c = mask[i];
      if (c < 0 || c >= n_cls) c = 0;
    }
    for (int q = lane; q < n_cls; q += 32) s_wcnt[warp][q] = 0;
    __syncwarp();
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    const int rank = __popc(peers & lanemask_lt());
    if (c > 0 && rank == 0) s_wcnt[warp][c] = __popc(peers);
    __syncthreads();
    // class q: exclusive prefix of the per-warp counts, then advance the running base
    if (t < n_cls) {
      int run = s_base[t];
      for (int w = 0; w < kCompactThreads / 32; ++w) {
        const int v = s_wcnt[w][t];
        s_wcnt[w][t] = run;
        run += v;
      }
      s_base[t] = run;
    }
    __syncthreads();
    if (c > 0) perm[s_wcnt[warp][c] + rank] = i;
    __syncthreads();
  }
}

// fits of the centre stage: f = b*n_cls + c
__global__ void ctr_fit_desc_kernel(const int *__restrict__ cls_off, int b_n, int n, int n_cls,
                                    int *__restrict__ fit_start, int *__restrict__ fit_count) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b_n * n_cls) return;
  const int b = f / n_cls, c = f % n_cls;
  const int *off = cls_off + static_cast<size_t>(b) * (n_cls + 1);
  fit_start[f] = b * n + off[c];
  fit_count[f] = c > 0 ? off[c + 1] - off[c] : 0;
}

// votes = pcld - offset, in compacted order (pvn3d_eval_utils.py:41: pred_ctr = pcld - ctr_of[0])
__global__ void build_ctr_votes_kernel(const float *__restrict__ pcld, const float *__restrict__ ofs,
                                       const int *__restrict__ perm,
                                       const int *__restrict__ cls_off, int n, int n_cls,
                                       float4 *__restrict__ pts) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = cls_off[static_cast<size_t>(b) * (n_cls + 1) + n_cls];
  if (q >= total) return;
  const int i = perm[static_cast<size_t>(b) * n + q];
  const float *p = pcld + (static_cast<size_t>(b) * n + i) * 3;
  const float *o = ofs + (static_cast<size_t>(b) * n + i) * 3;
  pts[static_cast<size_t>(b) * n + q] = make_float4(p[0] - o[0], p[1] - o[1], p[2] - o[2], 0.f);
}

// centre-cluster filter (pvn3d_eval_utils.py:58-72): every foreground point moves to the class of
// its nearest cluster centre if that centre is closer than 0.8 * class radius.
__global__ void relabel_kernel(const float *__restrict__ pcld, const float *__restrict__ ctr_of,
                               const int *__restrict__ mask, const float4 *__restrict__ ctrs,
                               const int *__restrict__ cls_off, const float *__restrict__ cls_radius,
                               int n, int n_cls, int *__restrict__ new_mask) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t g = static_cast<size_t>(b) * n + i;
  const int mk = mask[g];
  int out = mk;
  if (mk > 0) {
    const float vx = pcld[g * 3 + 0] - ctr_of[g * 3 + 0];
    const float vy = pcld[g * 3 + 1] - ctr_of[g * 3 + 1];
    const float vz = pcld[g * 3 + 2] - ctr_of[g * 3 + 2];
    const int *off = cls_off + static_cast<size_t>(b) * (n_cls + 1);
    float best = __int_as_float(0x7f800000);
    int bc = 0;
    for (int c = 1; c < n_cls; ++c) {
      if (off[c + 1] - off[c] <= 0) continue;  // class not in np.unique(mask[mask>0])
      const float4 k = ctrs[static_cast<size_t>(b) * n_cls + c];
      // ctr_dis = torch.norm(pred_ctr - ctrs, dim=2); torch.min keeps the first minimum (:62-63)
      const float d = __fsqrt_rn(torch_sqnorm(vx - k.x, vy - k.y, vz - k.z));
      if (bc == 0 || d < best) {
        best = d;
        bc = c;
      }
    }
    if (bc > 0 && best < cls_radius[bc]) out = bc;  // min_dis < ycb_r_lst[cls-1]*0.8 (:69)
  }
  new_mask[g] = out;
}

// per frame: rank of every inlier among the inliers (compacted order), per-class selected counts,
// and the (start,count) of every keypoint fit  f = (b*n_cls + c)*K + k.
// Layout of the keypoint vote buffer (which follows the centre votes at row `base` of the same
// allocation, so that one mean-shift launch can take centre AND keypoint fits): frame b owns rows
// base + [b*K*N, (b+1)*K*N); inside, class c starts at K*S_c (S_c = inliers of lower classes) and
// holds K runs of n_sel_c votes.
__global__ void __launch_bounds__(kCompactThreads)
kp_layout_kernel(const uint8_t *__restrict__ labels /*[B*N] in compacted order, or NULL = all*/,
                 const int *__restrict__ cls_off, int n, int n_cls, int k_kp, int base,
                 int *__restrict__ sel_pos /*[B*N]*/, int *__restrict__ sel_base /*[B*n_cls]*/,
                 int *__restrict__ fit_start, int *__restrict__ fit_count) {
  __shared__ int s_warp[kCompactThreads / 32];
  __shared__ int s_run;
  __shared__ int s_at[kMaxCls + 1];  // exclusive scan value at each class boundary
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = t & 31u, warp = t >> 5;
  const int *off = cls_off + static_cast<size_t>(b) * (n_cls + 1);
  const int total = off[n_cls];
  if (t == 0) s_run = 0;
  __syncthreads();
  for (int q0 = 0; q0 < total; q0 += kCompactThreads) {
    const int q = q0 + t;
    const int v = (q < total) ? (labels ? (labels[static_cast<size_t>(b) * n + q] ? 1 : 0) : 1) : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int wsum = s_warp[lane];  // 32 warps
    int wincl = wsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, wincl, o);
      if (lane >= o) wincl += u;
    }
    const int wexcl = __shfl_sync(0xffffffffu, wincl - wsum, warp);
    const int chunk_total = __shfl_sync(0xffffffffu, wincl, 31);
    const int excl = s_run + wexcl + incl - v;
    if (q < total) sel_pos[static_cast<size_t>(b) * n + q] = v ? excl : -1;
    // class boundaries that fall on this element
    if (q < total)
      for (int c = 1; c <= n_cls; ++c)
        if (off[c] == q) s_at[c] = excl;
    __syncthreads();
    if (t == 0) s_run += chunk_total;
    __syncthreads();
  }
  // boundaries at `total` (end) and for empty trailing classes
  if (t == 0) {
    for (int c = 0; c <= n_cls; ++c)
      if (off[c] >= total) s_at[c] = s_run;
    s_at[0] = 0;
  }
  __syncthreads();
  for (int c = t; c < n_cls; c += kCompactThreads) {
    const int sc = s_at[c], nsel = (c > 0) ? s_at[c + 1] - s_at[c] : 0;
    sel_base[static_cast<size_t>(b) * n_cls + c] = sc;
    for (int k = 0; k < k_kp; ++k) {
      const size_t f = (static_cast<size_t>(b) * n_cls + c) * k_kp + k;
      fit_start[f] = base + b * k_kp * n + k_kp * sc + k * nsel;
      fit_count[f] = nsel;
    }
  }
}

// keypoint votes of the inliers: pred_kp = pcld - pred_kp_of (pvn3d_eval_utils.py:42,83,91-94)
__global__ void build_kp_votes_kernel(const float *__restrict__ pcld, const float *__restrict__ kp_of,
                                      const int *__restrict__ perm, const int *__restrict__ cmask,
                                      const int *__restrict__ cls_off,
                                      const int *__restrict__ sel_pos,
                                      const int *__restrict__ sel_base,
                                      const int *__restrict__ fit_start, int n, int n_cls, int k_kp,
                                      float4 *__restrict__ pts) {
  const int b = blockIdx.z, k = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = cls_off[static_cast<size_t>(b) * (n_cls + 1) + n_cls];
  if (q >= total) return;
  const int sp = sel_pos[static_cast<size_t>(b) * n + q];
  if (sp < 0) return;
  const int i = perm[static_cast<size_t>(b) * n + q];
  const int c = cmask[static_cast<size_t>(b) * n + i];
  const int rank = sp - sel_base[static_cast<size_t>(b) * n_cls + c];
  const size_t f = (static_cast<size_t>(b) * n_cls + c) * k_kp + k;
  const float *p = pcld + (static_cast<size_t>(b) * n + i) * 3;
  const float *o = kp_of + ((static_cast<size_t>(b) * k_kp + k) * n + i) * 3;
  pts[static_cast<size_t>(fit_start[f]) + rank] =
      make_float4(p[0] - o[0], p[1] - o[1], p[2] - o[2], 0.f);
}

// ------------------------------------------------------------------------------------------------
// Kabsch / best_fit_transform in float64 (basic_utils.py:47-80)
// ------------------------------------------------------------------------------------------------
// svd3_jacobi / det3: kabsch.cuh (shared with icp.cu)

// A (model) -> B (camera): rt[3][4]
__device__ void kabsch_fit(const float *a, const float *bq, int p, float *rt) {
  double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0};
  for (int i = 0; i < p; ++i)
    for (int d = 0; d < 3; ++d) {
      ca[d] += a[i * 3 + d];
      cb[d] += bq[i * 3 + d];
    }
  for (int d = 0; d < 3; ++d) {
    ca[d] /= p;
    cb[d] /= p;
  }
  double h[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int i = 0; i < p; ++i)
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        h[r][c] += (a[i * 3 + r] - ca[r]) * (bq[i * 3 + c] - cb[c]);  // H = AA^T BB
  double u[3][3], s[3], v[3][3], rot[3][3];
  svd3_jacobi(h, u, s, v);
  for (int pass = 0; pass < 2; ++pass) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double acc = 0;
        for (int k = 0; k < 3; ++k) acc += v[r][k] * u[c][k];  // R = Vt^T U^T = V U^T
        rot[r][c] = acc;
      }
    if (pass == 0 && det3(rot) < 0) {
      for (int r = 0; r < 3; ++r) v[r][2] = -v[r][2];  // Vt[m-1,:] *= -1
    } else {
      break;
    }
  }
  for (int r = 0; r < 3; ++r) {
    double tr = cb[r];
    for (int c = 0; c < 3; ++c) {
      rt[r * 4 + c] = static_cast<float>(rot[r][c]);
      tr -= rot[r][c] * ca[c];  // t = centroid_B - R centroid_A
    }
    rt[r * 4 + 3] = static_cast<float>(tr);
  }
}

__device__ __forceinline__ void write_identity(float *rt) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) rt[r * 4 + c] = (r == c) ? 1.f : 0.f;
}

constexpr int kMaxKabschPts = 32;

__global__ void best_fit_kernel(const float *__restrict__ a, const float *__restrict__ b,
                                const uint8_t *__restrict__ valid, int nfit, int p,
                                float *__restrict__ rt) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nfit) return;
  if (valid && !valid[f]) {
    write_identity(rt + static_cast<size_t>(f) * 12);
    return;
  }
  kabsch_fit(a + static_cast<size_t>(f) * p * 3, b + static_cast<size_t>(f) * p * 3, p,
             rt + static_cast<size_t>(f) * 12);
}

// one thread per (frame, class): gather the 8 voted keypoints + centre and fit the pose
__global__ void pose_kernel(const float4 *__restrict__ ctr2, const float4 *__restrict__ kp_ctr,
                            const int *__restrict__ cls_off2, const uint8_t *__restrict__ present,
                            const float *__restrict__ mesh_kps, int b_n, int n_cls, int k_kp,
                            float *__restrict__ poses, float *__restrict__ cls_kps) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= b_n * n_cls) return;
  const int b = f / n_cls, c = f % n_cls;
  const int *off = cls_off2 + static_cast<size_t>(b) * (n_cls + 1);
  const int cnt = c > 0 ? off[c + 1] - off[c] : 0;
  float kps[(kMaxKabschPts + 1) * 3];
  const int p = k_kp + 1;
  for (int k = 0; k < p * 3; ++k) kps[k] = 0.f;
  float *pose = poses + static_cast<size_t>(f) * 12;
  if (c == 0 || !present[f] || cnt < 1) {
    // absent class, or a class that lost every point in the filter pass: identity
    // (pvn3d_eval_utils.py:79-81)
    write_identity(pose);
  } else {
    for (int k = 0; k < k_kp; ++k) {
      const float4 v = kp_ctr[static_cast<size_t>(f) * k_kp + k];
      kps[k * 3 + 0] = v.x;
      kps[k * 3 + 1] = v.y;
      kps[k * 3 + 2] = v.z;
    }
    const float4 cc = ctr2[f];  // cls_kps[cls_id, n_kps, :] = ctr  (:88-89)
    kps[k_kp * 3 + 0] = cc.x;
    kps[k_kp * 3 + 1] = cc.y;
    kps[k_kp * 3 + 2] = cc.z;
    kabsch_fit(mesh_kps + static_cast<size_t>(c) * p * 3, kps, p, pose);
  }
  if (cls_kps)
    for (int k = 0; k < p * 3; ++k) cls_kps[static_cast<size_t>(f) * p * 3 + k] = kps[k];
}

struct PoseLayout {
  size_t perm, cls_off, perm2, cls_off2, new_mask, fs_ctr, fc_ctr, fs_kp, fc_kp, ctr1, ctr2, kp_ctr,
      mi, ni, labels, sel_pos, sel_base, pts_ctr, pts_kp, present, ms, total;
};
PoseLayout pose_layout(int b, int n, int k, int n_cls, int max_iter) {
  PoseLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t at = off;
    off = align_up(off + (bytes ? bytes : 1), 256);
    return at;
  };
  const size_t bn = static_cast<size_t>(b) * n, bc = static_cast<size_t>(b) * n_cls;
  L.perm = take(bn * 4);
  L.cls_off = take(static_cast<size_t>(b) * (n_cls + 1) * 4);
  L.perm2 = take(bn * 4);
  L.cls_off2 = take(static_cast<size_t>(b) * (n_cls + 1) * 4);
  L.new_mask = take(bn * 4);
  // fit tables / results hold the centre fits [0, bc) followed by the keypoint fits [bc, bc + bc*k)
  L.fs_ctr = take(bc * (k + 1) * 4);
  L.fc_ctr = take(bc * (k + 1) * 4);
  L.fs_kp = L.fs_ctr + bc * 4;
  L.fc_kp = L.fc_ctr + bc * 4;
  L.ctr1 = take(bc * 16);
  L.ctr2 = take(bc * (k + 1) * 16);
  L.kp_ctr = L.ctr2 + bc * 16;
  L.mi = take(bc * (k + 1) * 4);
  L.ni = take(bc * (k + 1) * 4);
  L.labels = take(bn);
  L.sel_pos = take(bn * 4);
  L.sel_base = take(bc * 4);
  // one vote buffer: centre votes [0, bn) then keypoint votes [bn, bn + bn*k)
  L.pts_ctr = take(bn * (k + 1) * 16);
  L.pts_kp = L.pts_ctr + bn * 16;
  L.present = take(bc);
  L.ms = take(meanshift_ws_bytes(static_cast<int>(bn * (k + 1)), static_cast<int>(bc * (k + 1)), max_iter));
  L.total = off;
  return L;
}

}  // namespace

// the stable per-frame class compaction above, for icp.cu's scene-point selection (n_cls <= 64)
int class_compact_launch(const int *mask, int b, int n, int n_cls, int *perm, int *cls_off,
                         uint8_t *present, cudaStream_t st) {
  class_compact_kernel<<<b, kCompactThreads, 0, st>>>(mask, n, n_cls, perm, cls_off, present);
  return check_launch("class_compact_kernel");
}

}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_best_fit_transform_batch(const float *a, const float *b, const uint8_t *valid,
                                              int nfit, int p, float *rt, pvn3d_stream_t stream) {
  if (!a || !b || !rt || nfit < 0 || p < 1) return PVN3D_ERR_INVALID_ARG;
  if (nfit == 0) return PVN3D_OK;
  best_fit_kernel<<<ceil_div(nfit, 64), 64, 0, as_stream(stream)>>>(a, b, valid, nfit, p, rt);
  return check_launch("best_fit_kernel");
}

extern "C" size_t pvn3d_frame_poses_workspace_bytes(int b, int n, int k, int n_cls, int max_iter) {
  if (b <= 0 || n <= 0 || k <= 0 || n_cls <= 0 || max_iter < 0 || max_iter > 4094) return 0;
  if (static_cast<long long>(b) * n * (k + 1) > 0x7fffffffll) return 0;
  return pose_layout(b, n, k, n_cls, max_iter).total;
}

extern "C" size_t pvn3d_frame_poses_ms_workspace_offset(int b, int n, int k, int n_cls, int max_iter) {
  if (b <= 0 || n <= 0 || k <= 0 || n_cls <= 0 || max_iter < 0 || max_iter > 4094) return 0;
  return pose_layout(b, n, k, n_cls, max_iter).ms;
}

extern "C" int pvn3d_frame_poses_batch(const float *pcld, const int *mask, const float *ctr_of,
                                       const float *kp_of, int b, int n, int k, int n_cls,
                                       const float *mesh_kps, const float *cls_radius,
                                       int use_ctr_clus_flter, double bandwidth, int max_iter,
                                       unsigned ms_flags, float *poses, uint8_t *present,
                                       float *cls_kps, int *new_mask, void *workspace,
                                       size_t workspace_bytes, pvn3d_stream_t stream) {
  if (!pcld || !mask || !ctr_of || !kp_of || !mesh_kps || !poses || !workspace || b < 0 || n <= 0 ||
      k <= 0 || n_cls < 2 || !(bandwidth > 0.0))
    return PVN3D_ERR_INVALID_ARG;
  if (use_ctr_clus_flter && !cls_radius) return PVN3D_ERR_INVALID_ARG;
  if (b == 0) return PVN3D_OK;
  if (n_cls > kMaxCls || k > kMaxKabschPts || b > 65535) return PVN3D_ERR_UNSUPPORTED;
  if (static_cast<long long>(b) * n * (k + 1) > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  if (max_iter < 0 || max_iter > 4094) return PVN3D_ERR_UNSUPPORTED;
  const PoseLayout L = pose_layout(b, n, k, n_cls, max_iter);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  cudaStream_t st = as_stream(stream);
  auto I = [&](size_t o) { return reinterpret_cast<int *>(ws + o); };
  auto F4 = [&](size_t o) { return reinterpret_cast<float4 *>(ws + o); };
  uint8_t *present_w = present ? present : reinterpret_cast<uint8_t *>(ws + L.present);
  int *nm = new_mask ? new_mask : I(L.new_mask);
  const int bc = b * n_cls;
  const dim3 gpts(ceil_div(n, 256), b);
  int rc;

  // pred_cls_ids = np.unique(mask[mask>0])  +  per-class index lists            (:50,53-54)
  class_compact_kernel<<<b, kCompactThreads, 0, st>>>(mask, n, n_cls, I(L.perm), I(L.cls_off),
                                                      present_w);
  if ((rc = check_launch("class_compact_kernel")) != PVN3D_OK) return rc;

  const int *perm_v = I(L.perm);
  const int *off_v = I(L.cls_off);
  const int *mask_v = mask;
  if (use_ctr_clus_flter) {
    ctr_fit_desc_kernel<<<ceil_div(bc, 128), 128, 0, st>>>(I(L.cls_off), b, n, n_cls, I(L.fs_ctr),
                                                          I(L.fc_ctr));
    if ((rc = check_launch("ctr_fit_desc_kernel")) != PVN3D_OK) return rc;
    build_ctr_votes_kernel<<<gpts, 256, 0, st>>>(pcld, ctr_of, I(L.perm), I(L.cls_off), n, n_cls,
                                                 F4(L.pts_ctr));
    if ((rc = check_launch("build_ctr_votes_kernel")) != PVN3D_OK) return rc;
    rc = meanshift_launch(F4(L.pts_ctr), I(L.fs_ctr), I(L.fc_ctr), bc, b * n, bandwidth, max_iter,
                          ms_flags, F4(L.ctr1), nullptr, I(L.mi), I(L.ni), ws + L.ms, st, false);
    if (rc != PVN3D_OK) return rc;
    relabel_kernel<<<gpts, 256, 0, st>>>(pcld, ctr_of, mask, F4(L.ctr1), I(L.cls_off), cls_radius,
                                         n, n_cls, nm);
    if ((rc = check_launch("relabel_kernel")) != PVN3D_OK) return rc;
    class_compact_kernel<<<b, kCompactThreads, 0, st>>>(nm, n, n_cls, I(L.perm2), I(L.cls_off2),
                                                        nullptr);
    if ((rc = check_launch("class_compact_kernel(2)")) != PVN3D_OK) return rc;
    perm_v = I(L.perm2);
    off_v = I(L.cls_off2);
    mask_v = nm;
  } else if (new_mask) {
    PVN3D_CUDA_TRY(cudaMemcpyAsync(new_mask, mask, sizeof(int) * static_cast<size_t>(b) * n,
                                   cudaMemcpyDeviceToDevice, st),
                   "new_mask copy");
  }

  // vote pass: centre + inlier labels per class                                   (:75-89)
  ctr_fit_desc_kernel<<<ceil_div(bc, 128), 128, 0, st>>>(off_v, b, n, n_cls, I(L.fs_ctr),
                                                        I(L.fc_ctr));
  if ((rc = check_launch("ctr_fit_desc_kernel(2)")) != PVN3D_OK) return rc;
  build_ctr_votes_kernel<<<gpts, 256, 0, st>>>(pcld, ctr_of, perm_v, off_v, n, n_cls,
                                               F4(L.pts_ctr));
  if ((rc = check_launch("build_ctr_votes_kernel(2)")) != PVN3D_OK) return rc;
  // exact pass of the centre fits only: the inlier labels depend on the INPUT votes alone
  // (meanshift_pytorch.py:46-50), so the keypoint vote sets can be formed before any iteration runs
  uint8_t *labels = reinterpret_cast<uint8_t *>(ws + L.labels);
  rc = meanshift_launch(F4(L.pts_ctr), I(L.fs_ctr), I(L.fc_ctr), bc, b * n, bandwidth, max_iter,
                        ms_flags, F4(L.ctr2), labels, I(L.mi), I(L.ni), ws + L.ms, st, true);
  if (rc != PVN3D_OK) return rc;

  // keypoint votes of the centre-cluster inliers, one fit per (class, keypoint)     (:91-97)
  kp_layout_kernel<<<b, kCompactThreads, 0, st>>>(use_ctr_clus_flter ? labels : nullptr, off_v, n,
                                                  n_cls, k, b * n, I(L.sel_pos), I(L.sel_base),
                                                  I(L.fs_kp), I(L.fc_kp));
  if ((rc = check_launch("kp_layout_kernel")) != PVN3D_OK) return rc;
  build_kp_votes_kernel<<<dim3(ceil_div(n, 256), k, b), 256, 0, st>>>(
      pcld, kp_of, perm_v, mask_v, off_v, I(L.sel_pos), I(L.sel_base), I(L.fs_kp), n, n_cls, k,
      F4(L.pts_ctr));
  if ((rc = check_launch("build_kp_votes_kernel")) != PVN3D_OK) return rc;
  // ONE mean-shift launch for the centre fit and the K keypoint fits of every class of every frame
  rc = meanshift_launch(F4(L.pts_ctr), I(L.fs_ctr), I(L.fc_ctr), bc * (k + 1), b * n * (k + 1),
                        bandwidth, max_iter, ms_flags, F4(L.ctr2), nullptr, I(L.mi), I(L.ni),
                        ws + L.ms, st, false);
  if (rc != PVN3D_OK) return rc;

  // least-squares pose per class                                                   (:99-107)
  pose_kernel<<<ceil_div(bc, 64), 64, 0, st>>>(F4(L.ctr2), F4(L.kp_ctr), off_v, present_w, mesh_kps,
                                               b, n_cls, k, poses, cls_kps);
  return check_launch("pose_kernel");
}
