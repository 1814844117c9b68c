/*
 * pvn3d_b200.h -- C ABI of libpvn3d_b200.so (hand-written sm_90a kernels).
 *
 * This is the drop-in boundary of the PVN3D per-frame keypoint-voting hot path:
 *   Boundary 1  the nine PointNet++ ops the reference exports from its pybind11 module
 *               `lib.pointnet2_utils._ext`  (reference: pvn3d/_ext-src/src/bindings.cpp:6-19,
 *               declarations pvn3d/_ext-src/include/{sampling,ball_query,group_points,interpolate}.h)
 *   Boundary 2  the post-network vote clustering + pose fit reached through
 *               MeanShiftTorch.fit          (pvn3d/lib/utils/meanshift_pytorch.py:18-51)
 *               cal_frame_poses[_lm]        (pvn3d/lib/utils/pvn3d_eval_utils.py:37-110,156-201)
 *               best_fit_transform          (pvn3d/lib/utils/basic_utils.py:47-80)
 *
 * Conventions
 *   - plain pointers + sizes; no torch / ATen types.  All pointers are DEVICE pointers on the
 *     current CUDA device unless the name ends in `_host`.
 *   - tensors are dense, row-major, float32 / int32, batch-major -- exactly the layouts the
 *     reference ops take (AT_CHECK contiguity, pvn3d/_ext-src/include/utils.h:5-25).
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it, never
 *     synchronises, keeps no global state and is re-entrant (reference: launches on
 *     at::cuda::getCurrentCUDAStream(), e.g. ball_query_gpu.cu:49).
 *   - outputs are fully written by the callee (the reference zero-fills them with torch::zeros
 *     first; rows the reference leaves at zero are written as zero here).
 *   - return value: 0 = PVN3D_OK, negative = error code (pvn3d_strerror()).  The library never
 *     calls exit() (the reference does: pvn3d/_ext-src/include/cuda_utils.h:30-39).
 */
#ifndef PVN3D_B200_H
#define PVN3D_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PVN3D_OK 0
#define PVN3D_ERR_INVALID_ARG (-1)   /* null pointer / negative or inconsistent size            */
#define PVN3D_ERR_UNSUPPORTED (-2)   /* size outside what the kernels are built for             */
#define PVN3D_ERR_CUDA (-3)          /* a CUDA runtime call / launch failed (cudaGetLastError)  */
#define PVN3D_ERR_WORKSPACE (-4)     /* caller-provided workspace too small                     */

typedef void *pvn3d_stream_t; /* cudaStream_t */

int pvn3d_version(void);                 /* ABI version, currently 1                         */
const char *pvn3d_strerror(int code);    /* static string                                    */
const char *pvn3d_last_cuda_error(void); /* thread-local text of the last PVN3D_ERR_CUDA     */
int pvn3d_device_sm_count(int *sm_count, int *cc_major, int *cc_minor);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
unsigned long long pvn3d_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Boundary 1: lib.pointnet2_utils._ext
 * ---------------------------------------------------------------------------------------- */

/* furthest_point_sampling(points[B,N,3], nsamples) -> idx[B,nsamples] int32
 * replaces sampling.h:6 / sampling.cpp:65-86 / sampling_gpu.cu:69-229.
 * Bit-exact with the reference, including its tie-break (512-thread strided ownership +
 * shared-memory tree whose ties go to the lower tree slot) and the |p|^2 <= 1e-3 skip rule.
 * No [B,N] scratch tensor is needed (running min-distances live in registers). */
int pvn3d_furthest_point_sampling(const float *xyz, int b, int n, int m, int *idx,
                                  pvn3d_stream_t stream);

/* gather_points(points[B,C,N], idx[B,M]) -> out[B,C,M]        (sampling.h:4, sampling_gpu.cu:8-30) */
int pvn3d_gather_points(const float *points, const int *idx, int b, int c, int n, int m,
                        float *out, pvn3d_stream_t stream);
/* new_xyz[B,M,3] = xyz[B, idx[B,M], :]: the point-major form of the reference's
 * gather_operation(xyz.transpose(1,2), idx).transpose(1,2) (pointnet2_modules.py:47-53), no transposes */
int pvn3d_gather_xyz(const float *xyz, const int *idx, int b, int n, int m, float *out, pvn3d_stream_t stream);
/* gather_points_grad(grad_out[B,C,M], idx[B,M], N) -> grad_points[B,C,N]  (sampling_gpu.cu:34-57);
 * grad_points is zero-filled by the callee, then scatter-added. */
int pvn3d_gather_points_grad(const float *grad_out, const int *idx, int b, int c, int n, int m,
                             float *grad_points, pvn3d_stream_t stream);

/* ball_query(new_xyz[B,M,3], xyz[B,N,3], radius, nsample) -> idx[B,M,nsample] int32
 * replaces ball_query.h:4-5 / ball_query_gpu.cu:9-54: first `nsample` indices in ascending
 * order with d2 < radius^2 (strict), first hit pre-fills the row, empty ball -> zeros.
 * d2 is evaluated as fma(dz,dz,fma(dx,dx,dy*dy)) like the reference SASS => bit-exact idx. */
int pvn3d_ball_query(const float *new_xyz, const float *xyz, int b, int n, int m, float radius,
                     int nsample, int *idx, pvn3d_stream_t stream);

/* group_points(points[B,C,N], idx[B,M,S]) -> out[B,C,M,S]       (group_points_gpu.cu:8-39) */
int pvn3d_group_points(const float *points, const int *idx, int b, int c, int n, int npoints,
                       int nsample, float *out, pvn3d_stream_t stream);
/* group_points_grad(grad_out[B,C,M,S], idx[B,M,S], N) -> grad_points[B,C,N]  (:43-75) */
int pvn3d_group_points_grad(const float *grad_out, const int *idx, int b, int c, int n,
                            int npoints, int nsample, float *grad_points, pvn3d_stream_t stream);

/* three_nn(unknown[B,n,3], known[B,m,3]) -> dist2[B,n,3] f32 (SQUARED), idx[B,n,3] i32
 * replaces interpolate.h:6 / interpolate_gpu.cu:9-68: ascending d2, strict '<' cascade
 * (first index wins ties); unused slots when m < 3 hold +inf / 0. */
int pvn3d_three_nn(const float *unknown, const float *known, int b, int n, int m, float *dist2,
                   int *idx, pvn3d_stream_t stream);

/* three_interpolate(points[B,C,M], idx[B,N,3], weight[B,N,3]) -> out[B,C,N]
 * (interpolate_gpu.cu:72-111); p1*w1 + p2*w2 + p3*w3 contracted as the reference SASS does
 * (t = p2*w2; t = fma(p1,w1,t); fma(p3,w3,t)) => bit-exact. */
int pvn3d_three_interpolate(const float *points, const int *idx, const float *weight, int b, int c,
                            int m, int n, float *out, pvn3d_stream_t stream);
/* three_interpolate_grad(grad_out[B,C,N], idx, weight, M) -> grad_points[B,C,M].
 * NOTE: implements the mathematically correct scatter of interpolate_gpu.cu:116-143; the
 * reference host wrapper launches the forward kernel by mistake (interpolate.cpp:89-93). */
int pvn3d_three_interpolate_grad(const float *grad_out, const int *idx, const float *weight, int b,
                                 int c, int n, int m, float *grad_points, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused forms of the same path (what QueryAndGroup.forward / PointnetFPModule.forward compose
 * from the ops above: pointnet2_utils.py:293-330, pointnet2_modules.py:183-190).
 * ---------------------------------------------------------------------------------------- */

/* channel-major [B,C,N] <-> point-major [B,N,C] (staging layout of the fused kernels) */
int pvn3d_transpose_cn_to_nc(const float *src_bcn, int b, int c, int n, float *dst_bnc,
                             pvn3d_stream_t stream);
int pvn3d_transpose_nc_to_cn(const float *src_bnc, int b, int n, int c, float *dst_bcn,
                             pvn3d_stream_t stream);

/* query_and_group: ball_query + group(xyz) - centre + group(features) + concat in ONE call (a scan
 * kernel that finds idx and a gather/transpose kernel that writes the grouped tensor; neither the
 * transposed cloud, nor the two grouped tensors, nor the concat copy of the reference exist).
 *   xyz[B,N,3], new_xyz[B,M,3], feat_pm[B,N,ldf] point-major rows whose first C columns are the
 *   descriptors (ldf >= C; C may be 0 -> feat_pm NULL)
 *   -> idx[B,M,S] (may be NULL), out[B,3+C,M,S]   == QueryAndGroup(radius,S,use_xyz=True).forward
 * idx bit-exact with pvn3d_ball_query; out bit-exact with the composed reference ops.
 * Supported: S <= 256 per scale (larger S: compose pvn3d_ball_query + pvn3d_group_points). */
int pvn3d_query_and_group(const float *xyz, const float *new_xyz, const float *feat_pm, int ldf,
                          int b, int n, int m, int c, float radius, int nsample, int *idx,
                          float *out, pvn3d_stream_t stream);

/* The two scales of one multi-scale-grouping level in ONE call (same centres, same cloud: every
 * squared distance is evaluated once and compared with both radii).  Per scale either output may be
 * NULL: out NULL = ball query only (idx), idx NULL = grouped tensor only. */
int pvn3d_query_and_group2(const float *xyz, const float *new_xyz, const float *feat_pm, int ldf,
                           int b, int n, int m, int c, float radius0, int nsample0, int *idx0,
                           float *out0, float radius1, int nsample1, int *idx1, float *out1,
                           pvn3d_stream_t stream);

/* three_nn + (1/(sqrt(d2)+1e-8) normalised) weights + three_interpolate, point-major features:
 *   unknown[B,n,3], known[B,m,3], known_feat_pm[B,m,C] -> out_pm[B,n,ldo] columns [col0,col0+C)
 *   (ldo >= col0+C lets the caller interpolate straight into the concat buffer of the FP module),
 *   optionally also dist2[B,n,3], idx[B,n,3] (NULL to skip).
 * Weights follow pointnet2_modules.py:184-186 in fp32 (sqrt.rn, div.rn). */
int pvn3d_three_nn_interpolate(const float *unknown, const float *known, const float *known_feat_pm,
                               int b, int n, int m, int c, float *out_pm, int ldo, int col0,
                               float *dist2, int *idx, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Shared-MLP layers of set abstraction / feature propagation on the Hopper tensor cores (wgmma)
 * (reference: SharedMLP = Conv2d 1x1 (no bias) + BatchNorm2d + ReLU, pytorch_utils.py:25-50, and the
 * max-pool over nsample of pointnet2_modules.py:64-67).  One call = one layer:
 *      out[p, col0 + 0:n_pad] = act( A[p, 0:k_pad] . W^T + bias ),   optionally max over `pool` rows
 *   w    [n_pad, k_pad] f32, BN folded into rows, values rounded to TF32, zero padded
 *        (k_pad multiple of 32, n_pad multiple of 16), 16-byte aligned (else PVN3D_ERR_INVALID_ARG: it is
 *        read 16 bytes at a time); bias [n_pad] (folded BN shift, 0 in the pad)
 *   out  point-major rows of length ldo (ldo, col0 multiples of 4); pool in {0, 8, 16, 32}
 * Arithmetic: TF32 operands (round-to-nearest), fp32 accumulation.
 * flags: PVN3D_MLP_RELU       apply ReLU (flags = 1 / 0 is the plain relu switch)
 *        PVN3D_MLP_ROUND_OUT  store the activations (pooled or not) already rounded to TF32
 *        PVN3D_MLP_A_TF32     (mlp_dense) `a` was produced with ROUND_OUT and is
 *                             16-byte aligned with a leading dimension % 4 == 0: its rows are copied global ->
 *                             shared asynchronously, without the rounding pass (unrounded values would be
 *                             TRUNCATED by the tensor core)
 * ---------------------------------------------------------------------------------------- */
#define PVN3D_MLP_RELU 1
#define PVN3D_MLP_ROUND_OUT 2
#define PVN3D_MLP_A_TF32 4
#define PVN3D_MLP_OUT_CN 16   /* pvn3d_mlp_fp_fact only: out is [b][n_pad][n_unknown] -- the channel-major [B, C, N] layout
                                 Pointnet2MSG.forward returns (pvn3d.py:154) -- written straight from the accumulator;
                                 n_pad 128 or 256, n_unknown % 32 == 0, ldo / col0 ignored (else PVN3D_ERR_UNSUPPORTED) */
/* leave n SMs (0..255) to kernels running concurrently on other streams: the persistent grid is
 * sm_count - n CTAs instead of one per SM (a persistent CTA that cannot be placed stalls its kernel) */
#define PVN3D_MLP_RESERVE_SMS(n) (((n) & 0xff) << 8)

/* A = point-major activations a[rows, lda]; columns >= a_cols read as zero. */
int pvn3d_mlp_dense(const float *a, int lda, int a_cols, long long rows, const float *w,
                    const float *bias, int k_pad, int n_pad, int flags, int pool, float *out, int ldo,
                    int col0, pvn3d_stream_t stream);
/* pvn3d_mlp_dense with ONE BIAS VECTOR PER BATCH ELEMENT: bias is [rows / rows_per_frame][n_pad] and row p uses
 * vector p / rows_per_frame (rows_per_frame % 128 == 0).  Lets a layer whose input contains a per-frame constant
 * (DenseFusion's broadcast global feature, pvn3d.py:178-182) drop those K columns: W_c . g_b is folded into the bias. */
int pvn3d_mlp_dense_frame_bias(const float *a, int lda, int a_cols, long long rows, int rows_per_frame,
                               const float *w, const float *bias, int k_pad, int n_pad, int flags, float *out,
                               int ldo, int col0, pvn3d_stream_t stream);
/* out[g, :] = sum over the 32 rows p in [32 g, 32 g + 32) of relu(a[p] . W^T + bias)  -- partial sums of a mean over
 * points (AvgPool1d of DenseFusion, pvn3d.py:165,178) without storing the per-point activations; out rows = ceil(rows/32).
 * Summation order is fixed (reproducible). */
int pvn3d_mlp_dense_sum32(const float *a, int lda, int a_cols, long long rows, const float *w, const float *bias,
                          int k_pad, int n_pad, int flags, float *out, int ldo, int col0, pvn3d_stream_t stream);
/* First layer of an FP module with three_interpolate + concat fused: row (b,j) =
 * [ sum_t nn_w[b,j,t] * known_feat_pm[b, nn_idx[b,j,t], 0:c2] | skip_pm[b, j, 0:c1] | 0.. ] */
int pvn3d_mlp_fp_first(const float *known_feat_pm, int c2, const int *nn_idx, const float *nn_w,
                       const float *skip_pm, int lds, int c1, int b, int n_unknown, int m_known,
                       const float *w, const float *bias, int k_pad, int n_pad, int flags, float *out,
                       int ldo, int col0, pvn3d_stream_t stream);
/* one folded layer: w [n_pad][k_pad] TF32-rounded, bias [n_pad] */
typedef struct {
  const float *w;
  const float *bias;
  int k_pad, n_pad;
} pvn3d_mlp_layer_t;
/* FACTORED first layer of an SA scale.  Conv1x1 + BN is linear before its ReLU, and QueryAndGroup's row is
 * [f_j | x_j - c_i] (pointnet2_utils.py:311-321), so  W1.[f_j | x_j - c_i] + b1 = U_j - V_i  with
 *   U_j = W1f.f_j + W1x.x_j   once per POINT    (pvn3d_sa_factor_table + pvn3d_mlp_dense without ReLU), and
 *   V_i = W1x.c_i - b1        once per CENTRE   (pvn3d_sa_centre_term),
 * instead of one GEMM row per (centre, neighbour) pair: 5-16x fewer rows.  The second layer then takes
 * relu(U[idx] - V) as its operand (pvn3d_mlp_sa_fact).  The table carries x as hi + lo TF32 parts (columns
 * [c_feat, c_feat+3) and [c_feat+3, c_feat+6)), to be multiplied by [W1f | W1x | W1x]: the coordinate term is
 * evaluated to ~2^-21, MORE accurately than rounding the difference x_j - c_i to TF32 as cuDNN's TF32 path
 * does.
 *   pvn3d_sa_factor_table: xyz [rows,3], feat_pm [rows, ldf] (c_feat columns) -> out [rows, k_pad] TF32-rounded
 *   pvn3d_sa_centre_term : centres [rows,3], wx [n_pad,3] (TF32-rounded), bias [n_pad] -> out [rows, n_pad]
 *   pvn3d_mlp_sa_fact    : u [B*n, ldu], v [B*m, ldu] (c_valid columns), idx [B,m,ns] -> layer (w, bias) as
 *                          pvn3d_mlp_dense: out rows = B*m*ns (or B*m with pool = ns) */
int pvn3d_sa_factor_table(const float *xyz, const float *feat_pm, int ldf, int c_feat, long long rows, int k_pad,
                          float *out, pvn3d_stream_t stream);
int pvn3d_sa_centre_term(const float *centres, const float *wx, const float *bias, long long rows, int n_pad,
                         float *out, pvn3d_stream_t stream);
int pvn3d_mlp_sa_fact(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m,
                      int ns, const float *w, const float *bias, int k_pad, int n_pad, int flags, int pool,
                      float *out, int ldo, int col0, pvn3d_stream_t stream);
/* Layers 2 AND 3 of a factored SA scale plus the max-pool over nsample, in one launch: the layer-2 activations
 * stay in shared memory instead of going through HBM.  Same result, bit for bit, as
 *   pvn3d_mlp_sa_fact(.., layer2, PVN3D_MLP_RELU | PVN3D_MLP_ROUND_OUT, pool = 0)  ->  h
 *   pvn3d_mlp_dense(h, .., layer3, PVN3D_MLP_RELU [| PVN3D_MLP_ROUND_OUT], pool = ns) -> out
 * pool must equal ns.  Both layers apply ReLU; flags: PVN3D_MLP_ROUND_OUT (pooled output) and
 * PVN3D_MLP_RESERVE_SMS(n).  layer3->k_pad >= layer2->n_pad.  Any number of layer-2 K chunks.
 * PVN3D_ERR_UNSUPPORTED (nothing launched) unless pvn3d_mlp_sa_fact2_supported(layer2, layer3, ns) is 1: ns 16 or 32,
 * both n_pad <= 128, and both weight matrices, the layer-2 tile and two operand stages fit in a block's shared memory.
 * The query is host-only and touches no device memory. */
int pvn3d_mlp_sa_fact2(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m,
                       int ns, const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int flags, int pool,
                       float *out, int ldo, int col0, pvn3d_stream_t stream);
int pvn3d_mlp_sa_fact2_supported(const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int ns);
/* The same for a WIDE last layer (layer3->n_pad > 128: SA3, SA4), where the weights cannot stay resident: 64-row
 * tiles, both layers in 128-column blocks, W2 and W3 streamed from L2 by TMA once per tile, the layer-2 activations
 * in shared memory.  Same arguments, same bit-identical result as the two launches above.
 * PVN3D_ERR_UNSUPPORTED (nothing launched) unless pvn3d_mlp_sa_fact2w_supported(layer2, layer3, ns) is 1: ns 16 or
 * 32, layer3->n_pad > 128, layer2->k_pad <= 256, layer3->k_pad within the 128-column blocks of layer 2, the A and H
 * tiles and three weight stages within a block's shared memory.
 * The query is host-only and touches no device memory. */
int pvn3d_mlp_sa_fact2w(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m,
                        int ns, const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int flags, int pool,
                        float *out, int ldo, int col0, pvn3d_stream_t stream);
int pvn3d_mlp_sa_fact2w_supported(const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int ns);
/* Both layers of an FP module with a two-layer MLP (FP2-FP4), in one launch: the interpolated first-layer operand is
 * produced once per pair of 128-column blocks instead of once per block, and the layer-1 activations stay in shared
 * memory instead of going through HBM.  Same result, bit for bit, as
 *   pvn3d_mlp_fp_first(.., layer1, PVN3D_MLP_RELU | PVN3D_MLP_ROUND_OUT) -> h [b*n_unknown, layer1->n_pad]
 *   pvn3d_mlp_dense(h, .., layer2, PVN3D_MLP_RELU [| PVN3D_MLP_ROUND_OUT] | PVN3D_MLP_A_TF32) -> out
 * Arguments as pvn3d_mlp_fp_first; out rows = b * n_unknown, columns col0 .. col0 + layer2->n_pad of rows ldo apart.
 * Both layers apply ReLU; flags: PVN3D_MLP_ROUND_OUT (output) and PVN3D_MLP_RESERVE_SMS(n).  Weight pointers must be
 * 16-byte aligned (else PVN3D_ERR_INVALID_ARG, before any CUDA call).
 * PVN3D_ERR_UNSUPPORTED (nothing launched) unless pvn3d_mlp_fp2_supported(layer1, layer2) is 1: layer1->n_pad 256 or
 * 512, layer2->k_pad == layer1->n_pad, layer2->n_pad a multiple of 128, and the layer-1 tile, three operand stages and
 * four weight stages within a block's shared memory.  The query is host-only and touches no device memory. */
int pvn3d_mlp_fp2(const float *known_feat_pm, int c2, const int *nn_idx, const float *nn_w, const float *skip_pm, int lds,
                  int c1, int b, int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2,
                  int flags, float *out, int ldo, int col0, pvn3d_stream_t stream);
int pvn3d_mlp_fp2_supported(const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2);
/* FACTORED first layer of an FP module: three_interpolate commutes with the (linear) first layer, so
 *   P = W1k . known      once per KNOWN point   (pvn3d_mlp_dense without ReLU on the known table),
 *   S = W1s . skip + b1  over the skip columns  (pvn3d_mlp_dense without ReLU on the skip table),
 * and the second layer takes relu(sum_t nn_w[b,j,t] * P[b, nn_idx[b,j,t], :] + S[b,j,:]) as its operand:
 * the gathered rows shrink from the known descriptors (256-1024 floats) to the layer width (128-512).
 *   p [B*m_known, ld], s [B*n_unknown, ld], ld == c_valid (multiple of 4) */
int pvn3d_mlp_fp_fact(const float *p, const float *s, int ld, int c_valid, const int *nn_idx, const float *nn_w,
                      int b, int n_unknown, int m_known, const float *w, const float *bias, int k_pad, int n_pad,
                      int flags, float *out, int ldo, int col0, pvn3d_stream_t stream);
/* The skip term and the second layer of a factored FP module whose skip is an SA factor table (FP1), in one launch:
 * S never goes through HBM.  Same result, bit for bit, as
 *   pvn3d_mlp_dense(table, k, k, b*n_unknown, layer_s, PVN3D_MLP_A_TF32) -> s    (k = layer_s->k_pad, no ReLU)
 *   pvn3d_mlp_fp_fact(p, s, 128, 128, nn_idx, nn_w, b, n_unknown, m_known, layer2,
 *                     PVN3D_MLP_RELU | PVN3D_MLP_OUT_CN) -> out [b][128][n_unknown]
 * for ANY n_unknown (a tile may hold the end of one frame and the start of the next).
 *   p [b*m_known, 128], table [b*n_unknown, 32] TF32-rounded (pvn3d_sa_factor_table), both 16-byte aligned.
 * flags: PVN3D_MLP_RESERVE_SMS(n) only.  Pointers not 16-byte aligned or other flags: PVN3D_ERR_INVALID_ARG, before any
 * CUDA call.  PVN3D_ERR_UNSUPPORTED (nothing launched) unless pvn3d_mlp_fp_fact2_supported(layer_s, layer2) is 1:
 * layer_s 32 -> 128 (k_pad 32, n_pad 128) and layer2 128 -> 128.  The query is host-only and touches no device memory. */
int pvn3d_mlp_fp_fact2(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b, int n_unknown,
                       int m_known, const pvn3d_mlp_layer_t *layer_s, const pvn3d_mlp_layer_t *layer2, int flags, float *out,
                       pvn3d_stream_t stream);
int pvn3d_mlp_fp_fact2_supported(const pvn3d_mlp_layer_t *layer_s, const pvn3d_mlp_layer_t *layer2);
/* pvn3d_mlp_fp_fact2 with the output POINT-MAJOR in a caller's row table: row r = f * n_unknown + i gets
 * tf32(relu(acc + b2)) in columns col0 .. col0 + 127 of rows ldo floats apart; other columns are not touched.  The same
 * bits as tf32(transpose(pvn3d_mlp_fp_fact2's [b][128][n_unknown])).  This is how PVN3D's network forward writes the
 * PointNet++ features straight into the DenseFusion activation table.  Arguments, flags and coverage as
 * pvn3d_mlp_fp_fact2; ldo and col0 multiples of 4, col0 >= 0, col0 + 128 <= ldo and out 16-byte aligned, else
 * PVN3D_ERR_INVALID_ARG before any CUDA call. */
int pvn3d_mlp_fp_fact2_rows(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b, int n_unknown,
                            int m_known, const pvn3d_mlp_layer_t *layer_s, const pvn3d_mlp_layer_t *layer2, int flags,
                            float *out, int ldo, int col0, pvn3d_stream_t stream);
/* The CNN embedding at the sampled pixels, point-major: PVN3D.forward's
 *   torch.gather(emb.view(B, C, H*W), 2, choose.repeat(1, C, 1))            (pvn3d.py:288-292)
 * written as out[f * n + p][col0 + ch] = tf32(emb[f][ch][choose[f][0][p]]) -- bit for bit the reference's gather,
 * transposed to rows and rounded to TF32 (cvt.rna) -- without the [B, C, N] int64 index the reference materialises.
 *   emb [b][c][hw] f32 (4-byte aligned), choose [b][1][n] int64 (8-byte aligned), out rows ldo floats apart (16-byte
 *   aligned; ldo, col0 multiples of 4, col0 + c <= ldo), c a multiple of 4.
 * An index outside [0, hw) writes a row of NaN (torch.gather raises instead; the library never aborts).
 * PVN3D_ERR_INVALID_ARG for null pointers, misalignment or a bad column range, PVN3D_ERR_UNSUPPORTED for b * n >= 2^31
 * or c > 256 -- both before any CUDA call. */
int pvn3d_gather_pixel_rows(const float *emb, int b, int c, long long hw, const long long *choose, int n, float *out,
                            int ldo, int col0, pvn3d_stream_t stream);
/* weight[p,0:3] = (1/(sqrt(dist2)+1e-8)) / sum  (pointnet2_modules.py:184-186), fp32 IEEE ops */
int pvn3d_three_nn_weights(const float *dist2, long long rows, float *weight, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Boundary 2: MeanShiftTorch.fit, cal_frame_poses / cal_frame_poses_lm, best_fit_transform
 * ---------------------------------------------------------------------------------------- */

/* Flags for the mean-shift iteration */
#define PVN3D_MS_STRICT 0u      /* the reference's global stop rule decides the iteration count T */
#define PVN3D_MS_EARLY_EXIT 1u  /* additionally stop a fit once the RETURNED seed is stationary    */
#define PVN3D_MS_NO_FREEZE 2u   /* validation: keep sweeping seeds that have stopped moving        */
#define PVN3D_MS_DEBUG_TIMING 4u /* phase time stamps in the head of the workspace                 */
/* PVN3D_MS_CERTIFIED (the default of the Python surface): the returned seed is iterated on its own
 * until it is stationary (iteration s); it0 <= s is the first iteration from which its remaining
 * path to C_s is shorter than 1e-5*bandwidth.  A fit is CERTIFIED when, for every iteration
 * it < it0, some witness seed (far-from-mode / low-density inputs, iterated alongside) still moves by
 * >= bandwidth*1e-3 -- then the reference's global stop rule cannot fire before it0 (T >= it0), and
 * the returned C_s is within 1e-5*bandwidth (+ the drift of a stationary seed) of the reference's
 * C_T.  ctr.w reports it0 (a lower bound of the reference's T).  Fits that cannot be certified fall
 * back to PVN3D_MS_EARLY_EXIT over all seeds, which applies the reference's rule exactly. */
#define PVN3D_MS_CERTIFIED 8u
/* validation: count the inliers of every input point by the brute-force n^2 pass instead of the pruned one
 * (radial sort + triangle inequality; both are exact and must agree bit for bit) */
#define PVN3D_MS_BRUTE_DENSITY 16u

/* A batch of F independent MeanShiftTorch(bandwidth, max_iter).fit(A_f) problems.
 *   pts        [cap,4] f32  vote clouds (x,y,z,unused); fit f owns rows
 *                           [fit_start[f], fit_start[f]+fit_count[f])  (segments may have gaps)
 *   fit_start  [F] i32, fit_count [F] i32   (device; count 0 = empty fit: outputs zeroed)
 *   n_fits     F
 *   cap        number of float4 rows addressable in pts / labels / workspace
 *   bandwidth  double, as the Python float the reference holds: the fp32 thresholds
 *              float(bandwidth) and float(bandwidth*1e-3) are derived from it exactly as torch
 *              does when a float32 tensor is compared with a Python scalar.
 * outputs
 *   ctr      [F,4]  f32   C[max_idx] (x,y,z) and the iteration count as float in .w
 *   labels   [cap]   u8   1 where |A[max_idx]-A_j| < bandwidth, indexed like pts (NULL to skip)
 *   max_idx  [F]    i32   first index (within the fit) of the densest input point
 *   n_in     [F]    i32   its inlier count
 * workspace: pvn3d_meanshift_workspace_bytes(cap, n_fits, max_iter) bytes, 256-B aligned
 *            (max_iter <= 4094).
 * Semantics follow meanshift_pytorch.py:24-51 (stop when max_i |dC_i| < bandwidth*1e-3 or
 * it > max_iter; densest *input* point selects the returned seed; first-index arg-max). */
size_t pvn3d_meanshift_workspace_bytes(int cap, int n_fits, int max_iter);
/* byte offset, inside a pvn3d_meanshift_fit_batch workspace, of the int32 inlier count of every input point
 * (indexed like pts) left by the exact pass of the last launch -- test / diagnostics access */
size_t pvn3d_meanshift_workspace_counts_offset(int cap, int n_fits, int max_iter);
int pvn3d_meanshift_fit_batch(const float *pts, const int *fit_start, const int *fit_count,
                              int n_fits, int cap, double bandwidth, int max_iter, unsigned flags,
                              float *ctr, uint8_t *labels, int *max_idx, int *n_in,
                              void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* best_fit_transform(A[P,3], B[P,3]) for a batch: least-squares rigid fit A -> B (Kabsch, SVD
 * with reflection fix), basic_utils.py:47-80.  valid[i]==0 -> identity(3x4) (reference:
 * pvn3d_eval_utils.py:79-81).  Computation in float64 on device from float32 inputs.
 *   a[nfit,P,3], b[nfit,P,3], valid[nfit] (NULL = all valid) -> rt[nfit,3,4] f32 */
int pvn3d_best_fit_transform_batch(const float *a, const float *b, const uint8_t *valid, int nfit,
                                   int p, float *rt, pvn3d_stream_t stream);

/* cal_frame_poses / cal_frame_poses_lm for a batch of frames, fully on device, no host sync.
 *   pcld   [B,N,3] f32, mask [B,N] i32 (class id per point, 0 = background),
 *   ctr_of [B,N,3] f32 (reference ctr_of[0]), kp_of [B,K,N,3] f32
 *   mesh_kps [n_cls,K+1,3] f32  object-frame keypoints, centre LAST (pvn3d_eval_utils.py:99-103);
 *            row 0 unused.  LineMOD: n_cls=2 and row 1 = fixtures of obj_id.
 *   cls_radius [n_cls] f32   float32(r*0.8) thresholds of the centre-cluster filter
 *            (pvn3d_eval_utils.py:69), row 0 unused; NULL when use_ctr_clus_flter==0.
 * outputs
 *   poses    [B,n_cls,3,4] f32   identity for classes that are absent or lost all points
 *   present  [B,n_cls] u8        1 where the class id was in np.unique(mask[mask>0])  (:50)
 *   cls_kps  [B,n_cls,K+1,3] f32 voted keypoints + centre (NULL to skip)
 *   new_mask [B,N] i32           relabelled mask of the filter pass (NULL to skip)        (:66-72)
 * use_ctr must be 1 (the reference's use_ctr=False branch is never exercised: SURVEY App. A.5). */
size_t pvn3d_frame_poses_workspace_bytes(int b, int n, int k, int n_cls, int max_iter);
/* byte offset, inside that workspace, of the mean-shift workspace of the LAST launch (all centre +
 * keypoint fits); int32 word PVN3D_MS_STAT_CERTIFIED of it counts the fits PVN3D_MS_CERTIFIED closed
 * without sweeping all seeds (diagnostics for bench.py; same word at the head of a
 * pvn3d_meanshift_fit_batch workspace). */
#define PVN3D_MS_STAT_CERTIFIED 8
size_t pvn3d_frame_poses_ms_workspace_offset(int b, int n, int k, int n_cls, int max_iter);
int pvn3d_frame_poses_batch(const float *pcld, const int *mask, const float *ctr_of,
                            const float *kp_of, int b, int n, int k, int n_cls,
                            const float *mesh_kps, const float *cls_radius, int use_ctr_clus_flter,
                            double bandwidth, int max_iter, unsigned ms_flags, float *poses,
                            uint8_t *present, float *cls_kps, int *new_mask, void *workspace,
                            size_t workspace_bytes, pvn3d_stream_t stream);

/* ICP pose refinement: my_icp(A, B, init_pose, max_iterations, tolerance) of the reference
 * (lib/utils/icp/icp.py:141-192) as pvn3d/eval_icp.py:94-185 applies it per object, in float64.
 *
 * Model set: object-frame points of n_models models, pts [total_pts,3] f32, model m owning rows
 * [model_off[m], model_off[m+1]) (model_off [n_models+1] i32, device; an empty range = no model).
 * pvn3d_icp_build_models builds, on device, the exact nearest-neighbour structure every fit
 * searches into `buf` (pvn3d_icp_models_bytes(n_models, total_pts) bytes, 256-B aligned).  Its
 * layout is private to the library; `pts` may be freed once the build has run.
 *
 * Fit semantics, per fit with scene set B [n,3] and init pose P_0 (3x4, rigid):
 *   for i in 0..max_iter-1: d_j, idx_j = nearest model point of every scene point under P_i
 *     (exact: equal to a float64 brute-force scan, lowest model index on exact ties);
 *     P_{i+1} = Kabsch(A[idx], B) (float64, reflection-fixed);
 *     stop when |prev - mean(d)| < tol, prev starting at 0.
 *   result: P_{i+1}, the distances d of iteration i, and i (max_iter-1 when it never stopped).
 * The per-iteration sums run in a fixed order: results are reproducible bit for bit.
 * The first 8 bytes of the workspace count (u64) the model points the call's searches tested. */
size_t pvn3d_icp_models_bytes(int n_models, int total_pts);
int pvn3d_icp_build_models(const float *pts, const int *model_off, int n_models, int total_pts,
                           void *buf, size_t bytes, pvn3d_stream_t stream);
/* workspace of pvn3d_icp_refine_batch(b, n, n_cls, max_pts); (1, n, 1, n) also sizes pvn3d_icp_fit */
size_t pvn3d_icp_workspace_bytes(int b, int n, int n_cls, int max_pts);
/* One fit per (frame b, class c), c in 1..n_cls-1, model c of the set (n_cls <= 64):
 *   pcld [B,N,3] f32, mask [B,N] i32 (class per point), init_poses [B,n_cls,3,4] f32 (promoted to
 *   f64), present [B,n_cls] u8 -- the outputs of pvn3d_frame_poses_batch.
 *   Scene set: the class's points in ascending index; with cnt > max_pts of them, the points at
 *   positions floor(j*cnt/max_pts), j < max_pts.  Skipped (pose = init, iters = 0, err = 0,
 *   refined = 0): c == 0, present == 0, cnt < min_pts, cnt == 0, or no model for c.
 * outputs: poses_out [B,n_cls,3,4] f64, iters_out [B,n_cls] i32 (the loop index i),
 *   err_out [B,n_cls] f64 (mean of the last iteration's distances), refined_out [B,n_cls] u8.
 * max_iter >= 1, tol >= 0. */
int pvn3d_icp_refine_batch(const void *models, const float *pcld, const int *mask, int b, int n,
                           int n_cls, const float *init_poses, const uint8_t *present, int max_pts,
                           int min_pts, int max_iter, double tol, double *poses_out, int *iters_out,
                           double *err_out, uint8_t *refined_out, void *workspace,
                           size_t workspace_bytes, pvn3d_stream_t stream);
/* One fit of an explicit scene set scene [n,3] f32 against model `model`, init_pose [3,4] f64
 * (same kernel as the batch): pose_out [3,4] f64, dist_out [n] f64 (NULL to skip), iter_out [1]
 * i32, err_out [1] f64.  A missing or empty model leaves pose = init and iter = -1. */
int pvn3d_icp_fit(const void *models, int model, const float *scene, int n, const double *init_pose,
                  int max_iter, double tol, double *pose_out, double *dist_out, int *iter_out,
                  double *err_out, void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* Flat-kernel mean shift: sklearn's MeanShift(bandwidth, bin_seeding=True).fit(X) with min_bin_freq=1
 * and cluster_all=True, as pvn3d/eval_icp.py:56-64 (get_cld_bigest_clus) runs it on float64 points.
 * One CTA per fit; at most PVN3D_FLAT_MS_MAX_PTS points per fit.
 *   1. bin keys rint(x / bw) per coordinate (float64 division, round-half-even), bins in order of first
 *      occurrence, seed = float32(key) * float32(bw) in float32; the points themselves when every point
 *      has its own bin.
 *   2. per seed: members d2 <= bw*bw, d2 = (dx*dx + dy*dy) + dz*dz without FMA; no member -> the seed
 *      is dropped; mean = float64 sum of the members in ascending index order / count; stop when
 *      sqrt((ddx*ddx + ddy*ddy) + ddz*ddz) <= 1e-3*bw or after max_iter completed iterations.
 *   3. equal centres (==) collapse into the first seed's centre with the last seed's count.
 *   4. order by (count, x, y, z) descending; 5. a kept centre removes every later one with
 *      d2 <= bw*bw; 6. label = nearest kept centre by the same d2, the lower index on ties.
 * Results are bit-identical run to run.  (sklearn itself sums the members in its neighbour search's
 * order, so it agrees to rounding.) */
#define PVN3D_FLAT_MS_MAX_PTS 4096
/* Fit f clusters X [fit_off[f], fit_off[f+1]) (X [total,3] f64, fit_off [n_fits+1] i32, device).
 *   max_fit_pts  an upper bound on every fit's point count (sizes shared memory): above
 *                PVN3D_FLAT_MS_MAX_PTS the call returns PVN3D_ERR_UNSUPPORTED and launches nothing;
 *                a fit larger than it is not clustered (labels -1, n_clusters -1).
 * outputs, rows indexed like X: labels_out [total] i32; centres_out [total,3] f64 (fit f's K kept
 *   centres at rows fit_off[f]..fit_off[f]+K-1, the rest untouched); counts_out [total] i32 (their
 *   member counts; NULL to skip); per fit n_clusters_out [n_fits] i32 (K; 0 when no seed had a member,
 *   labels then -1) and n_iter_out [n_fits] i32 (max completed iterations over the seeds).
 * bandwidth > 0, max_iter >= 0. */
int pvn3d_flat_ms_fit_batch(const double *X, const int *fit_off, int n_fits, int max_fit_pts,
                            double bandwidth, int max_iter, int *labels_out, double *centres_out,
                            int *counts_out, int *n_clusters_out, int *n_iter_out, pvn3d_stream_t stream);
/* pvn3d_icp_refine_batch with eval_icp's pre-filter: each fit's scene set (the strided selection, after
 * the skip rules) is clustered as above with cluster_bw / cluster_max_iter, and the fit uses only the
 * points labelled 0, in ascending order.  cluster_pts_out [B,n_cls] i32: points the fit used (0 when
 * skipped; a fit whose filter keeps nothing is skipped).  max_pts <= PVN3D_FLAT_MS_MAX_PTS.
 * Workspace: pvn3d_icp_clustered_workspace_bytes(b, n, n_cls, max_pts) (0 when unsupported).  From byte
 * pvn3d_icp_workspace_bytes(b, n, n_cls, max_pts) of it, int32 [B,N]: in row b, fit (b, c)'s
 * cluster_pts_out[b,c] frame point indices (into pcld[b]) that the fit used, ascending, start at position
 * (number of points of frame b with class id in 1..c-1). */
size_t pvn3d_icp_clustered_workspace_bytes(int b, int n, int n_cls, int max_pts);
int pvn3d_icp_refine_batch_clustered(const void *models, const float *pcld, const int *mask, int b, int n,
                                     int n_cls, const float *init_poses, const uint8_t *present,
                                     int max_pts, int min_pts, int max_iter, double tol, double cluster_bw,
                                     int cluster_max_iter, double *poses_out, int *iters_out,
                                     double *err_out, uint8_t *refined_out, int *cluster_pts_out,
                                     void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* The full-resolution scene of eval_icp's refinement (pvn3d/eval_icp.py:224-291, 388-422).
 *
 * pvn3d_depth_to_cloud: Basic_Utils.dpt_2_cld (lib/utils/basic_utils.py:381-399) for every pixel, in
 * raster order.  depth [B,H,W] f32, K [B,3,3] f32 (per frame), cam_scale [B] f32 ->
 * cloud [B,H*W,3] f32, valid [B,H*W] u8.  A pixel is valid when dpt > 1e-6; then, one float32
 * operation per step, pt2 = dpt / cam_scale, pt0 = ((col - cx) * pt2) / fx,
 * pt1 = ((row - cy) * pt2) / fy.  An invalid pixel gets (0, 0, 0) and valid = 0.
 * B*H*W < 2^31, else PVN3D_ERR_UNSUPPORTED (nothing launched). */
int pvn3d_depth_to_cloud(const float *depth, const float *K, const float *cam_scale, int b, int h, int w,
                         float *cloud, uint8_t *valid, pvn3d_stream_t stream);
/* pvn3d_label_fill: eval_icp's fill_label_item.  Every valid pixel of cloud [B,hw,3] / valid [B,hw]
 * takes point_labels[b, j] of the sampled point j of pcld [B,N,3] f32 nearest to it: float64 squared
 * distance (dx*dx + dy*dy) + dz*dz without FMA, lowest j on exact ties.  labels_out [B,hw] i32;
 * nn_idx_out [B,hw] i32 (j; NULL to skip).  Invalid pixels get label 0 and index -1.
 * Each call builds the search grid of every frame's pcld into the workspace
 * (pvn3d_label_fill_workspace_bytes(b, n), 256-B aligned; 0 = unsupported) on the stream.
 * B*hw < 2^31, B*N < 2^31 and B <= 65535, else PVN3D_ERR_UNSUPPORTED (nothing launched). */
size_t pvn3d_label_fill_workspace_bytes(int b, int n);
int pvn3d_label_fill(const float *cloud, const uint8_t *valid, int hw, const float *pcld, const int *point_labels,
                     int b, int n, int *labels_out, int *nn_idx_out, void *workspace, size_t workspace_bytes,
                     pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Callers either side of the path (SURVEY section 8 f4)
 * ---------------------------------------------------------------------------------------- */

/* labels[p] = argmax_c logits[p, c] -- `_, classes_rgbd = torch.max(pred_rgbd_seg, -1)` (demo.py:108):
 * first maximal index; the int32 output is the `mask` pvn3d_frame_poses_batch takes.
 *   logits [rows, n_cls] f32 -> labels [rows] i32 */
int pvn3d_seg_argmax(const float *logits, long long rows, int n_cls, int *labels, pvn3d_stream_t stream);

/* ADD and ADD-S of n_poses (predicted, ground-truth) pose pairs over one mesh: Basic_Utils.cal_add_cuda /
 * cal_adds_cuda (basic_utils.py:617-635).
 *   pred_rt, gt_rt [n_poses,3,4] f32, p3ds [n_points,3] f32 (object frame)
 *   add[i]  = mean_k | (R_p x_k + t_p) - (R_g x_k + t_g) |
 *   adds[i] = mean_k min_j | (R_p x_j + t_p) - (R_g x_k + t_g) |          (either output may be NULL)
 * fp32 with fused multiply-adds; the per-block sums are combined in a fixed order (reproducible). */
size_t pvn3d_pose_add_adds_workspace_bytes(int n_poses, int n_points);
int pvn3d_pose_add_adds(const float *pred_rt, const float *gt_rt, int n_poses, const float *p3ds,
                        int n_points, float *add, float *adds, void *workspace, size_t workspace_bytes,
                        pvn3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PVN3D_B200_H */
