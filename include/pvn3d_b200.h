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

int pvn3d_version(void);                 /* ABI version, currently 2                         */
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
 * grad_points is zero-filled by the callee, then scatter-added.
 * Precision of the three *_grad entry points: fp32 atomic scatter-adds, so the summation order is unspecified and
 * results are not bit-reproducible from run to run.  Each element is within gamma_k * sum|t| of the exact sum of its
 * k contributions t (gamma_k = k u / (1 - k u), u = 2^-24; three_interpolate_grad's t = g * w, its product rounding
 * included); k = 0 gives +0.0 and k = 1 gives fl32(t).  Integer-valued inputs (and dyadic weights) whose partial sums
 * stay below 2^24 are exact.  An input with no elements may be null. */
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
/* group_points_grad(grad_out[B,C,M,S], idx[B,M,S], N) -> grad_points[B,C,N]  (:43-75)
 * Zero-filled, then scatter-added; precision as gather_points_grad above. */
int pvn3d_group_points_grad(const float *grad_out, const int *idx, int b, int c, int n,
                            int npoints, int nsample, float *grad_points, pvn3d_stream_t stream);

/* three_nn(unknown[B,n,3], known[B,m,3]) -> dist2[B,n,3] f32 (SQUARED), idx[B,n,3] i32
 * replaces interpolate.h:6 / interpolate_gpu.cu:9-68: ascending d2, strict '<' cascade
 * (first index wins ties); unused slots when m < 3 hold +inf / 0. */
int pvn3d_three_nn(const float *unknown, const float *known, int b, int n, int m, float *dist2,
                   int *idx, pvn3d_stream_t stream);
/* three_nn and the inverse-distance weights of pvn3d_three_nn_weights for nlev <= 4 levels of one batch in one call:
 * level l is unknown[l][B,n[l],3] against known[l][B,m[l],3] -> dist2[l], idx[l] (as pvn3d_three_nn) and weight[l]
 * [B,n[l],3] (as pvn3d_three_nn_weights), bit for bit.  The levels pvn3d_three_nn_grid_supported takes are searched on
 * per-frame cell grids of their known points: one launch builds every grid, one searches every level and writes the
 * weights.  Other levels run pvn3d_three_nn and pvn3d_three_nn_weights.  The pointer arrays are host memory; no host
 * sync, scratch from the stream-ordered pool. */
int pvn3d_three_nn_grid_supported(int n, int m);
int pvn3d_three_nn_weights_levels(int nlev, const float *const *unknown, const float *const *known, const int *n,
                                  const int *m, int b, float *const *dist2, int *const *idx, float *const *weight,
                                  pvn3d_stream_t stream);
/* ball query of both radii of nlev <= 4 MSG levels of one batch in one call: level l searches xyz[l][B,n[l],3] around
 * new_xyz[l][B,m[l],3] -> idx0[l][B,m[l],ns0[l]] (radius0[l]) and idx1[l][B,m[l],ns1[l]] (radius1[l]), the same values
 * as pvn3d_query_and_group2 (first ns in index order, padded with the first hit, zeros for an empty ball).  The levels
 * pvn3d_ball_grid_supported takes are binned into per-frame cell grids no finer than the larger radius (one launch
 * for every grid) and searched a warp per centre (one launch); a centre with more hits than the warp buffers scans the
 * whole cloud in index order.  Other levels run pvn3d_query_and_group2.  The arrays are host memory; no host sync,
 * scratch from the stream-ordered pool. */
int pvn3d_ball_grid_supported(int n, int m, int ns0, int ns1);
int pvn3d_ball_query2_levels(int nlev, const float *const *xyz, const float *const *new_xyz, const int *n, const int *m,
                             int b, const float *radius0, const int *ns0, int *const *idx0, const float *radius1,
                             const int *ns1, int *const *idx1, pvn3d_stream_t stream);

/* three_interpolate(points[B,C,M], idx[B,N,3], weight[B,N,3]) -> out[B,C,N]
 * (interpolate_gpu.cu:72-111); p1*w1 + p2*w2 + p3*w3 contracted as the reference SASS does
 * (t = p2*w2; t = fma(p1,w1,t); fma(p3,w3,t)) => bit-exact. */
int pvn3d_three_interpolate(const float *points, const int *idx, const float *weight, int b, int c,
                            int m, int n, float *out, pvn3d_stream_t stream);
/* three_interpolate_grad(grad_out[B,C,N], idx, weight, M) -> grad_points[B,C,M].
 * NOTE: implements the mathematically correct scatter of interpolate_gpu.cu:116-143; the
 * reference host wrapper launches the forward kernel by mistake (interpolate.cpp:89-93).
 * Zero-filled, then scatter-added; precision as gather_points_grad above. */
int pvn3d_three_interpolate_grad(const float *grad_out, const int *idx, const float *weight, int b,
                                 int c, int n, int m, float *grad_points, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * 16-bit forms of group_points, three_interpolate and their grads, for training under torch.autocast (bf16 or fp16
 * features; coordinates, idx and weight stay f32 / int32).  `dtype` is PVN3D_F16 (IEEE binary16, torch.float16) or
 * PVN3D_BF16 (bfloat16, torch.bfloat16); any other code returns PVN3D_ERR_INVALID_ARG before any CUDA call.  The
 * 16-bit pointers hold elements of that type.  Arithmetic is float32; each output element is rounded once, to nearest
 * even; inf and NaN propagate, and a float32 result beyond float16's largest finite value (65504) rounds to inf.
 * Argument checks, empty shapes and the batch limit as the float32 entry points.
 *   group_points_16: a copy, bit-equal to torch.gather of the same elements.  Two adjacent slots per 4-byte store when
 *     the slot count is even (idx 8-byte and out 4-byte aligned).
 *   three_interpolate_16: weight is float32; out[b,c,j] = round16(the float32 value pvn3d_three_interpolate gives for
 *     the widened features), the same fma(p3,w3, fma(p1,w1, p2*w2)) order.
 *   *_grad_16 (atomic): float32 atomics into `scratch`, b*c*n (group) or b*c*m (interpolate) floats the caller
 *     allocates (8-byte aligned for paired rounding), zero-filled by the callee, then rounded once into grad_points.
 *     Each element is within gamma_k * sum|t| of the exact sum (as the float32 grads above) plus half a 16-bit ulp of
 *     the result.  No 16-bit atomics (those would round at every add).  Three launches (memset, scatter, round).
 * ---------------------------------------------------------------------------------------- */
#define PVN3D_F16 1
#define PVN3D_BF16 2
int pvn3d_group_points_16(int dtype, const void *points, const int *idx, int b, int c, int n, int npoints, int nsample,
                          void *out, pvn3d_stream_t stream);
int pvn3d_group_points_grad_16(int dtype, const void *grad_out, const int *idx, int b, int c, int n, int npoints,
                               int nsample, float *scratch, void *grad_points, pvn3d_stream_t stream);
int pvn3d_three_interpolate_16(int dtype, const void *points, const int *idx, const float *weight, int b, int c, int m,
                               int n, void *out, pvn3d_stream_t stream);
int pvn3d_three_interpolate_grad_16(int dtype, const void *grad_out, const int *idx, const float *weight, int b, int c,
                                    int n, int m, float *scratch, void *grad_points, pvn3d_stream_t stream);

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
 *      out[p, col0 + 0:n_pad] = act( A[p, 0:k_pad] . W^T + bias )
 *   w    [n_pad, k_pad] f32, BN folded into rows, values rounded to TF32, zero padded
 *        (k_pad multiple of 32, n_pad multiple of 16), 16-byte aligned (else PVN3D_ERR_INVALID_ARG: it is
 *        read 16 bytes at a time); bias [n_pad] (folded BN shift, 0 in the pad)
 *   out  point-major rows of length ldo (ldo, col0 multiples of 4)
 * Arithmetic: TF32 operands (round-to-nearest), fp32 accumulation.
 * flags: PVN3D_MLP_RELU       apply ReLU (flags = 1 / 0 is the plain relu switch)
 *        PVN3D_MLP_ROUND_OUT  store the activations already rounded to TF32
 *        PVN3D_MLP_A_TF32     (mlp_dense) `a` was produced with ROUND_OUT and is
 *                             16-byte aligned with a leading dimension % 4 == 0: its rows are copied global ->
 *                             shared asynchronously, without the rounding pass (unrounded values would be
 *                             TRUNCATED by the tensor core)
 * ---------------------------------------------------------------------------------------- */
#define PVN3D_MLP_RELU 1
#define PVN3D_MLP_ROUND_OUT 2
#define PVN3D_MLP_A_TF32 4
/* leave n SMs (0..255) to kernels running concurrently on other streams: the persistent grid is
 * sm_count - n CTAs instead of one per SM (a persistent CTA that cannot be placed stalls its kernel) */
#define PVN3D_MLP_RESERVE_SMS(n) (((n) & 0xff) << 8)

/* A = point-major activations a[rows, lda]; columns >= a_cols read as zero. */
int pvn3d_mlp_dense(const float *a, int lda, int a_cols, long long rows, const float *w,
                    const float *bias, int k_pad, int n_pad, int flags, float *out, int ldo, int col0,
                    pvn3d_stream_t stream);
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
 * relu(U[idx] - V) as its operand (pvn3d_mlp_sa_fact2(w)).  The table carries x as hi + lo TF32 parts (columns
 * [c_feat, c_feat+3) and [c_feat+3, c_feat+6)), to be multiplied by [W1f | W1x | W1x]: the coordinate term is
 * evaluated to ~2^-21, MORE accurately than rounding the difference x_j - c_i to TF32 as cuDNN's TF32 path
 * does.
 *   pvn3d_sa_factor_table: xyz [rows,3], feat_pm [rows, ldf] (c_feat columns) -> out [rows, k_pad] TF32-rounded
 *   pvn3d_sa_centre_term : centres [rows,3], wx [n_pad,3] (TF32-rounded), bias [n_pad] -> out [rows, n_pad] */
int pvn3d_sa_factor_table(const float *xyz, const float *feat_pm, int ldf, int c_feat, long long rows, int k_pad,
                          float *out, pvn3d_stream_t stream);
int pvn3d_sa_centre_term(const float *centres, const float *wx, const float *bias, long long rows, int n_pad,
                         float *out, pvn3d_stream_t stream);
/* Layers 2 AND 3 of a factored SA scale plus the max-pool over nsample, in one launch: the layer-2 activations
 * stay in shared memory instead of going through HBM.
 *   u [B*n, ldu], v [B*m, ldu] (c_valid columns), idx [B,m,ns]
 *   A row (b*m + i)*ns + s = relu(u[b*n + idx[b,i,s]] - v[b*m + i])
 *   pvn3d_mlp_dense(A, .., layer2, PVN3D_MLP_RELU | PVN3D_MLP_ROUND_OUT) -> h
 *   pvn3d_mlp_dense(h, .., layer3, PVN3D_MLP_RELU [| PVN3D_MLP_ROUND_OUT] | PVN3D_MLP_A_TF32) -> y
 *   out[b*m + i, col0 + c] = max over s of y[(b*m + i)*ns + s, c]
 * bit for bit.  pool must equal ns.  Both layers apply ReLU; flags: PVN3D_MLP_ROUND_OUT (pooled output) and
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
 * in shared memory.  Same arguments, and bit for bit the same operation as pvn3d_mlp_sa_fact2.
 * PVN3D_ERR_UNSUPPORTED (nothing launched) unless pvn3d_mlp_sa_fact2w_supported(layer2, layer3, ns) is 1: ns 16 or
 * 32, layer3->n_pad > 128, layer2->k_pad <= 256, layer3->k_pad within the 128-column blocks of layer 2, the A and H
 * tiles and three weight stages within a block's shared memory.
 * The query is host-only and touches no device memory. */
int pvn3d_mlp_sa_fact2w(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m,
                        int ns, const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int flags, int pool,
                        float *out, int ldo, int col0, pvn3d_stream_t stream);
int pvn3d_mlp_sa_fact2w_supported(const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int ns);
/* Both layers of an FP module with a two-layer MLP (FP2-FP4), in one launch: three_interpolate and the concat are
 * fused into the first layer's operand, which is produced once per pair of 128-column blocks, and the layer-1
 * activations stay in shared memory instead of going through HBM.  Bit for bit:
 *   A row (b,j) = [ sum_t nn_w[b,j,t] * known_feat_pm[b, nn_idx[b,j,t], 0:c2] | skip_pm[b*n_unknown + j, 0:c1] | 0.. ]
 *                 (skip rows lds floats apart; the sum as pvn3d_three_interpolate evaluates it)
 *   pvn3d_mlp_dense(A, .., layer1, PVN3D_MLP_RELU | PVN3D_MLP_ROUND_OUT) -> h [b*n_unknown, layer1->n_pad]
 *   pvn3d_mlp_dense(h, .., layer2, PVN3D_MLP_RELU [| PVN3D_MLP_ROUND_OUT] | PVN3D_MLP_A_TF32) -> out
 * out rows = b * n_unknown, columns col0 .. col0 + layer2->n_pad of rows ldo apart.
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
 * the gathered rows shrink from the known descriptors (256-1024 floats) to the layer width (128-512). */
/* The skip term and the second layer of a factored FP module whose skip is an SA factor table (FP1), in one launch:
 * S never goes through HBM.  Bit for bit:
 *   pvn3d_mlp_dense(table, k, k, b*n_unknown, layer_s, PVN3D_MLP_A_TF32) -> s    (k = layer_s->k_pad, no ReLU)
 *   A row (b,j) = relu(sum_t nn_w[b,j,t] * p[b*m_known + nn_idx[b,j,t], :] + s[b*n_unknown + j, :])
 *                 (the sum as pvn3d_three_interpolate evaluates it, then one fp32 add)
 *   pvn3d_mlp_dense(A, 128, 128, b*n_unknown, layer2, PVN3D_MLP_RELU) -> rows [b*n_unknown][128], transposed per
 *                 frame -> out [b][128][n_unknown]
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

/* ------------------------------------------------------------------------------------------
 * BF16 forms of the dense layer and of the two producers of the DenseFusion activation table (PVN3D's heads in mixed
 * precision).  A pvn3d_bf16_t holds the bit pattern of one bfloat16 (torch.bfloat16).
 *      out[p, col0 + 0:n_pad] = act( A[p, 0:k_pad] . W^T + bias )
 *   a    [rows, lda] bf16 rows, 16-byte aligned, lda and a_cols multiples of 8; columns >= a_cols read as zero
 *   w    [n_pad, k_pad] bf16 (BN folded, then rounded to nearest even), zero padded, 16-byte aligned; k_pad a multiple
 *        of 64 (one 128-byte row segment), n_pad a multiple of 16; bias [n_pad] f32
 *   out  rows of ldo elements of the output type, 16-byte aligned; ldo, col0 multiples of 4, col0 + n_pad <= ldo
 * Arithmetic: bf16 operands, fp32 accumulation, fp32 bias and ReLU; a bf16 output is rounded to nearest even once.
 * flags: PVN3D_MLP_RELU, PVN3D_MLP_OUT_BF16 (out is bf16, else f32) and PVN3D_MLP_RESERVE_SMS(n); any other flag, a null
 * pointer, misalignment or a bad shape: PVN3D_ERR_INVALID_ARG before any CUDA call.
 * ---------------------------------------------------------------------------------------- */
typedef uint16_t pvn3d_bf16_t;
#define PVN3D_MLP_OUT_BF16 8
int pvn3d_mlp_dense_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, const pvn3d_bf16_t *w,
                         const float *bias, int k_pad, int n_pad, int flags, void *out, int ldo, int col0,
                         pvn3d_stream_t stream);
/* pvn3d_mlp_dense_bf16 with one bias vector per batch element, as pvn3d_mlp_dense_frame_bias (rows_per_frame % 128 == 0,
 * rows % rows_per_frame == 0) */
int pvn3d_mlp_dense_frame_bias_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, int rows_per_frame,
                                    const pvn3d_bf16_t *w, const float *bias, int k_pad, int n_pad, int flags, void *out,
                                    int ldo, int col0, pvn3d_stream_t stream);
/* f32 out[g, :] = sum over the 32 rows p in [32 g, 32 g + 32) of relu(a[p] . W^T + bias), as pvn3d_mlp_dense_sum32: the
 * sums are fp32 in a fixed order (reproducible).  ReLU always; flags: PVN3D_MLP_RELU and PVN3D_MLP_RESERVE_SMS(n). */
int pvn3d_mlp_dense_sum32_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, const pvn3d_bf16_t *w,
                               const float *bias, int k_pad, int n_pad, int flags, float *out, int ldo, int col0,
                               pvn3d_stream_t stream);
/* pvn3d_mlp_fp_fact2_rows with bf16 rows: the same arithmetic, relu(acc + b2) rounded to nearest even bf16 instead of
 * TF32 -- the bits of pvn3d_mlp_fp_fact2's [b][128][n_unknown], transposed and converted to bf16.  Arguments, flags and
 * coverage as pvn3d_mlp_fp_fact2; ldo and col0 (in bf16 elements) multiples of 8, col0 >= 0, col0 + 128 <= ldo and out
 * 16-byte aligned, else PVN3D_ERR_INVALID_ARG before any CUDA call. */
int pvn3d_mlp_fp_fact2_rows_bf16(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b,
                                 int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer_s,
                                 const pvn3d_mlp_layer_t *layer2, int flags, pvn3d_bf16_t *out, int ldo, int col0,
                                 pvn3d_stream_t stream);
/* pvn3d_gather_pixel_rows with bf16 rows: out[f * n + p][col0 + ch] = bf16(emb[f][ch][choose[f][0][p]]).  emb is f32
 * (emb_bf16 = 0, 4-byte aligned; rounded to nearest even, as torch's .to(torch.bfloat16)) or bf16 (emb_bf16 = 1, 2-byte
 * aligned; copied), so a CNN that ran under bf16 autocast needs no f32 copy.  c, ldo and col0 multiples of 8, out 16-byte
 * aligned; otherwise checks, NaN rows and PVN3D_ERR_UNSUPPORTED as pvn3d_gather_pixel_rows. */
int pvn3d_gather_pixel_rows_bf16(const void *emb, int emb_bf16, int b, int c, long long hw, const long long *choose, int n,
                                 pvn3d_bf16_t *out, int ldo, int col0, pvn3d_stream_t stream);
/* The full-resolution tail of PVN3D's CNN (pspnet.py:88-90 of Modified_PSPNet: up_3 = bilinear x2 with align_corners ->
 * Conv2d(64,64,3,padding 1) -> BatchNorm2d -> PReLU, then final = Conv2d(64,128,1)) evaluated only at the sampled pixels:
 * the rows pvn3d_gather_pixel_rows would copy out of the dense [b][128][2h][2w] embedding, to TF32 accuracy, without
 * the dense maps.  Row r = f * n + p, with (y, x) = divmod(choose[f][0][p], 2w):
 *     out[r][col0 + 0:128] = tf32( W2 . prelu(W1 . taps + b1) + b2 )
 *     taps[(3 (dy+1) + (dx+1)) * 64 + c] = the align_corners bilinear sample of x[f][:, :, c] at up-sampled pixel
 *                                          (y+dy, x+dx), dy, dx in {-1, 0, 1}; zero outside [0, 2h) x [0, 2w)
 *   x       [b][h][w][64] f32, CHANNELS-LAST, 16-byte aligned: the input of up_3 (the output of up_2); h, w >= 2
 *   choose  [b][1][n] int64 indices into the 2h x 2w image (8-byte aligned)
 *   layer1  k_pad 576, n_pad 64: the 3x3 conv with the BatchNorm folded in, K tap-major as above, TF32-rounded;
 *   layer2  k_pad 64, n_pad 128: final.  Both w 16-byte aligned, layer2->bias 8-byte aligned.
 *   slope   [64] f32: the PReLU slope of each channel (prelu(v) = v >= 0 ? v : slope * v)
 *   out     rows ldo floats apart, 16-byte aligned; ldo, col0 multiples of 4, col0 >= 0, col0 + 128 <= ldo; other
 *           columns are not touched
 * Arithmetic: taps combined in fp32 and rounded to TF32, TF32 wgmma with fp32 accumulation in both layers, the
 * layer-1 activation rounded to TF32.  An index outside [0, 4 h w) writes a row of NaN.
 * flags: PVN3D_MLP_RESERVE_SMS(n) only.  PVN3D_ERR_INVALID_ARG for null pointers, misalignment, other flags or a bad
 * column range; PVN3D_ERR_UNSUPPORTED unless pvn3d_psp_tail_supported(layer1, layer2) is 1 (the shapes above), for
 * h or w >= 2^15, b * h * w >= 2^31 or b * n >= 2^31, or when the driver cannot encode the weights' tensor maps -- all
 * before any launch.  The query is host-only and touches no device memory. */
int pvn3d_psp_tail_rows(const float *x, int b, int h, int w, const long long *choose, int n,
                        const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2, const float *slope, int flags,
                        float *out, int ldo, int col0, pvn3d_stream_t stream);
int pvn3d_psp_tail_supported(const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2);
/* pvn3d_psp_tail_rows with bf16 rows: the same arithmetic (TF32 MMAs), acc + b2 rounded to nearest even bf16 instead of
 * TF32; ldo and col0 (in bf16 elements) multiples of 8. */
int pvn3d_psp_tail_rows_bf16(const float *x, int b, int h, int w, const long long *choose, int n,
                             const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2, const float *slope, int flags,
                             pvn3d_bf16_t *out, int ldo, int col0, pvn3d_stream_t stream);
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

/* The network input of an RGB-D frame: the datasets' get_item (pvn3d/datasets/ycb/ycb_dataset.py:185-233,
 * pvn3d/datasets/linemod/linemod_dataset.py:211-271) after depth_to_cloud, batched and sync-free.
 *
 * pvn3d_frame_sample: choose_2 and the assembly of the network's input, per frame b of cloud [B,hw,3] f32 /
 * valid [B,hw] u8 (pvn3d_depth_to_cloud's outputs).  n_v = the number of valid pixels.
 *   key(p) = mix(mix(seed + (b + 1) * 0x9E3779B97F4A7C15) + p) in uint64 arithmetic (wrapping), mix = the
 *   splitmix64 finaliser z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB;
 *   z ^= z >> 31.  The keys of one frame are distinct.
 *   n_v > N: the N valid pixels with the smallest keys; 400 <= n_v <= N: every valid pixel, repeated
 *   cyclically to N (np.pad 'wrap'); both in ascending pixel order within each cycle.  n_v < 400: ok = 0 and
 *   every output row of the frame is zero.
 * outputs: choose [B,N] i64 (pixel indices), ok [B] u8, cld_rgb_nrm rows b*N + j with row_stride (>= 6)
 *   floats: columns 0..2 = cloud[b, choose], 3..5 = rgb[b, c, choose] as f32 (rgb [B,3,hw], u8 when
 *   rgb_u8 = 1, else f32); pcld [B,N,3] f32 = cloud[b, choose]; labels_out [B,N] i32 =
 *   label_image[b, choose] (label_image [B,hw] i32; labels_out NULL to skip).
 * Workspace: pvn3d_frame_sample_workspace_bytes(b, hw, n), 256-B aligned; 0 = unsupported.
 * B*hw < 2^31 and B*N < 2^31, else PVN3D_ERR_UNSUPPORTED (nothing launched). */
size_t pvn3d_frame_sample_workspace_bytes(int b, int hw, int n);
int pvn3d_frame_sample(const float *cloud, const uint8_t *valid, const void *rgb, int rgb_u8, const int *label_image,
                       int b, int hw, int n, unsigned long long seed, float *cld_rgb_nrm, long long row_stride,
                       float *pcld, long long *choose, int *labels_out, uint8_t *ok, void *workspace,
                       size_t workspace_bytes, pvn3d_stream_t stream);
/* pvn3d_knn_normals: PCL's NormalEstimation with setKSearch(50) (get_normal) at n_query query points of each
 * frame.  Reference set of frame b: the points ref[b, i] [B,n_ref,3] f32 with ref_valid[b, i] != 0 (ref_valid
 * NULL: all) and finite coordinates.  Query j of frame b: query[b, j] [B,n_query,3] f32.
 *   neighbours: the 50 reference points with the smallest float64 (dx*dx + dy*dy) + dz*dz of the float32
 *   coordinates (no FMA), lowest index first on exact ties; a query that is a reference point is its own
 *   neighbour at distance 0.
 *   C = (1/50) sum (p - mean)(p - mean)^T in float64 (two passes); n = the unit eigenvector of C's smallest
 *   eigenvalue lambda0, negated when n . q > 0 (flipped towards the viewpoint at the origin); curvature =
 *   lambda0 / trace(C).  trace(C) == 0, fewer than 50 reference points, a non-finite query or
 *   frame_ok[b] == 0 (frame_ok NULL: every frame) give n = (0, 0, 0) and curvature 0.
 * outputs: normals_out rows b*n_query + j with row_stride (>= 3) floats (n as f32); curv_out [B,n_query] f32,
 *   normals64_out [B,n_query,3] f64 and nn_idx_out [B,n_query,50] i32 (reference indices by rank, -1 where
 *   there is none) when not NULL.
 * Each call builds a search grid of every frame's reference set into the workspace
 * (pvn3d_knn_normals_workspace_bytes(b, n_ref, n_query), 256-B aligned; 0 = unsupported) on the stream.
 * B*(2*n_ref + 65) < 2^31, B*n_query*32 < 2^31 and B <= 65535, else PVN3D_ERR_UNSUPPORTED (nothing launched). */
size_t pvn3d_knn_normals_workspace_bytes(int b, int n_ref, int n_query);
int pvn3d_knn_normals(const float *ref, const uint8_t *ref_valid, int n_ref, const float *query, int n_query, int b,
                      const uint8_t *frame_ok, float *normals_out, long long row_stride, float *curv_out,
                      double *normals64_out, int *nn_idx_out, void *workspace, size_t workspace_bytes,
                      pvn3d_stream_t stream);

/* pvn3d_depth_fill: Basic_Utils.fill_missing(dpt, cam_scale, scale_2_80m) (lib/utils/basic_utils.py:436-456), i.e.
 * ip_basic's fill_in_multiscale with max_depth M = 3, extrapolate False and blur 'bilateral'
 * (lib/utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443), per frame b of depth [B,H,W] f32 (raw units, as
 * the depth PNG holds them; finite) with cam_scale[b] ([B] f32, device) -> out [B,H,W] f32.  T = 0.01f; "under
 * top" means row >= top[col], where top[col] is the first row with a value > T (0 when the column has none).
 *   1  d = (depth / cam_scale) * scale_2_80m; s1 = M - d where d > T, else d.  Bins: near T < d <= 1,
 *      med 1 < d <= 2, far d > 2.  Depth beyond 3 m makes s1 negative, which stays invalid to the end and is
 *      returned negative (after the rescale of step 11).
 *   2  s2 = s1, overwritten where > T by the dilation of s1*far (cross 3), then s1*med (cross 5), then s1*near
 *      (cross 7).  3  s3 = 5x5 dilation, then 5x5 erosion.  4  s4 = 5x5 median of s3 where s3 > T.
 *   5  top1 from s4.  6  s5 = 9x9 dilation of s4 where !(s4 > T) and under top1.  7  top2 from s5.
 *   8  six times: s = 5x5 dilation of s where s < T (not <=) and under top2.
 *   9  V = (s > T) & under top2, then s = 5x5 median of s at V.
 *  10  s = cv2.bilateralFilter(s, 5, 0.5, 2.0) at V (filtering the whole image).
 *  11  s = M - s where s > T; out = (s / scale_2_80m) * cam_scale.
 * Dilations ignore pixels outside the image, erosions likewise; medians replicate the edge.  Every
 * arithmetic step is one round-to-nearest float32 operation, so steps 1-9 (s4, s5, the pre-bilateral image
 * and both top rows) are bit-exact against a float32 restatement (equal as values: -0 == +0).
 * The bilateral is cv2's float32 algorithm: over [min, max] of the whole pre-bilateral image (zero and
 * negative pixels included) len = (float)(max - min), scale = 4096 / len, lut[i] = (float)exp(-2 (i / scale)^2),
 * i < 4098; max - min < FLT_EPSILON returns the image unfiltered.  The 13 taps with dy^2 + dx^2 <= 4, reflect-101
 * border, weight w = (float)exp(-r^2 / 8) * interp(lut, |val - s| * scale), each in float32 as cv2 does, and
 * sum(val w) / sum(w) accumulated in float32 in a fixed tap order.  Against the same weights summed in float64
 * the result differs by at most 3 * 2^-20 * max(|min|, |max|): the sums of 13 products carry at most
 * 13u and 12u relative error (u = 2^-24) of sum |val| w <= max|val| sum w, the quotient one more u, and the
 * comparison's own rounding of the float64 result one more: 27u, under 48u = 3 * 2^-20, which leaves room for
 * a one-ulp difference in a lut entry (device exp).
 * Optional outputs: stages [B,4,H,W] f32 = s4, s5, the pre-bilateral image (after step 9) and the image after
 * step 10; top_rows [B,2,W] i32 = top1, top2.  Either may be NULL.
 * Workspace: pvn3d_depth_fill_workspace_bytes(b, h, w) (two [B,H,W] images and per-frame tables), 256-B aligned;
 * 0 = unsupported.  scale_2_80m must be finite and > 0.  B*H*W < 2^31, B <= 65535 and ceil(H/8) <= 65535, else
 * PVN3D_ERR_UNSUPPORTED; a workspace that is too small gives PVN3D_ERR_WORKSPACE (nothing launched).  15
 * launches on the stream, no host sync. */
size_t pvn3d_depth_fill_workspace_bytes(int b, int h, int w);
int pvn3d_depth_fill(const float *depth, const float *cam_scale, float scale_2_80m, int b, int h, int w, float *out,
                     float *stages, int *top_rows, void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training augmentation: get_item's ColorJitter, rgb_add_noise and add_real_back
 * (ycb_dataset.py:84-177,191-204, linemod_dataset.py:103-188,211-240) from a per-frame record
 * ---------------------------------------------------------------------------------------- */
#define PVN3D_AUG_YCB 0
#define PVN3D_AUG_LINEMOD 1
/* frame kinds: YCB 0 real, 1 syn; LineMOD 0 real png, 1 render, 2 fuse */

/* One rgb_add_noise pass (80 B).  Only the fields of the pass's dataset are drawn; the others are 0. */
typedef struct {
  double s_factor, v_factor; /* HSV S and V factors: YCB U[1.25,1.45], U[1.15,1.35]; LineMOD U[.75,1.25], U[.85,1.15] */
  double sharpen_w;          /* sharpen centre weight rand*3+9 (YCB)                                             */
  double sigma;              /* GaussianBlur sigma rand()                                                         */
  int32_t sharpen;           /* p = 0.2 (YCB)                                                                     */
  int32_t motion;            /* p = 0.2                                                                           */
  int32_t angle, length;     /* int(rand*360), int(rand*15)+1                                                     */
  int32_t gauss;             /* p = 0.2                                                                           */
  int32_t ksize;             /* 3 (p = 0.8) or 5                                                                  */
  int32_t noise_sigma;       /* YCB: randint(15) (p = 0.8) else randint(25)                                       */
  int32_t extra;             /* YCB: the extra sigma-7 noise, p = 0.2                                             */
  uint64_t noise_key, extra_key; /* Philox keys of the two standard-normal fields                                 */
} pvn3d_augment_pass_t;

/* The record of one frame (208 B). */
typedef struct {
  int32_t kind;                       /* as given to the draw                                                     */
  int32_t jitter;                     /* ColorJitter runs: every YCB frame, LineMOD real png frames               */
  int32_t order[4];                   /* torch.randperm(4): 0 brightness, 1 contrast, 2 saturation, 3 hue          */
  float brightness, contrast, saturation; /* U[0.8, 1.2]                                                          */
  float hue;                          /* U[-0.05, 0.05]                                                           */
  int32_t n_pass;                     /* rgb_add_noise passes: 0, or on YCB syn / LineMOD render 1 + (p = 0.2)    */
  int32_t back;                       /* add_real_back runs after the first pass                                  */
  pvn3d_augment_pass_t passes[2];
} pvn3d_augment_params_t;

/* pvn3d_augment_draw: records [B] of the frames kinds[B] (device i32) of `dataset`, from Philox4x32-10 keyed by
 * seed with frame b's stream at subsequence b: the reference's decision structure and distributions, not its random
 * streams.  One launch, no host sync. */
int pvn3d_augment_draw(unsigned long long seed, const int32_t *kinds, int b, int dataset,
                       pvn3d_augment_params_t *params, pvn3d_stream_t stream);

/* pvn3d_augment_apply: get_item's augmentation of B frames from their records (device), in its order --
 *   YCB      jitter (RGB); if n_pass: pass 1, add_real_back, [pass 2]
 *   LineMOD  jitter if record.jitter; flip to BGR; if n_pass: pass 1, add_real_back (background flipped), [pass 2]
 * A pass is rgb_add_noise: cv2 BGR2HSV 8U (YCB feeds it RGB), S and V times the float64 factors truncated into
 * uint16 and clipped, HSV2BGR 8U (truncating in cv2's 32-pixel vector loop, rounding in the last W % 32 pixels
 * of a row, as cv2 4.13's AVX2 dispatch does); [YCB: sharpen filter2D]; [motion blur filter2D]; [GaussianBlur 8U fixed point];
 * YCB: + N(0,1) * noise_sigma, clip, uint8 truncation; [+ N(0,1) * 7, clip, truncation] -- float32, the normals
 * from Philox keyed by (key, pixel y*W+x), channel c the c-th of curand_normal4.  The jitter is PIL 12.2's
 * Image.blend in float32 and RGB<->HSV; every colour conversion, the Gaussian blur and the composite are
 * bit-exact to cv2 / PIL, filter2D sums its float32 taps in row-major order (cv2 is within 1).
 * Inputs: rgb [B,H,W,3] u8 RGB, depth [B,H,W] f32, labels [B,H,W] u8 (0 = background), back_rgb [B,H,W,3] u8
 * RGB, back_labels [B,H,W,back_label_channels] u8 (1 or 3; the reference's mask test per channel), back_depth
 * [B,H,W] f32.  Outputs: rgb_out [B,3,H,W] u8 (YCB RGB, LineMOD BGR), depth_out [B,H,W] f32.  Optional debug
 * outputs (NULL to skip): stages [B,12,H,W,3] u8 = after the jitter (and flip), pass 1's hsv, sharpen, motion,
 * gauss, noise, the composite, pass 2's five (a step that does not run repeats its input); noise [B,2,2,H,W,3] f32
 * = per pass the noise and extra fields (written where the pass adds them).
 * Workspace pvn3d_augment_workspace_bytes(b, h, w), 256-B aligned; 0 = unsupported (B*H*W*3 >= 2^31).
 * 18 launches, no host sync; capturable in a CUDA graph once one call has run on the device. */
size_t pvn3d_augment_workspace_bytes(int b, int h, int w);
int pvn3d_augment_apply(const uint8_t *rgb, const float *depth, const uint8_t *labels, const uint8_t *back_rgb,
                        const uint8_t *back_labels, int back_label_channels, const float *back_depth,
                        const pvn3d_augment_params_t *params, int b, int h, int w, int dataset, uint8_t *rgb_out,
                        float *depth_out, uint8_t *stages, float *noise, void *workspace, size_t workspace_bytes,
                        pvn3d_stream_t stream);

/* pvn3d_augment_probe: the augmentation's building blocks one at a time, for checking them exhaustively.
 *   op 0..4  colour ops on n u8 triples in -> out: 0 cv2 BGR2HSV, 1 cv2 HSV2BGR, 2 PIL RGB->HSV, 3 PIL HSV->RGB,
 *            4 PIL convert("L") (one byte out per triple), 7 cv2 HSV2BGR as its per-pixel row tail computes it
 *   op 5     GaussianBlur's fixed-point taps: in n (double ksize, double sigma) -> out n x 5 i32 (ksize used)
 *   op 6     the motion-blur line: in n (i32 angle, i32 length) -> out n x 64 i32: a, tap count, then each tap
 *            row * 256 + col in row-major order
 * One launch. */
int pvn3d_augment_probe(int op, const void *in, long long n, void *out, pvn3d_stream_t stream);

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

/* ADD and ADD-S of every ground-truth object of a batch in one call: TorchEval's eval_metric (YCB) and
 * eval_metric_lm (LineMOD), pvn3d_eval_utils.py:113-137,204-220, over the pose table of pvn3d_frame_poses_batch /
 * pvn3d_icp_refine_batch.
 *   poses [b,n_cls,3,4] f32, present [b,n_cls] u8       predicted pose and presence of each class
 *   gt_rt [b,slots,3,4] f32, cls_ids [b,slots] i32      ground-truth pose and class of each slot
 *   meshes [mesh_off[n_cls],3] f32                      object-frame points of every class, class c at rows
 *                                                        mesh_off[c] .. mesh_off[c+1]-1
 *   mesh_off [n_cls+1] i32, HOST memory                  read at call time: it sizes the grid and travels to the
 *                                                        kernels by value (a captured graph keeps those values)
 *   absent  PVN3D_ADD_ABSENT_ZEROS: a class with present == 0 is scored with the zero pose (YCB,
 *           pvn3d_eval_utils.py:123-124); PVN3D_ADD_ABSENT_IDENTITY: with [I | 0] (LineMOD's empty mask, :172-173)
 *   add, adds [b,slots] f32 (either may be NULL).  Slot (f, i) is scored when cls_ids[f, 0..i] holds no 0 (the
 *           `break` at :118-119) and cls_ids[f, i] lies in [1, n_cls); every other slot is written as NaN.
 * The arithmetic per slot is pvn3d_pose_add_adds's (same kernels): with n_cls = 2, one mesh at class 1, all ids 1 and
 * all present, the outputs equal pvn3d_pose_add_adds's bit for bit.  No host sync; the grid depends only on b, slots
 * and the largest mesh, so the call can be captured in a CUDA graph.
 * Refused before any launch: mesh_off[0] != 0, a class c >= 1 without points, n_cls < 2 or an unknown `absent`
 * (PVN3D_ERR_INVALID_ARG); n_cls > PVN3D_ADD_MAX_CLASSES, b*slots > 65535 or mesh_off[n_cls] > (2^31-1)/3
 * (PVN3D_ERR_UNSUPPORTED).  Workspace: pvn3d_frame_add_adds_workspace_bytes(b, slots, largest mesh of classes >= 1),
 * 8-byte aligned. */
#define PVN3D_ADD_ABSENT_ZEROS 0
#define PVN3D_ADD_ABSENT_IDENTITY 1
#define PVN3D_ADD_MAX_CLASSES 64
size_t pvn3d_frame_add_adds_workspace_bytes(int b, int slots, int max_points);
int pvn3d_frame_add_adds(const float *poses, const uint8_t *present, int n_cls, const float *gt_rt, const int *cls_ids,
                         int b, int slots, const float *meshes, const int *mesh_off, int absent, float *add,
                         float *adds, void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training: get_item's regression targets and model_fn's losses (csrc/train.cu)
 * ---------------------------------------------------------------------------------------- */

/* The offset targets of get_item (ycb_dataset.py:241-278, linemod_dataset.py:275-310) for a batch of sampled clouds.
 *   pcld [b,n,3] f32, labels [b,n] i32        the sampled points and their labels
 *   cls_ids [b,s] i32                          class of each meta slot in meta order, 0 = empty slot
 *   rts [b,s,3,4] f64                          the meta pose of each slot
 *   kp_table [n_cls,k,3] f32, ctr_table [n_cls,3] f32   object-frame keypoints / centre of each class id
 * ->kp_targ [b,n,k,3], ctr_targ [b,n,3], kp3ds [b,s,k,3], ctr3ds [b,s,3] f32 (every element written).
 * kp = kp_f32 . r^T + t and ctr likewise in float64 (numpy promotes to the pose's dtype); an offset is
 * float32(float64(p) - kp).  A point takes the offsets of the LAST slot whose id equals its label (the reference loop
 * overwrites); a point whose label is in no slot gets zeros.  A slot id outside [1, n_cls) is an empty slot (zero
 * kp3ds / ctr3ds, the tables are never read); a label outside [0, n_cls) matches no slot.  LineMOD is s = 2 with
 * cls_ids = [1, 0].  Refused: b > 65535, n_cls > 4096 or s*(k+1)*24 + 4*n_cls + 1024 > 48 KB (PVN3D_ERR_UNSUPPORTED).
 * One launch, no host sync. */
int pvn3d_train_targets(const float *pcld, const int *labels, const int *cls_ids, const double *rts, int b, int n,
                        int s, const float *kp_table, const float *ctr_table, int n_cls, int k, float *kp_targ,
                        float *ctr_targ, float *kp3ds, float *ctr3ds, pvn3d_stream_t stream);

/* model_fn's losses (train_ycb_pvn3d.py:172-184, lib/loss.py): any subset of
 *   focal  FocalLoss(gamma) of seg against seg_target: logpt = log_softmax(z)[t], pt = exp(logpt) DETACHED,
 *          row loss -(1-pt)^gamma logpt, mean over the rows (seg_mean = 1) or sum (0).  A target outside
 *          [0, n_cls) makes its row's loss and gradient NaN.  seg is [rows, n_cls] (seg_inner = 1) or
 *          [rows / inner, n_cls, inner] (the N,C,H,W input FocalLoss reshapes, inner = H*W).
 *   kp     OFLoss of kp_pred [b,n_kp,n,3] against kp_targ [b,n,n_kp,3] with w = labels[b,n] > 0:
 *          kp_loss[b,k] = sum_{n,c} w |pred - targ| / (sum_n w + 1e-3), float32 as lib/loss.py
 *   ctr    the same for ctr_pred [b,n_ctr,n,3] / ctr_targ [b,n,n_ctr,3]
 * loss = w_seg focal + w_kp sum(kp_loss) + w_ctr sum(ctr_loss); parts = (focal, sum(kp_loss), sum(ctr_loss));
 * acc = #(first argmax of the row == target) / M.  ok [b] u8 (or NULL; needs seg with rows = b*n) leaves the rows
 * of frames with ok = 0 out of the focal mean and the accuracy: M = n * #ok, and with no ok frame focal = acc = 0.
 * A NULL pointer turns a term off.  Sums are per-block partials combined in a fixed order: no atomics, the same bits
 * on every call.  Limits: n_cls <= 128, n_kp, n_ctr <= 48 (PVN3D_ERR_UNSUPPORTED). */
typedef struct pvn3d_loss_args {
  const float *seg;            /* logits, or NULL: no focal term                                    */
  const long long *seg_target; /* [rows] i64                                                         */
  long long seg_rows;
  int n_cls;
  int seg_inner;
  float gamma;                 /* >= 0                                                               */
  int seg_mean;
  const float *kp_pred, *kp_targ;   /* or NULL */
  int n_kp;
  const float *ctr_pred, *ctr_targ; /* or NULL */
  int n_ctr;
  const long long *labels;     /* [b,n] i64: the OF weights                                          */
  int b, n;
  const uint8_t *ok;           /* [b] or NULL                                                        */
  float w_seg, w_kp, w_ctr;
} pvn3d_loss_args_t;

/* workspace of a forward / backward pair (the backward reads what the forward kept there); 0 = invalid arguments.
 * The workspace must be 256-byte aligned. */
size_t pvn3d_train_loss_workspace_bytes(const pvn3d_loss_args_t *args);
/* loss [1], parts [3], kp_loss [b,n_kp], ctr_loss [b,n_ctr], acc [1]: any may be NULL.  Two launches. */
int pvn3d_train_loss_forward(const pvn3d_loss_args_t *args, float *loss, float *parts, float *kp_loss,
                             float *ctr_loss, float *acc, void *workspace, size_t workspace_bytes,
                             pvn3d_stream_t stream);
/* Gradients of the terms the args enable, after pvn3d_train_loss_forward on the same args and workspace.  The
 * incoming gradient of the focal term is w_seg g_loss + g_parts[0], of kp_loss[b,k] w_kp g_loss + g_parts[1] +
 * g_kp[b,k], of ctr_loss[b,k] w_ctr g_loss + g_parts[2] (NULL pointers count as 0; not all NULL).  Writes d_seg (seg's
 * layout), d_kp [b,n_kp,n,3], d_ctr [b,n_ctr,n,3] in full:
 *   d_seg[i,j] = (g / M) (-(1-pt_i)^gamma) (delta_jt - p_ij)    (M = 1 for a sum; 0 on ok = 0 rows)
 *   d_kp[b,k,n,c] = (g[b,k] / den[b]) w[b,n] sgn(diff)          (sgn 0 = 0, as torch.abs's backward)
 * One launch, no host sync. */
int pvn3d_train_loss_backward(const pvn3d_loss_args_t *args, const float *g_loss, const float *g_parts,
                              const float *g_kp, float *d_seg, float *d_kp, float *d_ctr, const void *workspace,
                              size_t workspace_bytes, pvn3d_stream_t stream);

/* ---- pose overlay (csrc/vis.cu): demo.py's mesh drawing, demo.py:122-145 ------------------------------------------ */

/* Stamp plane of the two drawing calls: b*h*w int32, 256-byte aligned; 0 = invalid arguments.  Host only. */
size_t pvn3d_vis_workspace_bytes(int b, int h, int w);

/* Draw the mesh of every predicted slot into its frame, in place:
 *   img [b,h,w,3] u8 C-contiguous; mesh_pts [P_total,3] f32 and mesh_off [n_cls+1] i32 on the device
 *   (eval_utils.pack_meshes), max_pts = the largest mesh's point count; poses [b,n_cls,3,4] f32 (poses_f64 = 0) or f64
 *   (1); present [b,n_cls] u8; order [b,s] i32 class ids in draw order; k [b,3,3] f64; colors [n_cls,3] u8.
 * Slot j of frame f draws class c = order[f,j] unless c is outside [1, n_cls) or present[f,c] is 0.  Each mesh point
 * p (promoted to f64) goes to q = (p . R^T + t) * cam_scale, (u, v, d) = q . K^T (three products summed left to right,
 * no FMA), d = 1 where d < 1e-8 (NaN stays NaN), x = rint(u / d), y = rint(v / d) converted as numpy does on x86-64
 * (NaN or outside int32: INT_MIN), clipped to [0, w] and [0, h], and paints the disc dx^2 + dy^2 <= r^2 cut to the
 * image (cv2.circle(..., -1)).  Where discs of several slots meet, the last slot wins.  Refused: null pointers,
 * n_cls < 2, s < 1, r < 0 (PVN3D_ERR_INVALID_ARG); b > 65535, s > 65535, r > 32767, h or w >= 65534
 * (PVN3D_ERR_UNSUPPORTED); a short workspace (PVN3D_ERR_WORKSPACE).  A memset and two launches, no host sync. */
int pvn3d_vis_draw_poses(uint8_t *img, int b, int h, int w, const float *mesh_pts, const int *mesh_off, int n_cls,
                         int max_pts, const void *poses, int poses_f64, const uint8_t *present, const int *order, int s,
                         const double *k, double cam_scale, const uint8_t *colors, int r, void *workspace,
                         size_t workspace_bytes, pvn3d_stream_t stream);

/* Basic_Utils.draw_p2ds (basic_utils.py:315-323) on one image [h,w,3] u8: p2ds [n,2] i32 on the device are clipped in
 * place to [0, w] x [0, h] and each paints its disc of radius r in color = c0 | c1 << 8 | c2 << 16 (the three uint8
 * channels in image order).  n = 0 does nothing.  Refusals as pvn3d_vis_draw_poses.  A memset and two launches. */
int pvn3d_vis_draw_p2ds(uint8_t *img, int h, int w, int *p2ds, int n, int r, unsigned color, void *workspace,
                        size_t workspace_bytes, pvn3d_stream_t stream);

/* ---- mesh rasteriser (csrc/render.cu): LineMOD's synthetic render / fuse frames ----------------------------------- */

/* Workspace of pvn3d_render_meshes for b frames of h x w over packed meshes of n_vtx vertices and n_faces faces: the
 * per-pixel depth keys (b*h*w u64), the snapped vertex records (b*n_vtx x 16 B), the fragment-count scan of the b*n_faces
 * face slots and its block offsets, 256-byte aligned pieces.  0 = refused sizes (any size < 1, h or w > 4096, b > 65535,
 * b*n_faces or b*n_vtx >= 2^31).  Host only. */
size_t pvn3d_render_workspace_bytes(int b, int h, int w, int n_vtx, int n_faces);

/* Rasterise vertex-coloured triangle meshes at per-frame poses into rgb [b,h,w,3] u8, depth [b,h,w] f32 (the pose's
 * units; metres for LineMOD, cam_scale = 1) and labels [b,h,w] u8 (the visible surface's class id):
 *   vtx [n_vtx,3] f32, colors [n_vtx,3] u8, faces [n_faces,3] i32 packed vertex indices; vtx_off / face_off [n_cls+1]
 *   i32, class c owning vertices [vtx_off[c], vtx_off[c+1]) and faces [face_off[c], face_off[c+1]) (faces packed by
 *   class, then by face index); poses [b,n_cls,3,4] f32 (poses_f64 = 0) or f64 (1); present [b,n_cls] u8; k [b,3,3]
 *   f64; all on the device.  Class c of frame f is drawn when 1 <= c < n_cls and present[f,c] != 0; class 0 and classes
 *   without faces draw nothing.
 * The contract (the header comment of csrc/render.cu has it in full): float64 vertex stage without FMA, q = R p + t,
 * sx = (fx q0) / q2 + cx, sy = (fy q1) / q2 + cy, so pixel (v, u) samples the ray ((u - cx) / fx, (v - cy) / fy, 1);
 * snapped to 1/256 px half to even; exact int64 edge functions with a top-left fill rule; perspective-correct 1/z and
 * colour from those edge functions in float64, depth rounded to f32, colour rint and clamped; the smallest f32 depth
 * wins, then the lower packed face index.  Triangles are skipped with zero snapped area, a vertex with z < z_near, a
 * vertex outside +-16384 px, or a vertex index outside the face's class.  Uncovered pixels are 0 in all three outputs,
 * or take back_rgb [b,h,w,3] u8 and back_depth [b,h,w] f32 (both or neither) with label 0.
 * Refused: null pointers, n_cls < 2, sizes < 1, z_near not finite and > 0, only one background buffer, an unaligned
 * workspace (PVN3D_ERR_INVALID_ARG); n_cls > 256, h or w > 4096, sizes pvn3d_render_workspace_bytes refuses
 * (PVN3D_ERR_UNSUPPORTED); a short workspace (PVN3D_ERR_WORKSPACE).  A memset and five launches, no host sync, no
 * allocation: it can be captured in a CUDA graph.  Work grows with the faces' clipped bounding-box areas. */
int pvn3d_render_meshes(const float *vtx, const uint8_t *colors, const int *faces, const int *vtx_off,
                        const int *face_off, int n_cls, int n_vtx, int n_faces, const void *poses, int poses_f64,
                        const uint8_t *present, const double *k, int b, int h, int w, double z_near,
                        const uint8_t *back_rgb, const float *back_depth, uint8_t *rgb, float *depth, uint8_t *labels,
                        void *workspace, size_t workspace_bytes, pvn3d_stream_t stream);

/* ---- fixed-order backward (csrc/determinism.cu): torch.use_deterministic_algorithms ------------------------------- */

/* Workspace of the three *_grad_ordered calls below for b frames of `slots` index entries into n points (gather: m,
 * group: npoints * nsample, three_interpolate: 3 n): the inverse index (two key and two slot-number buffers of the
 * radix sort, its per-tile digit counts and their scan, the run starts), 256-byte aligned pieces; 0 = nothing to size
 * (an empty or refused shape).  Host only: arithmetic on the arguments, no CUDA call. */
size_t pvn3d_ordered_grad_workspace_bytes(int b, int n, long long slots);

/* The gradients of pvn3d_gather_points_grad, pvn3d_group_points_grad and pvn3d_three_interpolate_grad with a fixed
 * summation order: each output element is the float32 sum of its contributions, starting from +0.0 and adding one
 * term at a time in ascending slot order (gather: slot j of idx[b,j]; group: m*S + s of idx[b,m,s]; interpolate:
 * 3*j + k of idx[b,j,k], whose term is fl(grad_out[b,c,j] * weight[b,j,k])).  The same bits on every call, stream and
 * schedule.  Indices outside [0, n) contribute nothing.  Argument checks, empty shapes (a zero fill) and the batch
 * limit as the atomic entry points; a workspace shorter than pvn3d_ordered_grad_workspace_bytes is refused
 * (PVN3D_ERR_WORKSPACE).  No host sync; 3 + 3 p launches, p = the 8-bit digits of b * n (keys, p radix passes of
 * count / scan / scatter, run starts, sums). */
int pvn3d_gather_points_grad_ordered(const float *grad_out, const int *idx, int b, int c, int n, int m,
                                     float *grad_points, void *workspace, size_t workspace_bytes,
                                     pvn3d_stream_t stream);
int pvn3d_group_points_grad_ordered(const float *grad_out, const int *idx, int b, int c, int n, int npoints,
                                    int nsample, float *grad_points, void *workspace, size_t workspace_bytes,
                                    pvn3d_stream_t stream);
int pvn3d_three_interpolate_grad_ordered(const float *grad_out, const int *idx, const float *weight, int b, int c,
                                         int n, int m, float *grad_points, void *workspace, size_t workspace_bytes,
                                         pvn3d_stream_t stream);

/* Backward of torch's adaptive_avg_pool2d on NCHW float32: grad_out [nc,oh,ow] -> grad_in [nc,ih,iw], every element
 * written once.  Bin o of an axis covers [floor(o in / out), ceil((o + 1) in / out)); input element (y, x) sums, in
 * ascending (oy, ox) over the bins holding it, (g / kW) / kH with kH, kW the bin's height and width (the order of
 * torch's own backward, pinned against it).  One launch.
 * Sides of 2^15 or more, or planes above 2^30 elements, are refused (PVN3D_ERR_UNSUPPORTED). */
int pvn3d_adaptive_avg_pool2d_backward(const float *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                       float *grad_in, pvn3d_stream_t stream);

/* Backward of torch's upsample_bilinear2d on NCHW float32: grad_out [nc,oh,ow] -> grad_in [nc,ih,iw], every element
 * written once.  Taps and lambdas as torch computes them (scale (in-1)/(out-1) with align_corners, else 1/scale_h when
 * scale_h > 0, else in/out; source fma(scale, o + 0.5, -0.5) clamped at 0 without align_corners).  Input element
 * (y, x) sums, in ascending output index and, within an output, in torch's tap order, fl(fl(lh lw) g) of the taps that
 * land on it.  One launch; sizes refused as pvn3d_adaptive_avg_pool2d_backward. */
int pvn3d_upsample_bilinear2d_backward(const float *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                       int align_corners, double scale_h, double scale_w, float *grad_in,
                                       pvn3d_stream_t stream);

/* 16-bit forms of the fixed-order grads and of the two PSPNet backward ops (dtype, element types, checks and the
 * unknown-code refusal as pvn3d_group_points_16 above).  The same inverse index, workspace and launches as the float32
 * calls: each element is the float32 sum of the widened 16-bit terms in the same ascending order, rounded once to
 * nearest even, so it is bit-equal to round16(the float32 call on grad_out converted to float32), with the same bits
 * on every call. */
int pvn3d_group_points_grad_ordered_16(int dtype, const void *grad_out, const int *idx, int b, int c, int n,
                                       int npoints, int nsample, void *grad_points, void *workspace,
                                       size_t workspace_bytes, pvn3d_stream_t stream);
int pvn3d_three_interpolate_grad_ordered_16(int dtype, const void *grad_out, const int *idx, const float *weight, int b,
                                            int c, int n, int m, void *grad_points, void *workspace,
                                            size_t workspace_bytes, pvn3d_stream_t stream);
int pvn3d_adaptive_avg_pool2d_backward_16(int dtype, const void *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                          void *grad_in, pvn3d_stream_t stream);
int pvn3d_upsample_bilinear2d_backward_16(int dtype, const void *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                          int align_corners, double scale_h, double scale_w, void *grad_in,
                                          pvn3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PVN3D_B200_H */
