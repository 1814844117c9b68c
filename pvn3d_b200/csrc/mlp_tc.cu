// mlp_tc.cu -- the shared-MLP contractions of set abstraction / feature propagation on the Hopper
// tensor cores (wgmma.mma_async tf32, fp32 accumulators in registers), with the PointNet++ data movement
// fused into the operand producers and the activation / max-pool fused into the epilogues.
//
// Replaces, per SharedMLP layer of the reference (pytorch_utils.py:25-50: Conv2d 1x1 (no bias) ->
// BatchNorm2d -> ReLU, plus F.max_pool2d over nsample at pointnet2_modules.py:64-67): one cuDNN conv,
// one cuDNN BN, one clamp kernel, [one max-pool kernel] and -- for the first layer of a scale -- the
// whole materialised grouped tensor [B,3+C,M,S] (61 MB / frame over the eight scales).
//
//   out[p, :] = act( A[p, :] . W^T + bias )            W: BN folded, K-major, TF32-rounded
//
// mlp_layer_kernel runs one dense layer on the rows of a point-major matrix [P, lda] (SA factor tables, FP1's P, the
// heads, DenseFusion).  Its producers (warps 4-11, eight lanes per row of the 128-row tile) stage the operands in the
// canonical K-major SWIZZLE_128B layout (32 fp32 = 128 B per row per stage; weights arrive by TMA, pre-rounded
// activations by cp.async).  Two MMA warpgroups (warps 12-19) each issue wgmma m64nNk8 (N = 16, 32, 64 or 128 columns
// per tile) for one 64-row half of the tile, keep the accumulator in registers, release stages once wgmma.wait_group
// has retired the MMAs that read them, and hand each finished tile to the epilogue through a swizzled shared-memory
// accumulator tile; the kernel is persistent (one CTA per SM, tiles strided), so staging of tile j+1 and the epilogue
// of tile j-1 overlap the MMAs of tile j.  The epilogue warps (0-3) read the accumulator tile one row per thread, add
// the folded-BN bias, apply ReLU and store the row, or sum relu(row) over 32 rows (DenseFusion's average pool).
//
// The SA and FP modules run on the fused kernels further down, which build the rows of their first contracted layer
// on chip: relu(U[b, idx[b,i,s]] - V[b, i]) for SA (the factored QueryAndGroup rows, pointnet2_utils.py:311-321, then
// a max over nsample), [three_interpolate(known) | skip | 0] for FP2-FP4 (pointnet2_modules.py:188-199) and
// relu(three_interpolate(P) + S) for FP1.  Each rounds its rows to TF32 as the dense producer does and keeps the dense
// layer's MMA order and epilogue arithmetic, so it equals mlp_layer_kernel run on those rows, bit for bit.
//
// TF32: operands are rounded to nearest (cvt.rna.tf32.f32) when staged, accumulation is fp32 -- the
// precision class of the reference's default cuDNN convolutions (torch.backends.cudnn.allow_tf32).
#include <cuda.h>  // CUtensorMap + the cuTensorMapEncodeTiled prototype (entry point fetched through the runtime)

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kMlpBM = 128;
constexpr int kMlpEpiWarps = 4;  // warps 0-3: epilogue (warp w drains rows 32w..32w+31 of the accumulator tile)
constexpr int kMlpProWarps = 8;  // warps 4-11: two producer groups of 128 threads, alternate K chunks
constexpr int kMlpMmaWarps = 8;  // warps 12-19: two MMA warpgroups, rows 0-63 / 64-127 of the tile
constexpr int kMlpThreads = (kMlpEpiWarps + kMlpProWarps + kMlpMmaWarps) * 32;
constexpr int kMlpMaxStages = 6;
constexpr int kMlpSmemMax = 227 * 1024;  // dynamic shared memory a block may opt into on sm_90

enum : int { PRO_DENSE = 0, PRO_FP_INTERP = 2, PRO_SA_FACT = 3 };   // row layouts of rows_setup / stage_a_chunk
enum : int { EPI_STORE = 0, EPI_SUMPOOL = 2 };

struct MlpArgs {
  // W as a TMA tensor map ([n_pad][k_pad] fp32, box 32 columns x bn rows, SWIZZLE_128B): one
  // cp.async.bulk.tensor.2d per K chunk lands the B operand in the wgmma layout
  alignas(64) CUtensorMap tmap;
  // GEMM
  const float *w;     // [n_pad][k_pad]
  const float *bias;  // [n_pad]
  long long rows;     // P
  int k_pad;          // multiple of 32
  int n_pad;          // multiple of 16
  int bn;             // columns per tile = wgmma N: 16, 32, 64 or 128 (the last tile of a row may be partial)
  int stages;
  int acc_ld;         // floats per row of the shared-memory accumulator tile: max(32, bn)
  // DENSE
  const float *a;
  int lda;
  int a_cols;  // valid columns of a (multiple of 4); the rest of k_pad reads as zero
  int a_tf32;  // a is already TF32-rounded and 16-byte aligned: copied with cp.async, no registers
  // SA_FACT: feat = U [B*n, ldf], new_xyz = V [B*m, ldf], c_feat valid columns
  const float *new_xyz, *feat;
  const int *idx;
  int ldf, c_feat, n, m, ns;
  // FP_INTERP
  const float *known_feat, *nn_w, *skip;
  const int *nn_idx;
  int c2, lds, c1, n_unknown, m_known;
  // epilogue
  float *out;
  int ldo, col0, relu;
  int round_out;  // store TF32-rounded values (the next layer then takes them with a_tf32)
  int pool;       // rows per pooled output: nsample of the fused SA kernels (16 or 32), 32 for EPI_SUMPOOL
  int reserve_sms;  // host only: SMs left to concurrent kernels (PVN3D_MLP_RESERVE_SMS in flags)
  int bias_npb;     // > 0: bias is [rows / bias_npb][n_pad] -- one vector per batch element (bias_npb % 128 == 0)
};

// ---- PTX wrappers --------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// 8-byte global store kept in program order (the epilogue loop of mlp_fp_fact2_kernel<FPF2_OUT_ROWS> stays in registers)
__device__ __forceinline__ void stg64(float *p, float x, float y) {
  asm volatile("st.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(x), "f"(y) : "memory");
}
// 4-byte global store kept in program order (two bf16 of mlp_fp_fact2_kernel<FPF2_OUT_ROWS_BF16>)
__device__ __forceinline__ void stg32(uint16_t *p, uint32_t x) {
  asm volatile("st.global.b32 [%0], %1;" ::"l"(p), "r"(x) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
               : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 ldg128(const float *p) {
  return __ldg(reinterpret_cast<const float4 *>(p));
}
// 16-byte asynchronous copy global -> shared (LDGSTS, L2 only); src_bytes = 0 writes zeros
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, unsigned src_bytes = 16u) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// register transaction bytes on an mbarrier WITHOUT arriving (the thread arrives later like every producer)
__device__ __forceinline__ void mbar_expect_tx_only(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// one 2-D tile global -> shared through a tensor map (TMA), completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap *map, int x, int y,
                                            uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
          "r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}
// ---- wgmma (warpgroup MMA) ----------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of the accumulator registers across an asynchronous MMA
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 8] . B[N x 8]^T, both operands K-major in shared memory, fp32 accumulate.
// Accumulator fragment: thread (warp w of the warpgroup, lane l) holds in d[4j + e] the element
// row 16w + l/4 + 8 (e >> 1), column 8j + 2 (l % 4) + (e & 1).
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// One 32-column K chunk of a SWIZZLE_128B stage: four k8 steps, K = 8 tf32 = 32 bytes apart (+2 in the descriptors'
// 16-byte units).  `acc`: add to d; otherwise the first step overwrites it.
template <int N>
__device__ __forceinline__ void wgmma_chunk_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, bool acc) {
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4)
    wgmma_tf32<N>(d, adesc + static_cast<uint64_t>(k4 * 2), bdesc + static_cast<uint64_t>(k4 * 2), (acc || k4 > 0) ? 1u : 0u);
}
// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T with bf16 operands, both K-major (no transpose) in shared memory, fp32
// accumulate; the same fragment layout as wgmma_tf32.  K = 16 bf16 is 32 bytes, as K = 8 tf32 is.
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_bf16<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_bf16<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// two floats -> bf16x2 (round to nearest even), `lo` in the low half: the element at the lower address
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// K-major SWIZZLE_128B shared-memory matrix descriptor of wgmma: start >> 4, LBO = 1 (unused for
// swizzled K-major), SBO = 1024 B (8 rows x 128 B), layout type 1 (128-byte swizzle) in bits 62-63.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ---- shared-memory accumulator tile: 128 rows x acc_ld floats (acc_ld a multiple of 32), the 16-byte
// chunks of every 128-byte line XOR-swizzled by row & 7 so that a thread per row (epilogue) and the
// wgmma fragment stores both run without bank conflicts
__device__ __forceinline__ uint32_t acc_off(int r, int c, int ld) {
  return static_cast<uint32_t>(r * ld * 4 + ((c >> 5) << 7) + ((((c >> 2) & 7) ^ (r & 7)) << 4) + (c & 3) * 4);
}
// the warpgroup's 64 x N fragment into rows 64 wg.. of the tile (frag_row = 64 wg + 16 (warp & 3) + lane / 4)
template <int N>
__device__ __forceinline__ void acc_store(uint32_t acc_s, int ld, int frag_row, unsigned lane, const float (&d)[N / 2]) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
    asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(acc_s + acc_off(frag_row, c, ld)), "f"(d[4 * j]), "f"(d[4 * j + 1])
                 : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(acc_s + acc_off(frag_row + 8, c, ld)), "f"(d[4 * j + 2]),
                 "f"(d[4 * j + 3])
                 : "memory");
  }
}
// row r, columns c0..c0+31 (c0 % 32 == 0); cols = 16: columns c0..c0+15, the rest reads as zero
__device__ __forceinline__ void acc_ld_row(uint32_t acc_s, int ld, int r, int c0, int cols, float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q < 4 || cols == 32) x = lds128(acc_s + acc_off(r, c0 + 4 * q, ld));
    v[4 * q + 0] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
  }
}

// wgmma N for `n_pad` columns: the narrowest of 16 / 32 / 64 / 128 that covers them (wider layers: 128-column tiles;
// the MMA of a ragged last tile uses the N of its own width)
__host__ __device__ constexpr int mma_n(int n_pad) { return n_pad <= 16 ? 16 : n_pad <= 32 ? 32 : n_pad <= 64 ? 64 : 128; }

// byte offset of 16-byte chunk `c` (0..7) of row `r` inside a [rows x 128 B] SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return static_cast<uint32_t>(r) * 128u + (static_cast<uint32_t>(c ^ (r & 7)) << 4);
}
// byte offset of column c of row frag_row in a K-major SWIZZLE_128B tile stored as K chunks of 32 columns,
// `chunk_bytes` apart (rows x 128 B each)
__device__ __forceinline__ uint32_t frag_off(int c, int frag_row, uint32_t chunk_bytes) {
  return static_cast<uint32_t>(frag_row) * 128u + static_cast<uint32_t>(c >> 5) * chunk_bytes +
         ((static_cast<uint32_t>(((c & 31) >> 2) ^ (frag_row & 7))) << 4) + (c & 3) * 4u;
}
// a lane's fragment values d4[0..3] (columns c, c + 1 of rows frag_row and frag_row + 8) into that tile as
// tf32(act(value, e)), e = 0 / 1 the column c / c + 1
template <typename Act>
__device__ __forceinline__ void sts_frag_tf32(uint32_t tile, uint32_t chunk_bytes, int c, int frag_row, const float *d4, Act act) {
  const uint32_t off = frag_off(c, frag_row, chunk_bytes);
  asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(tile + off), "f"(to_tf32(act(d4[0], 0))), "f"(to_tf32(act(d4[1], 1)))
               : "memory");
  asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(tile + off + 8u * 128u), "f"(to_tf32(act(d4[2], 0))),
               "f"(to_tf32(act(d4[3], 1)))
               : "memory");
}

// ---- A-operand producers ---------------------------------------------------------------------------
// A producer group is 128 threads = 4 warps; warp pw stages rows 32pw..32pw+31 of the 128-row tile.
// Inside a warp, 8 consecutive lanes share a row (lane & 7 = the 16-byte chunk of the 128-byte K
// slice), so one warp-wide LDG.128 reads four full 128-byte lines and one STS.128 fills four swizzled
// rows without bank conflicts; the 32 rows take 8 passes (row of pass j = 32pw + 4j + lane/8), whose 8
// loads are all in flight before the first store.
struct RowState {
  unsigned live;        // bit j: row of pass j exists (p < rows)
  const float *row[8];  // DENSE: a + p*lda;  SA: U row of the grouped point (b*n + idx)
  int crow[8];                 // SA: row of its centre in V (b*m + j)
  int g1[8], g2[8], g3[8];     // FP: rows of the three neighbours in known_feat (b*m_known + idx)
  float w1[8], w2[8], w3[8];   // FP: their weights
};

// rows p_first, p_first+4, ..: batch index and offset inside the batch with ONE 64-bit division
template <int PRO>
__device__ __forceinline__ void rows_setup(const MlpArgs &a, long long p_first, RowState &s) {
  s.live = 0u;
  const unsigned per_b = PRO == PRO_SA_FACT
                             ? static_cast<unsigned>(a.m) * static_cast<unsigned>(a.ns)
                             : static_cast<unsigned>(a.n_unknown);
  unsigned b0 = 0, rem0 = 0;
  if (PRO != PRO_DENSE) {
    const long long pf = p_first < a.rows ? p_first : 0;
    b0 = static_cast<unsigned>(pf / per_b);
    rem0 = static_cast<unsigned>(pf - static_cast<long long>(b0) * per_b);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const long long p = p_first + 4 * j;
    const bool live = p < a.rows;
    if (live) s.live |= 1u << j;
    const long long pc = live ? p : 0;
    unsigned rem = rem0 + 4u * j, b = b0;
    if (PRO != PRO_DENSE) {
      if (rem >= per_b) {
        const unsigned over = rem / per_b;
        b += over;
        rem -= over * per_b;
      }
      if (!live) { b = 0; rem = 0; }
    }
    if (PRO == PRO_DENSE) {
      s.row[j] = a.a + pc * a.lda;
    } else if (PRO == PRO_SA_FACT) {
      const int q = __ldg(a.idx + pc);
      s.crow[j] = static_cast<int>(b) * a.m + static_cast<int>(rem / static_cast<unsigned>(a.ns));
      s.row[j] = a.feat + static_cast<size_t>(static_cast<int>(b) * a.n + q) * a.ldf;
    } else {
      const int base = static_cast<int>(b) * a.m_known;
      s.g1[j] = base + __ldg(a.nn_idx + pc * 3 + 0);
      s.g2[j] = base + __ldg(a.nn_idx + pc * 3 + 1);
      s.g3[j] = base + __ldg(a.nn_idx + pc * 3 + 2);
      s.w1[j] = __ldg(a.nn_w + pc * 3 + 0);
      s.w2[j] = __ldg(a.nn_w + pc * 3 + 1);
      s.w3[j] = __ldg(a.nn_w + pc * 3 + 2);
    }
  }
}

__device__ __forceinline__ void sts_tf32(uint32_t addr, const float4 &v) {
  sts128(addr, to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
}

// stage columns [k0 + 4*sub, +4) of this thread's 8 rows into the swizzled A tile at `sa` (PRO_DENSE or PRO_SA_FACT)
template <int PRO>
__device__ __forceinline__ void stage_a_chunk(const MlpArgs &a, const RowState &s, int r_first, int sub, int k0,
                                              uint32_t sa, bool vec_ok) {
  const int k = k0 + 4 * sub;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (PRO == PRO_SA_FACT) {
    // second layer of a FACTORED SA scale: row (b,i,s) = relu(U[b, idx[b,i,s], :] - V[b, i, :]), where
    // U = W1 . [f_j | x_j] for every POINT and V = W1x . c_i - bias1 for every CENTRE (the first layer is linear
    // before its ReLU, so it is evaluated once per point instead of once per (centre, neighbour) pair)
    if (k >= a.c_feat) {
#pragma unroll
      for (int j = 0; j < 8; ++j) sts128(sa + sw128_off(r_first + 4 * j, sub), 0.f, 0.f, 0.f, 0.f);
      return;
    }
    // the thread's 8 rows are 4 apart inside one 32-row block: at most two centres (nsample 16), one for nsample 32:
    // two V loads + all eight U loads are in flight together
    const float4 va = ldg128(a.new_xyz + static_cast<size_t>(s.crow[0]) * a.ldf + k);
    const float4 vb = ldg128(a.new_xyz + static_cast<size_t>(s.crow[4]) * a.ldf + k);
    float4 u[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) u[j] = ldg128(s.row[j] + k);
    const bool two = a.ns % 16 == 0;   // 16-row groups never straddle centres: rows j < 4 share crow[0], j >= 4 crow[4]
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 v = j < 4 ? va : vb;
      if (!two) v = ldg128(a.new_xyz + static_cast<size_t>(s.crow[j]) * a.ldf + k);   // other nsample: per-row centre
      float4 r = make_float4(fmaxf(u[j].x - v.x, 0.f), fmaxf(u[j].y - v.y, 0.f), fmaxf(u[j].z - v.z, 0.f),
                             fmaxf(u[j].w - v.w, 0.f));
      if (!((s.live >> j) & 1u)) r = zero;
      sts_tf32(sa + sw128_off(r_first + 4 * j, sub), r);
    }
    return;
  }
  if (vec_ok && k + 4 <= a.a_cols) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (s.live >> j) & 1u ? ldg128(s.row[j] + k) : zero;
#pragma unroll
    for (int j = 0; j < 8; ++j) sts_tf32(sa + sw128_off(r_first + 4 * j, sub), v[j]);
    return;
  }
  if (k >= a.a_cols) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(sa + sw128_off(r_first + 4 * j, sub), 0.f, 0.f, 0.f, 0.f);
    return;
  }
  // generic path (a chunk that straddles a_cols / unaligned rows): the loads of the 8 passes are issued together as
  // predicated loads (which exist depends on the column only) -- no per-element branches, one round trip instead of 32
  float vv[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const bool live = (s.live >> j) & 1u;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int kk = k + e;
      const bool on = live && kk < a.a_cols;
      vv[j][e] = on ? __ldg(s.row[j] + (on ? kk : 0)) : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    sts_tf32(sa + sw128_off(r_first + 4 * j, sub), make_float4(vv[j][0], vv[j][1], vv[j][2], vv[j][3]));
}

// ---- epilogue helpers ------------------------------------------------------------------------------
// After the call, lane l holds in v[0] the SUM over the 32 lanes of the ORIGINAL v[l] (fixed order: reproducible).
__device__ __forceinline__ void warp_colsum_32(float (&v)[32], unsigned lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool hi = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float keep = hi ? v[i + o] : v[i];
      const float send = hi ? v[i] : v[i + o];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
}
struct MlpSmemCtl {
  uint64_t full[kMlpMaxStages];   // 128 arrivals: every producer thread of the filling group
  uint64_t empty[kMlpMaxStages];  // 8 arrivals: one per MMA warp, once its MMAs that read the stage have retired
  uint64_t acc_full;              // 256 arrivals: the MMA threads, once their fragments are in the accumulator tile
  uint64_t acc_empty;             // 128 arrivals: the epilogue threads, once they have read it
};

// bytes of shared memory in front of the epilogue staging: 1024-byte alignment slack, the operand ring and the
// accumulator tile (the kernels and their launchers compute the layout with the same function)
static inline __host__ __device__ uint32_t mlp_smem_front(int stages, int bn, int acc_ld) {
  return 1024u + static_cast<uint32_t>(stages) * (kMlpBM * 128u + ((static_cast<uint32_t>(bn) * 128u + 1023u) & ~1023u)) +
         kMlpBM * static_cast<uint32_t>(acc_ld) * 4u;
}

// One tile of the MMA role for one of the two warpgroups: all K chunks of the ring into register accumulators
// (chunk kc is released once wgmma.wait_group has retired it, while chunk kc+1 runs), then the 64 x N fragment
// into the accumulator tile as soon as the epilogue has drained the previous tile.
template <int N>
__device__ __forceinline__ void mma_tile(uint32_t ring, uint32_t stage_bytes, int S, long long it_base, int kc_total,
                                         uint64_t *full, uint64_t *empty, uint64_t *acc_full, uint64_t *acc_empty,
                                         unsigned acc_parity, uint32_t acc_s, int acc_ld, unsigned wg, int frag_row,
                                         unsigned lane) {
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  int prev = -1;
  for (int kc = 0; kc < kc_total; ++kc) {
    const long long it = it_base + kc;
    const int s = static_cast<int>(it % S);
    mbar_wait(&full[s], static_cast<unsigned>((it / S) & 1));
    fence_proxy_async_smem();  // cp.async / st.shared (generic proxy) data of the stage -> async proxy
    const uint32_t sa = ring + static_cast<uint32_t>(s) * stage_bytes;
    // this warpgroup's 64 rows of A start 64 x 128 B = 8 KB into the stage (a multiple of the 1 KB swizzle atom)
    const uint64_t adesc = smem_desc_sw128(sa + wg * 8192u), bdesc = smem_desc_sw128(sa + kMlpBM * 128u);
    wgmma_fence();
    wgmma_chunk_tf32<N>(d, adesc, bdesc, kc > 0);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    prev = s;
  }
  wgmma_wait<0>();
  acc_fence(d);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
  mbar_wait(acc_empty, acc_parity ^ 1u);
  acc_store<N>(acc_s, acc_ld, frag_row, lane, d);
  mbar_arrive(acc_full);
}

#define MLP_MMA_TILE(N)                                                                                            \
  mma_tile<N>(ring, stage_bytes, S, it_base, kc_total, full, empty, acc_full, acc_empty, acc_parity, acc_s, acc_ld, wg, \
              frag_row, lane)
__device__ __forceinline__ void mma_tile_n(int n, uint32_t ring, uint32_t stage_bytes, int S, long long it_base,
                                           int kc_total, uint64_t *full, uint64_t *empty, uint64_t *acc_full,
                                           uint64_t *acc_empty, unsigned acc_parity, uint32_t acc_s, int acc_ld,
                                           unsigned wg, int frag_row, unsigned lane) {
  if (n == 16) MLP_MMA_TILE(16);
  else if (n == 32) MLP_MMA_TILE(32);
  else if (n == 64) MLP_MMA_TILE(64);
  else MLP_MMA_TILE(128);
}
#undef MLP_MMA_TILE

// One tile of the MMA role of mlp_dense_bf16_kernel: mma_tile with the bf16 MMAs (64 bf16 per stage row, four
// m64nNk16 steps at the same byte offsets as the tf32 k8 steps).  The ring position (stage s and its phase) is carried
// from tile to tile in two 32-bit registers instead of being recomputed from a 64-bit chunk count.
template <int N>
__device__ __forceinline__ void mma_tile_bf16(uint32_t ring, uint32_t stage_bytes, int S, int &s, unsigned &phase,
                                              int kc_total, uint64_t *full, uint64_t *empty, uint64_t *acc_full,
                                              uint64_t *acc_empty, unsigned acc_parity, uint32_t acc_s, int acc_ld,
                                              unsigned wg, int frag_row, unsigned lane) {
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  int prev = -1;
  for (int kc = 0; kc < kc_total; ++kc) {
    mbar_wait(&full[s], phase);
    fence_proxy_async_smem();
    const uint32_t sa = ring + static_cast<uint32_t>(s) * stage_bytes;
    const uint64_t adesc = smem_desc_sw128(sa + wg * 8192u), bdesc = smem_desc_sw128(sa + kMlpBM * 128u);
    wgmma_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4)  // K = 16 bf16 = 32 bytes per instruction: +2 in 16-byte units
      wgmma_bf16<N>(d, adesc + static_cast<uint64_t>(k4 * 2), bdesc + static_cast<uint64_t>(k4 * 2),
                    (kc > 0 || k4 > 0) ? 1u : 0u);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    prev = s;
    if (++s == S) {
      s = 0;
      phase ^= 1u;
    }
  }
  wgmma_wait<0>();
  acc_fence(d);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
  mbar_wait(acc_empty, acc_parity ^ 1u);
  acc_store<N>(acc_s, acc_ld, frag_row, lane, d);
  mbar_arrive(acc_full);
}

// Persistent, warp-specialised: CTA c works on tiles c, c+grid, ... (tile = 128 rows x bn columns).
//   producers  fill a ring of K-chunk stages (A: 128 rows x 128 B, B: bn rows x 128 B), running ahead
//              of the tensor core across tile boundaries;
//   MMA        two warpgroups accumulate tile j in registers (64 rows each) while the epilogue drains tile j-1
//              from the shared-memory accumulator tile;
//   epilogue   bias / ReLU / sum-pool / stores of the tile in the accumulator tile.
template <int EPI>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_layer_kernel(const __grid_constant__ MlpArgs a) {
  // dynamic shared memory only: [operand ring: stages x stage_bytes, 1024-byte aligned][accumulator tile
  // 128 x acc_ld floats][epilogue staging 4 x 4 KB][barriers]
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t ring = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const uint32_t a_bytes = kMlpBM * 128u;
  const uint32_t stage_bytes = a_bytes + ((static_cast<uint32_t>(a.bn) * 128u + 1023u) & ~1023u);
  const uint32_t acc_s = ring + static_cast<uint32_t>(a.stages) * stage_bytes;
  const uint32_t front = mlp_smem_front(a.stages, a.bn, a.acc_ld);
  MlpSmemCtl &ctl = *reinterpret_cast<MlpSmemCtl *>(mlp_smem_raw + front + kMlpEpiWarps * 4096);

  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int kc_total = a.k_pad / 32;
  const int S = a.stages;
  const long long row_tiles = (a.rows + kMlpBM - 1) / kMlpBM;
  const int n_blocks = (a.n_pad + a.bn - 1) / a.bn;
  const long long total_tiles = row_tiles * n_blocks;

  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.full[s], 128);
      mbar_init(&ctl.empty[s], kMlpMmaWarps);
    }
    mbar_init(&ctl.acc_full, kMlpMmaWarps * 32);
    mbar_init(&ctl.acc_empty, kMlpEpiWarps * 32);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kMlpEpiWarps && warp < kMlpEpiWarps + kMlpProWarps) {
    // ================= producers ======================================================================
    const int pt = (t - kMlpEpiWarps * 32) & 127;          // thread inside the group
    const unsigned grp = (warp - kMlpEpiWarps) >> 2;       // group 0 / 1 takes even / odd chunks
    const int pw = pt >> 5, sub = static_cast<int>(lane & 7u), rg = static_cast<int>(lane >> 3);
    const int r_first = 32 * pw + rg;
    const bool vec_ok = (a.lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.a) & 15u) == 0);
    // pre-rounded rows are copied global -> shared asynchronously: activations of a ROUND_OUT layer
    // (PVN3D_MLP_A_TF32); everything else is staged through registers
    const bool a_async = a.a_tf32 && vec_ok;
    int pend0 = 0, pend1 = 0, npend = 0;  // stages whose copies are committed but not yet published
    long long it_base = 0;  // number of K chunks staged before this tile (same in every role)
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, it_base += kc_total) {
      if (kc_total == 1 && static_cast<unsigned>(it_base & 1) != grp) continue;  // other group's tile
      const long long rt = tile / n_blocks;
      const int nb = static_cast<int>(tile - rt * n_blocks);
      const long long p0 = rt * kMlpBM;
      const int n0 = nb * a.bn;
      const long long p_first = p0 + r_first;
      RowState rs;
      rows_setup<PRO_DENSE>(a, p_first, rs);
      for (int kc = 0; kc < kc_total; ++kc) {
        const long long it = it_base + kc;
        if (static_cast<unsigned>(it & 1) != grp) continue;
        const int s = static_cast<int>(it % S);
        // asynchronous path: two chunks of copies stay in flight per thread; the older one is
        // published (complete -> proxy fence -> arrive) before this thread can block on a free stage
        if (npend == 2) {
          cp_async_wait<1>();
          fence_proxy_async_smem();  // landed cp.async data (generic proxy) -> tensor-core (async) proxy
          mbar_arrive(&ctl.full[pend0]);
          pend0 = pend1;
          npend = 1;
        }
        mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        const uint32_t sa = ring + static_cast<uint32_t>(s) * stage_bytes;
        const uint32_t sb = sa + a_bytes;
        // weights: rows n0..n0+bn of W, columns kc*32..+32 (TF32-rounded, zero-padded): one tensor-map copy,
        // completing on the stage's `full` barrier in bytes
        if (pt == 0) {
          mbar_expect_tx_only(&ctl.full[s], static_cast<unsigned>(a.bn) * 128u);
          tma_load_2d(sb, &a.tmap, kc * 32, n0, &ctl.full[s]);
        }
        if (a_async) {
          const int k = kc * 32 + 4 * sub;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            cp_async16(sa + sw128_off(r_first + 4 * j, sub), rs.row[j] + (k < a.a_cols ? k : 0),
                       (((rs.live >> j) & 1u) && k < a.a_cols) ? 16u : 0u);
          cp_async_commit();
          if (npend == 0) pend0 = s; else pend1 = s;
          ++npend;
        } else {
          cp_async_commit();
          stage_a_chunk<PRO_DENSE>(a, rs, r_first, sub, kc * 32, sa, vec_ok);
          cp_async_wait<0>();        // every asynchronous chunk still pending has landed
          fence_proxy_async_smem();  // generic-proxy stores / copies -> visible to the tensor-core proxy
          if (npend >= 1) mbar_arrive(&ctl.full[pend0]);
          if (npend == 2) mbar_arrive(&ctl.full[pend1]);
          npend = 0;
          mbar_arrive(&ctl.full[s]);
        }
      }
    }
    if (npend == 2) {
      cp_async_wait<1>();
      fence_proxy_async_smem();
      mbar_arrive(&ctl.full[pend0]);
      pend0 = pend1;
      npend = 1;
    }
    if (npend == 1) {
      cp_async_wait<0>();
      fence_proxy_async_smem();
      mbar_arrive(&ctl.full[pend0]);
    }
  } else if (warp < kMlpEpiWarps) {
    // ================= epilogue: warp w drains rows 32w..32w+31 = rows p0+32w.. of the accumulator tile ====
    long long j = 0;
    const uint32_t stg = raw + front + warp * 4096u;  // after the accumulator tile
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++j) {
      const long long rt = tile / n_blocks;
      const int nb = static_cast<int>(tile - rt * n_blocks);
      const long long p0 = rt * kMlpBM;
      const int n0 = nb * a.bn;
      const int bn = min(a.bn, a.n_pad - n0);
      mbar_wait(&ctl.acc_full, static_cast<unsigned>(j & 1));
      const long long prow = p0 + warp * 32 + lane;
      // per-frame bias (a 128-row tile never straddles batch elements: bias_npb % 128 == 0)
      const float *bias_t = a.bias + (a.bias_npb > 0 ? (p0 / a.bias_npb) * a.n_pad : 0);
      for (int c0 = 0; c0 < bn; c0 += 32) {
        float v[32];
        const int cw = min(32, bn - c0);
        const unsigned chunk = lane & 7u;                       // STORE: the lane's group of four columns
        const bool col_on = static_cast<int>(chunk) * 4 < cw;
        float4 bq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (EPI == EPI_STORE && col_on) bq = ldg128(bias_t + n0 + c0 + chunk * 4);
        acc_ld_row(acc_s, a.acc_ld, static_cast<int>(warp * 32 + lane), c0, cw, v);
        if (EPI == EPI_SUMPOOL) {
          // sum over the 32 rows of the warp of relu(acc + bias): partial sums of a mean over points
          // (DenseFusion's AvgPool1d, pvn3d.py:165,178); rows past the end contribute 0
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 bq = q * 4 < cw ? ldg128(bias_t + n0 + c0 + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool on = prow < a.rows && q * 4 < cw;
            v[q * 4 + 0] = on ? fmaxf(v[q * 4 + 0] + bq.x, 0.f) : 0.f;
            v[q * 4 + 1] = on ? fmaxf(v[q * 4 + 1] + bq.y, 0.f) : 0.f;
            v[q * 4 + 2] = on ? fmaxf(v[q * 4 + 2] + bq.z, 0.f) : 0.f;
            v[q * 4 + 3] = on ? fmaxf(v[q * 4 + 3] + bq.w, 0.f) : 0.f;
          }
          warp_colsum_32(v, lane);
          const int col = static_cast<int>(lane);
          if (col < cw && p0 + warp * 32 < a.rows)
            a.out[((p0 + warp * 32) / 32) * a.ldo + a.col0 + n0 + c0 + col] = v[0];
        } else {
          // raw accumulators through a swizzled 4 KB staging tile (thread = row going in, 8 lanes per row coming
          // out: the global stores are 128-byte row segments, 4 rows per STG.128); bias / ReLU / rounding on the
          // way out, where a lane keeps ONE group of four columns -- its bias is a single float4 (loaded before
          // the accumulator wait) and the eight rows it stores are independent instruction streams
          if (cw == 32) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
              sts128(stg + lane * 128u + ((static_cast<uint32_t>(q) ^ (lane & 7u)) << 4), v[q * 4 + 0], v[q * 4 + 1],
                     v[q * 4 + 2], v[q * 4 + 3]);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              sts128(stg + lane * 128u + ((static_cast<uint32_t>(q) ^ (lane & 7u)) << 4), v[q * 4 + 0], v[q * 4 + 1],
                     v[q * 4 + 2], v[q * 4 + 3]);
          }
          __syncwarp();
          if (col_on) {
            const bool full = p0 + kMlpBM <= a.rows;
            float4 r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const unsigned row = 4u * i + (lane >> 3);
              r[i] = lds128(stg + row * 128u + ((chunk ^ (row & 7u)) << 4));
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              r[i].x += bq.x; r[i].y += bq.y; r[i].z += bq.z; r[i].w += bq.w;
              if (a.relu) {
                r[i].x = fmaxf(r[i].x, 0.f); r[i].y = fmaxf(r[i].y, 0.f); r[i].z = fmaxf(r[i].z, 0.f); r[i].w = fmaxf(r[i].w, 0.f);
              }
              if (a.round_out) {
                r[i].x = to_tf32(r[i].x); r[i].y = to_tf32(r[i].y); r[i].z = to_tf32(r[i].z); r[i].w = to_tf32(r[i].w);
              }
            }
            float *o = a.out + (p0 + warp * 32 + (lane >> 3)) * a.ldo + a.col0 + n0 + c0 + chunk * 4;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (full || p0 + warp * 32 + 4 * i + (lane >> 3) < a.rows)
                *reinterpret_cast<float4 *>(o + static_cast<size_t>(4 * i) * a.ldo) = r[i];
          }
          __syncwarp();
        }
      }
      mbar_arrive(&ctl.acc_empty);  // the accumulator tile may be overwritten
    }
  } else {
    // ================= warps 12-19: MMA, warpgroup wg takes rows 64wg..64wg+63 of every tile ===========
    const unsigned mw = warp - (kMlpEpiWarps + kMlpProWarps), wg = mw >> 2;
    const int frag_row = static_cast<int>(64 * wg + 16 * (mw & 3) + (lane >> 2));
    long long it_base = 0, j = 0;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, it_base += kc_total, ++j)
      mma_tile_n(mma_n(min(a.bn, a.n_pad - static_cast<int>(tile % n_blocks) * a.bn)), ring, stage_bytes, S, it_base,
                 kc_total, ctl.full, ctl.empty, &ctl.acc_full, &ctl.acc_empty,
                 static_cast<unsigned>(j & 1), acc_s, a.acc_ld, wg, frag_row, lane);
  }
}

// cuTensorMapEncodeTiled lives in libcuda; the library links only the runtime, so the entry point is
// fetched once through cudaGetDriverEntryPoint
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    tried = true;
  }
  return fn;
}

// tensor map of one weight matrix, fp32 or (bf16) bfloat16 elements, boxes of one 128-byte row segment x bn rows;
// false: the driver cannot encode it (every launcher then returns PVN3D_ERR_UNSUPPORTED without launching)
bool weight_tensor_map(CUtensorMap *map, const void *w, int k_pad, int n_pad, int bn, bool bf16 = false) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc || (reinterpret_cast<uintptr_t>(w) & 15u)) return false;
  const cuuint64_t elem = bf16 ? 2u : 4u;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(k_pad), static_cast<cuuint64_t>(n_pad)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(k_pad) * elem};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / elem), static_cast<cuuint32_t>(bn)};
  const cuuint32_t estr[2] = {1u, 1u};
  return enc(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void *>(w), dims,
             strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// One persistent launch: a CTA per SM not reserved for other streams (PVN3D_MLP_RESERVE_SMS), at most one per tile.
// The shared-memory opt-in is made once per kernel and device -- the latch is a static of the instantiation for Kern.
template <auto Kern, typename Args>
int launch_persistent(const Args &g, long long tiles, int threads, size_t smem, int reserve_sms, cudaStream_t st,
                      const char *name) {
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once, cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMlpSmemMax), name);
  const int sms = std::max(1, sm_count() - reserve_sms);
  Kern<<<static_cast<unsigned>(std::min<long long>(tiles, sms)), threads, smem, st>>>(g);
  return check_launch(name);
}

// tile width, accumulator tile and ring stages of a layer (mlp_layer_kernel, mlp_dense_bf16_kernel) -> dynamic shared
// memory bytes, 0 when fewer than 3 stages fit (asynchronous producers keep two chunks in flight)
size_t mlp_layout(MlpArgs &a) {
  a.bn = mma_n(a.n_pad);
  a.acc_ld = std::max(32, a.bn);
  const size_t stage_bytes = kMlpBM * 128 + align_up(static_cast<size_t>(a.bn) * 128, 1024);
  const size_t fixed = mlp_smem_front(0, a.bn, a.acc_ld) + kMlpEpiWarps * 4096 + sizeof(MlpSmemCtl);
  int stages = static_cast<int>((kMlpSmemMax - fixed) / stage_bytes);
  if (stages > kMlpMaxStages) stages = kMlpMaxStages;
  if (stages < 3) return 0;
  a.stages = stages;
  return mlp_smem_front(stages, a.bn, a.acc_ld) + kMlpEpiWarps * 4096 + sizeof(MlpSmemCtl);
}

template <int EPI>
int launch_mlp(MlpArgs &a, cudaStream_t st) {
  if (a.rows <= 0) return PVN3D_OK;
  if (a.k_pad <= 0 || a.k_pad % 32 || a.n_pad <= 0 || a.n_pad % 16 || (reinterpret_cast<uintptr_t>(a.w) & 15u))
    return PVN3D_ERR_INVALID_ARG;   // the weights are read 16 bytes at a time, by TMA
  const size_t smem = mlp_layout(a);
  if (!smem) return PVN3D_ERR_UNSUPPORTED;
  if (!weight_tensor_map(&a.tmap, a.w, a.k_pad, a.n_pad, a.bn)) return PVN3D_ERR_UNSUPPORTED;
  const long long tiles = ((a.rows + kMlpBM - 1) / kMlpBM) * ceil_div(a.n_pad, a.bn);
  return launch_persistent<mlp_layer_kernel<EPI>>(a, tiles, kMlpThreads, smem, a.reserve_sms, st, "mlp_layer_kernel");
}

// =====================================================================================================
// The dense layer with BF16 operands: the DenseFusion and head layers of FusedHeads at precision "bf16".
//
// mlp_layer_kernel<EPI> with the same roles, ring, barriers and accumulator tile, and three differences:
//   * a K chunk is 64 bf16 (one 128-byte SWIZZLE_128B row segment), so k_pad is a multiple of 64.  The weights
//     ([n_pad][k_pad] bf16) arrive by TMA, the activation rows (bf16 already, a_cols a multiple of 8) by cp.async;
//   * the MMAs are wgmma m64nNk16 with bf16 operands and fp32 accumulators, N = BN = mma_n(n_pad) a template parameter
//     for every tile: a ragged last column block runs the full width on the zero rows TMA fills in past n_pad, and its
//     epilogue stores only its own columns.  One width per instantiation keeps the MMA role within the 96 registers
//     of a 640-thread CTA: with the four-way run-time choice of mlp_layer_kernel its loop state spills;
//   * EPI_STORE writes act(acc + bias) as bf16 rows (OUT_BF16: cvt.rn.bf16x2, round to nearest even) or fp32 rows;
//     EPI_SUMPOOL sums relu(acc + bias) over 32 rows in fp32, in the fixed order of the TF32 form.
// MlpArgs::a and ::out carry the bf16 addresses; lda, ldo and col0 count elements of the pointer's own type.
template <int EPI, bool OUT_BF16, int BN>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_dense_bf16_kernel(const __grid_constant__ MlpArgs a) {
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t ring = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const uint32_t a_bytes = kMlpBM * 128u;
  const uint32_t stage_bytes = a_bytes + ((static_cast<uint32_t>(a.bn) * 128u + 1023u) & ~1023u);
  const uint32_t acc_s = ring + static_cast<uint32_t>(a.stages) * stage_bytes;
  const uint32_t front = mlp_smem_front(a.stages, a.bn, a.acc_ld);
  MlpSmemCtl &ctl = *reinterpret_cast<MlpSmemCtl *>(mlp_smem_raw + front + kMlpEpiWarps * 4096);

  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int kc_total = a.k_pad / 64;
  const int S = a.stages;
  const long long row_tiles = (a.rows + kMlpBM - 1) / kMlpBM;
  const int n_blocks = (a.n_pad + a.bn - 1) / a.bn;
  const long long total_tiles = row_tiles * n_blocks;

  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.full[s], 128);
      mbar_init(&ctl.empty[s], kMlpMmaWarps);
    }
    mbar_init(&ctl.acc_full, kMlpMmaWarps * 32);
    mbar_init(&ctl.acc_empty, kMlpEpiWarps * 32);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kMlpEpiWarps && warp < kMlpEpiWarps + kMlpProWarps) {
    // ================= producers: the asynchronous path of mlp_layer_kernel, 8 bf16 per 16-byte copy ============
    const int pt = (t - kMlpEpiWarps * 32) & 127;
    const unsigned grp = (warp - kMlpEpiWarps) >> 2;       // group 0 / 1 takes even / odd chunks
    const int pw = pt >> 5, sub = static_cast<int>(lane & 7u), rg = static_cast<int>(lane >> 3);
    const int r_first = 32 * pw + rg;
    const uint16_t *abf = reinterpret_cast<const uint16_t *>(a.a);
    int pend0 = 0, pend1 = 0, npend = 0;
    long long it_base = 0;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, it_base += kc_total) {
      if (kc_total == 1 && static_cast<unsigned>(it_base & 1) != grp) continue;  // other group's tile
      const long long rt = tile / n_blocks;
      const int nb = static_cast<int>(tile - rt * n_blocks);
      const long long p_first = rt * kMlpBM + r_first;
      const int n0 = nb * a.bn;
      const uint16_t *row[8];
      unsigned live = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const long long p = p_first + 4 * j;
        if (p < a.rows) live |= 1u << j;
        row[j] = abf + (p < a.rows ? p : 0) * a.lda;
      }
      for (int kc = 0; kc < kc_total; ++kc) {
        const long long it = it_base + kc;
        if (static_cast<unsigned>(it & 1) != grp) continue;
        const int s = static_cast<int>(it % S);
        if (npend == 2) {
          cp_async_wait<1>();
          fence_proxy_async_smem();
          mbar_arrive(&ctl.full[pend0]);
          pend0 = pend1;
          npend = 1;
        }
        mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        const uint32_t sa = ring + static_cast<uint32_t>(s) * stage_bytes;
        if (pt == 0) {
          mbar_expect_tx_only(&ctl.full[s], static_cast<unsigned>(a.bn) * 128u);
          tma_load_2d(sa + a_bytes, &a.tmap, kc * 64, n0, &ctl.full[s]);
        }
        const int k = kc * 64 + 8 * sub;
        const bool k_on = k < a.a_cols;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          cp_async16(sa + sw128_off(r_first + 4 * j, sub), row[j] + (k_on ? k : 0), (((live >> j) & 1u) && k_on) ? 16u : 0u);
        cp_async_commit();
        if (npend == 0) pend0 = s; else pend1 = s;
        ++npend;
      }
    }
    if (npend == 2) {
      cp_async_wait<1>();
      fence_proxy_async_smem();
      mbar_arrive(&ctl.full[pend0]);
      pend0 = pend1;
      npend = 1;
    }
    if (npend == 1) {
      cp_async_wait<0>();
      fence_proxy_async_smem();
      mbar_arrive(&ctl.full[pend0]);
    }
  } else if (warp < kMlpEpiWarps) {
    // ================= epilogue: warp w drains rows 32w..32w+31 of the accumulator tile (as mlp_layer_kernel) ======
    long long j = 0;
    const uint32_t stg = raw + front + warp * 4096u;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++j) {
      const long long rt = tile / n_blocks;
      const int nb = static_cast<int>(tile - rt * n_blocks);
      const long long p0 = rt * kMlpBM;
      const int n0 = nb * a.bn;
      const int bn = min(a.bn, a.n_pad - n0);
      mbar_wait(&ctl.acc_full, static_cast<unsigned>(j & 1));
      const long long prow = p0 + warp * 32 + lane;
      const float *bias_t = a.bias + (a.bias_npb > 0 ? (p0 / a.bias_npb) * a.n_pad : 0);
      for (int c0 = 0; c0 < bn; c0 += 32) {
        float v[32];
        const int cw = min(32, bn - c0);
        const unsigned chunk = lane & 7u;
        const bool col_on = static_cast<int>(chunk) * 4 < cw;
        float4 bq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (EPI == EPI_STORE && col_on) bq = ldg128(bias_t + n0 + c0 + chunk * 4);
        acc_ld_row(acc_s, a.acc_ld, static_cast<int>(warp * 32 + lane), c0, cw, v);
        if constexpr (EPI == EPI_SUMPOOL) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 bq = q * 4 < cw ? ldg128(bias_t + n0 + c0 + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool on = prow < a.rows && q * 4 < cw;
            v[q * 4 + 0] = on ? fmaxf(v[q * 4 + 0] + bq.x, 0.f) : 0.f;
            v[q * 4 + 1] = on ? fmaxf(v[q * 4 + 1] + bq.y, 0.f) : 0.f;
            v[q * 4 + 2] = on ? fmaxf(v[q * 4 + 2] + bq.z, 0.f) : 0.f;
            v[q * 4 + 3] = on ? fmaxf(v[q * 4 + 3] + bq.w, 0.f) : 0.f;
          }
          warp_colsum_32(v, lane);
          const int col = static_cast<int>(lane);
          if (col < cw && p0 + warp * 32 < a.rows)
            a.out[((p0 + warp * 32) / 32) * a.ldo + a.col0 + n0 + c0 + col] = v[0];
        } else {
          // through the swizzled 4 KB staging tile: 8 lanes per row coming out, each with ONE group of four columns
          if (cw == 32) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
              sts128(stg + lane * 128u + ((static_cast<uint32_t>(q) ^ (lane & 7u)) << 4), v[q * 4 + 0], v[q * 4 + 1],
                     v[q * 4 + 2], v[q * 4 + 3]);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              sts128(stg + lane * 128u + ((static_cast<uint32_t>(q) ^ (lane & 7u)) << 4), v[q * 4 + 0], v[q * 4 + 1],
                     v[q * 4 + 2], v[q * 4 + 3]);
          }
          __syncwarp();
          if (col_on) {
            const bool full = p0 + kMlpBM <= a.rows;
            float4 r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const unsigned row = 4u * i + (lane >> 3);
              r[i] = lds128(stg + row * 128u + ((chunk ^ (row & 7u)) << 4));
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              r[i].x += bq.x; r[i].y += bq.y; r[i].z += bq.z; r[i].w += bq.w;
              if (a.relu) {
                r[i].x = fmaxf(r[i].x, 0.f); r[i].y = fmaxf(r[i].y, 0.f); r[i].z = fmaxf(r[i].z, 0.f); r[i].w = fmaxf(r[i].w, 0.f);
              }
            }
            const long long o_off = (p0 + warp * 32 + (lane >> 3)) * a.ldo + a.col0 + n0 + c0 + chunk * 4;
            if constexpr (OUT_BF16) {
              uint16_t *o = reinterpret_cast<uint16_t *>(a.out) + o_off;   // 8-byte stores: 4 bf16
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (full || p0 + warp * 32 + 4 * i + (lane >> 3) < a.rows)
                  *reinterpret_cast<uint2 *>(o + static_cast<size_t>(4 * i) * a.ldo) =
                      make_uint2(pack_bf16x2(r[i].x, r[i].y), pack_bf16x2(r[i].z, r[i].w));
            } else {
              float *o = a.out + o_off;
#pragma unroll
              for (int i = 0; i < 8; ++i)
                if (full || p0 + warp * 32 + 4 * i + (lane >> 3) < a.rows)
                  *reinterpret_cast<float4 *>(o + static_cast<size_t>(4 * i) * a.ldo) = r[i];
            }
          }
          __syncwarp();
        }
      }
      mbar_arrive(&ctl.acc_empty);
    }
  } else {
    // ================= warps 12-19: MMA, warpgroup wg takes rows 64wg..64wg+63 of every tile ===========
    const unsigned mw = warp - (kMlpEpiWarps + kMlpProWarps), wg = mw >> 2;
    const int frag_row = static_cast<int>(64 * wg + 16 * (mw & 3) + (lane >> 2));
    int s = 0;
    unsigned phase = 0u, acc_parity = 0u;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, acc_parity ^= 1u)
      mma_tile_bf16<BN>(ring, stage_bytes, S, s, phase, kc_total, ctl.full, ctl.empty, &ctl.acc_full, &ctl.acc_empty,
                        acc_parity, acc_s, a.acc_ld, wg, frag_row, lane);
  }
}

template <int EPI, bool OUT_BF16>
int launch_mlp_bf16(MlpArgs &a, cudaStream_t st) {
  if (a.rows <= 0) return PVN3D_OK;
  const size_t smem = mlp_layout(a);
  if (!smem || !weight_tensor_map(&a.tmap, a.w, a.k_pad, a.n_pad, a.bn, true)) return PVN3D_ERR_UNSUPPORTED;
  const long long tiles = ((a.rows + kMlpBM - 1) / kMlpBM) * ceil_div(a.n_pad, a.bn);
#define MLP_BF16_LAUNCH(BN)                                                                                          \
  launch_persistent<mlp_dense_bf16_kernel<EPI, OUT_BF16, BN>>(a, tiles, kMlpThreads, smem, a.reserve_sms, st,          \
                                                              "mlp_dense_bf16_kernel")
  switch (a.bn) {
    case 16: return MLP_BF16_LAUNCH(16);
    case 32: return MLP_BF16_LAUNCH(32);
    case 64: return MLP_BF16_LAUNCH(64);
    default: return MLP_BF16_LAUNCH(128);
  }
#undef MLP_BF16_LAUNCH
}

// =====================================================================================================
// Layers 2 and 3 of a FACTORED SA scale and the max-pool over nsample in ONE persistent kernel.
//
// As separate launches the TF32-rounded layer-2 activations H would go to HBM and straight back: 67-400 MB per scale
// and 32-frame batch, far more than L2 holds.  Here they never leave the SM.  Per 128-row tile (whole centres):
//   producers (warps 0-7)  stage A1 = tf32(relu(U[idx] - V)) into a ring of K-chunk stages (stage_a_chunk<PRO_SA_FACT>),
//                          running ahead across tiles;
//   MMA       (warps 8-15) warpgroup wg accumulates rows 64wg..64wg+63 of layer 2 in registers (W2 resident in
//                          shared memory), writes tf32(relu(acc + b2)) into ITS 64 rows of a K-major SWIZZLE_128B
//                          H tile, runs layer 3 from that tile (W3 resident), and pools the layer-3 fragment in
//                          registers: max over the 16 rows of a warp by a transposing shuffle butterfly (a
//                          32-row centre combines two warps through shared memory), then + b3, ReLU, rounding
//                          and the store into the column slice col0.. of the level table.
// Same operands, wgmma N, K order and epilogue arithmetic as mlp_layer_kernel on A1, then on H: bit-identical to those
// two layers followed by a max over nsample (the max commutes with the bias add, ReLU and rounding: all monotone).
constexpr int kSa2Threads = (kMlpProWarps + kMlpMmaWarps) * 32;
constexpr int kSa2MaxStages = 8;
constexpr uint32_t kSa2StageBytes = kMlpBM * 128u;   // one A chunk: 128 rows x 32 tf32

struct Sa2Args {
  MlpArgs a;            // PRO_SA_FACT producer fields, rows, out / ldo / col0 / round_out / pool; w, bias, k_pad, n_pad: layer 2
  const float *w3, *bias3;
  int k3_pad, n3_pad;   // k3_pad >= n_pad of layer 2; its columns past that are zero
};

struct Sa2SmemCtl {
  uint64_t full[kSa2MaxStages];   // 128 arrivals: every producer thread of the filling group
  uint64_t empty[kSa2MaxStages];  // 8 arrivals: one per MMA warp, once its layer-2 MMAs that read the stage have retired
};

// shared-memory layout behind the 1024-byte aligned base (kernel and launcher use the same function):
// [W2: k2_pad/32 chunks of n2 x 128 B][W3: k3_pad/32 chunks of n3 x 128 B][H: k3_pad/32 chunks of 128 x 128 B]
// [A ring: stages x 16 KB][pool exchange: 2 warpgroups x 2 warp pairs x max(n3, 32) floats][b2: n2 floats]
// [b3: n3 floats][barriers]
struct Sa2Smem {
  uint32_t w2, w3, h, ring, xchg, b2, b3, ctl, bytes;   // offsets from the aligned base; bytes = dynamic size incl. slack
};
static inline __host__ __device__ Sa2Smem sa2_smem(int k2_pad, int n2, int k3_pad, int n3, int stages) {
  Sa2Smem s;
  s.w2 = 0;
  s.w3 = s.w2 + static_cast<uint32_t>(k2_pad / 32) * static_cast<uint32_t>(n2) * 128u;
  s.h = s.w3 + static_cast<uint32_t>(k3_pad / 32) * static_cast<uint32_t>(n3) * 128u;
  s.ring = s.h + static_cast<uint32_t>(k3_pad / 32) * kMlpBM * 128u;
  s.xchg = s.ring + static_cast<uint32_t>(stages) * kSa2StageBytes;
  s.b2 = s.xchg + 4u * static_cast<uint32_t>(n3 > 32 ? n3 : 32) * 4u;   // 32 lanes x max(1, n3 / 32) maxima per warp pair
  s.b3 = s.b2 + static_cast<uint32_t>(n2) * 4u;
  s.ctl = s.b3 + static_cast<uint32_t>(n3) * 4u;
  s.bytes = 1024u + s.ctl + static_cast<uint32_t>(sizeof(Sa2SmemCtl));
  return s;
}

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// `count` floats of a bias -> n floats of shared memory (the rest zero)
__device__ __forceinline__ void stage_bias(float *dst, const float *bias, int count, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = i < count ? __ldg(bias + i) : 0.f;
}

// `rows` rows x `k_pad` columns of a TF32-rounded weight matrix -> n rows of K-major SWIZZLE_128B chunks (rows >= rows zero)
__device__ __forceinline__ void stage_weights(uint32_t dst, const float *w, int rows, int k_pad, int n) {
  const int per_chunk = n * 8;
  for (int i = threadIdx.x; i < (k_pad / 32) * per_chunk; i += blockDim.x) {
    const int kc = i / per_chunk, r = (i - kc * per_chunk) >> 3, c = i & 7;
    const float4 v = r < rows ? ldg128(w + static_cast<size_t>(r) * k_pad + kc * 32 + c * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    sts128(dst + static_cast<uint32_t>(kc * per_chunk) * 16u + sw128_off(r, c), v.x, v.y, v.z, v.w);
  }
}

// Layer 2 of one tile for warpgroup wg: K chunks of the ring x resident W2 into registers, then
// H[row, c] = tf32(relu(acc + b2[c])) into the warpgroup's rows of the H tile (columns c < k3_pad; the rest of a
// wgmma N wider than k3_pad is never read).  Stages are released once their MMAs have retired.  b2_s: the bias
// in shared memory, zero past n_pad.
template <int N2>
__device__ __forceinline__ void sa2_layer2(const Sa2Args &g, uint32_t ring, uint32_t w2_s, uint32_t h_s,
                                           const float *b2_s, int S, int it_base, int kc2, Sa2SmemCtl &ctl, unsigned wg,
                                           int frag_row, unsigned lane) {
  float d[N2 / 2];
#pragma unroll
  for (int i = 0; i < N2 / 2; ++i) d[i] = 0.f;
  // chunk kc-1 is released as soon as its MMAs have retired (while chunk kc runs), so a tile may have more K
  // chunks than the ring has stages
  int prev = -1;
  for (int kc = 0; kc < kc2; ++kc) {
    const int it = it_base + kc;
    const int s = it % S;
    mbar_wait(&ctl.full[s], static_cast<unsigned>((it / S) & 1));
    fence_proxy_async_smem();
    const uint64_t adesc = smem_desc_sw128(ring + static_cast<uint32_t>(s) * kSa2StageBytes + wg * 8192u);
    const uint64_t bdesc = smem_desc_sw128(w2_s + static_cast<uint32_t>(kc * N2) * 128u);
    wgmma_fence();
    wgmma_chunk_tf32<N2>(d, adesc, bdesc, kc > 0);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&ctl.empty[prev]);
    }
    prev = s;
  }
  wgmma_wait<0>();
  acc_fence(d);
  if (lane == 0) mbar_arrive(&ctl.empty[prev]);
  // the lane's bias pairs, all loaded before the first store (a load between the stores' memory clobbers could not
  // be hoisted, and each one would hold up the next store)
  float2 bv[N2 / 8];
#pragma unroll
  for (int j = 0; j < N2 / 8; ++j) bv[j] = *reinterpret_cast<const float2 *>(b2_s + 8 * j + 2 * static_cast<int>(lane & 3u));
  // every warp of the warpgroup has finished the previous tile's layer 3 (its reads of H and of the pool exchange)
  named_bar_sync(1 + static_cast<int>(wg), 128);
  const int k3_pad = g.k3_pad;
#pragma unroll
  for (int j = 0; j < N2 / 8; ++j) {
    if (8 * j < k3_pad) {
      const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
      sts_frag_tf32(h_s, kMlpBM * 128u, c, frag_row, d + 4 * j,
                    [&](float x, int e) { return fmaxf(x + (e ? bv[j].y : bv[j].x), 0.f); });
    }
  }
  fence_proxy_async_smem();   // generic-proxy stores of H -> visible to the tensor core
  named_bar_sync(1 + static_cast<int>(wg), 128);
}

// one level of a max over lanes that differ in bit O: lanes keep the lower (bit clear) or upper (bit set) HALF of
// their values, combined with the partner's; HALF == 0: plain reduction of p[0]
template <int HALF, int O, int NV>
__device__ __forceinline__ void rowmax_level(float (&p)[NV], unsigned lane) {
  if constexpr (HALF >= 1) {
    const bool hi = (lane & static_cast<unsigned>(O)) != 0;
#pragma unroll
    for (int i = 0; i < HALF; ++i) {
      const float keep = hi ? p[i + HALF] : p[i];
      const float send = hi ? p[i] : p[i + HALF];
      p[i] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, O));
    }
  } else {
    p[0] = fmaxf(p[0], __shfl_xor_sync(0xffffffffu, p[0], O));
  }
}

// N2 = mma_n(layer-2 n_pad), N3 = mma_n(layer-3 n_pad): both MMA widths are compile-time, so no wgmma sits in a
// branch on a run-time width (ptxas would then fence and serialise every one of them)
template <int N2, int N3>
__global__ void __launch_bounds__(kSa2Threads, 1) mlp_sa_fact2_kernel(const __grid_constant__ Sa2Args g) {
  const MlpArgs &a = g.a;
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const int kc2 = a.k_pad / 32, kc3 = g.k3_pad / 32;
  const int S = a.stages;   // what the launcher's budget left (it computes the layout with the same function)
  const Sa2Smem L = sa2_smem(a.k_pad, N2, g.k3_pad, N3, S);
  Sa2SmemCtl &ctl = *reinterpret_cast<Sa2SmemCtl *>(mlp_smem_raw + (base - raw) + L.ctl);
  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int tiles = static_cast<int>((a.rows + kMlpBM - 1) / kMlpBM);   // the launcher checks tiles * kc2 < 2^31

  stage_weights(base + L.w2, a.w, a.n_pad, a.k_pad, N2);
  stage_weights(base + L.w3, g.w3, g.n3_pad, g.k3_pad, N3);
  float *const b2_s = reinterpret_cast<float *>(mlp_smem_raw + (base - raw) + L.b2);
  float *const b3_s = reinterpret_cast<float *>(mlp_smem_raw + (base - raw) + L.b3);
  stage_bias(b2_s, a.bias, a.n_pad, N2);
  stage_bias(b3_s, g.bias3, g.n3_pad, N3);
  // H columns past the layer-2 MMA width are K padding of layer 3: zero once, never written again
  for (uint32_t i = t; i < static_cast<uint32_t>(kc3) * kMlpBM * 8u; i += kSa2Threads) sts128(base + L.h + i * 16u, 0.f, 0.f, 0.f, 0.f);
  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.full[s], 128);
      mbar_init(&ctl.empty[s], kMlpMmaWarps);
    }
    mbar_fence_init();
  }
  fence_proxy_async_smem();   // resident weights / zeroed H (generic stores) -> tensor-core proxy
  __syncthreads();

  if (warp < kMlpProWarps) {
    // ================= producers: group grp stages the chunks it & 1 == grp (whole tiles when K is one chunk) ====
    const int pt = t & 127;
    const unsigned grp = warp >> 2;
    const int pw = pt >> 5, sub = static_cast<int>(lane & 7u), rg = static_cast<int>(lane >> 3);
    const int r_first = 32 * pw + rg;
    int it_base = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, it_base += kc2) {
      if (kc2 == 1 && static_cast<unsigned>(it_base & 1) != grp) continue;
      const long long p_first = static_cast<long long>(tile) * kMlpBM + r_first;
      RowState rs;
      rows_setup<PRO_SA_FACT>(a, p_first, rs);
      for (int kc = 0; kc < kc2; ++kc) {
        const int it = it_base + kc;
        if (static_cast<unsigned>(it & 1) != grp) continue;
        const int s = static_cast<int>(it % S);
        mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        stage_a_chunk<PRO_SA_FACT>(a, rs, r_first, sub, kc * 32, base + L.ring + static_cast<uint32_t>(s) * kSa2StageBytes,
                                   true);
        fence_proxy_async_smem();
        mbar_arrive(&ctl.full[s]);
      }
    }
  } else {
    // ================= MMA + epilogue: warpgroup wg, warp w4 of it holds rows 64wg + 16w4 .. +15 of the tile ======
    const unsigned mw = warp - kMlpProWarps, wg = mw >> 2, w4 = mw & 3u;
    const int frag_row = static_cast<int>(64 * wg + 16 * w4 + (lane >> 2));
    const uint32_t h_wg = base + L.h + wg * 8192u;
    const uint32_t xchg = base + L.xchg + (wg * 2u + (w4 >> 1)) * ((N3 > 32 ? N3 : 32) * 4u);
    constexpr int NV = N3 / 4;                 // values per lane after the max over its two rows
    constexpr int NF = NV >= 8 ? NV / 8 : 1;   // ... and after the max over the 8 lane groups
    // the pooled columns this lane stores (the same for every tile) and their layer-3 bias, held in registers
    int pool_col[NF];
    float b3v[NF];
    {
      const unsigned b4 = (lane >> 4) & 1u, b3 = (lane >> 3) & 1u, b2 = (lane >> 2) & 1u;
#pragma unroll
      for (int i = 0; i < NF; ++i) {
        const int io = i + (b4 ? NV / 2 : 0) + (b3 && NV >= 4 ? NV / 4 : 0) + (b2 && NV >= 8 ? NV / 8 : 0);
        pool_col[i] = 8 * (io >> 1) + 2 * static_cast<int>(lane & 3u) + (io & 1);
        b3v[i] = b3_s[pool_col[i]];
      }
    }
    int it_base = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, it_base += kc2) {
      const long long p0 = static_cast<long long>(tile) * kMlpBM;
      sa2_layer2<N2>(g, base + L.ring, base + L.w2, base + L.h, b2_s, S, it_base, kc2, ctl, wg, frag_row, lane);
      // ---- layer 3: A = this warpgroup's 64 rows of H, B = resident W3, same K order as the per-layer kernel
      float d[N3 / 2];
#pragma unroll
      for (int i = 0; i < N3 / 2; ++i) d[i] = 0.f;
      // one commit group per K chunk: no wgmma of a group sits behind the loop's branch (the run-time kc3 would
      // otherwise make ptxas fence the accumulator across it)
      for (int kc = 0; kc < kc3; ++kc) {
        const uint64_t adesc = smem_desc_sw128(h_wg + static_cast<uint32_t>(kc) * (kMlpBM * 128u));
        const uint64_t bdesc = smem_desc_sw128(base + L.w3 + static_cast<uint32_t>(kc * N3) * 128u);
        wgmma_fence();
        wgmma_chunk_tf32<N3>(d, adesc, bdesc, kc > 0);
        wgmma_commit();
      }
      wgmma_wait<0>();
      acc_fence(d);
      // ---- max over the warp's 16 rows: the lane's two rows, then a transposing butterfly over lane bits 4, 3, 2
      // (lanes that differ there hold the same columns); p[2j + e] is column 8j + 2 (lane & 3) + e
      float p[NV];
#pragma unroll
      for (int j = 0; j < N3 / 8; ++j) {
        p[2 * j] = fmaxf(d[4 * j], d[4 * j + 2]);
        p[2 * j + 1] = fmaxf(d[4 * j + 1], d[4 * j + 3]);
      }
      rowmax_level<NV / 2, 16>(p, lane);
      rowmax_level<NV / 4, 8>(p, lane);
      rowmax_level<NV / 8, 4>(p, lane);
      // a 32-row centre: the odd warp of each pair hands its 16-row maxima to the even one
      bool owner = true;
      long long grow = (p0 + 64 * wg + 16 * w4) / 16;
      if (a.pool == 32) {
        if (w4 & 1u) {
#pragma unroll
          for (int i = 0; i < NF; ++i)
            asm volatile("st.shared.f32 [%0], %1;" ::"r"(xchg + (lane * NF + i) * 4u), "f"(p[i]) : "memory");
          named_bar_arrive(3 + static_cast<int>(wg * 2 + (w4 >> 1)), 64);
          owner = false;
        } else {
          named_bar_sync(3 + static_cast<int>(wg * 2 + (w4 >> 1)), 64);
#pragma unroll
          for (int i = 0; i < NF; ++i) {
            float q;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(q) : "r"(xchg + (lane * NF + i) * 4u) : "memory");
            p[i] = fmaxf(p[i], q);
          }
        }
        grow = (p0 + 64 * wg + 32 * (w4 >> 1)) / 32;
      }
      // the group's rows exist entirely or not at all (rows % pool == 0); NV < 8 leaves duplicates in lane bit 2
      if (owner && grow * a.pool < a.rows && (NV >= 8 || !(lane & 4u))) {
        float *o = a.out + grow * a.ldo + a.col0;
#pragma unroll
        for (int i = 0; i < NF; ++i) {
          const int col = pool_col[i];
          if (col < g.n3_pad) {
            float r = fmaxf(p[i] + b3v[i], 0.f);
            if (a.round_out) r = to_tf32(r);
            o[col] = r;
          }
        }
      }
    }
  }
}

// ring stages pvn3d_mlp_sa_fact2 runs a scale with; 0: the scale is not covered (nsample other than 16 / 32, a layer
// wider than 128 columns, or resident weights + H tile + two stages beyond the shared memory of a block)
int sa2_stages(int k2_pad, int n2_pad, int k3_pad, int n3_pad, int ns) {
  if ((ns != 16 && ns != 32) || n2_pad > 128 || n3_pad > 128) return 0;
  const uint32_t fixed = sa2_smem(k2_pad, mma_n(n2_pad), k3_pad, mma_n(n3_pad), 0).bytes;
  if (fixed >= static_cast<uint32_t>(kMlpSmemMax)) return 0;
  const int stages = std::min<int>(kSa2MaxStages, static_cast<int>((kMlpSmemMax - fixed) / kSa2StageBytes));
  return stages >= 2 ? stages : 0;   // the two producer groups alternate stages
}

template <int N2, int N3>
int launch_sa_fact2(Sa2Args &g, int stages, cudaStream_t st) {
  MlpArgs &a = g.a;
  if (a.rows <= 0) return PVN3D_OK;
  a.stages = stages;
  const size_t smem = sa2_smem(a.k_pad, N2, g.k3_pad, N3, stages).bytes;
  const long long tiles = (a.rows + kMlpBM - 1) / kMlpBM;
  if (tiles * (a.k_pad / 32) > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;   // the kernel counts K chunks in 32 bits
  return launch_persistent<mlp_sa_fact2_kernel<N2, N3>>(g, tiles, kSa2Threads, smem, a.reserve_sms, st, "mlp_sa_fact2_kernel");
}

template <int N2>
int launch_sa_fact2_n3(Sa2Args &g, int stages, cudaStream_t st) {
  switch (mma_n(g.n3_pad)) {
    case 16: return launch_sa_fact2<N2, 16>(g, stages, st);
    case 32: return launch_sa_fact2<N2, 32>(g, stages, st);
    case 64: return launch_sa_fact2<N2, 64>(g, stages, st);
    default: return launch_sa_fact2<N2, 128>(g, stages, st);
  }
}

// =====================================================================================================
// Layers 2 and 3 of a factored SA scale with a WIDE last layer (n3_pad > 128: SA3, SA4) and the max-pool, in ONE
// persistent kernel.  mlp_sa_fact2_kernel keeps both weight matrices resident and a whole layer-3 row in registers;
// for 256 / 512 output columns neither fits (W3 of SA3 alone is 229 KB).  Here the weights STREAM and both layers
// run in 128-column blocks, so a thread never holds more than one 64 x 128 fragment.  Per 64-row tile (whole
// centres: 64 % ns == 0):
//   producers (warps 0-3)   stage A = tf32(relu(U[idx] - V)) ONCE into a resident A tile (stage_a_chunk<PRO_SA_FACT>);
//   loader    (warp 12)     streams 32-column K chunks of W2 and W3 (128 output columns each) by TMA through a ring,
//                           in the order the warpgroups consume them;
//   MMA       (warps 4-11)  both warpgroups work on the same 64 rows; warpgroup wg takes the column blocks
//                           nb % 2 == wg of each layer.  Layer 2: wgmma N = 128 over the K chunks of the A tile,
//                           then tf32(relu(acc + b2)) into the block's columns of a K-major SWIZZLE_128B H tile;
//                           layer 3: the same from the H tile, max-pooled in registers (shuffle butterfly; a
//                           32-row centre combines two warps through shared memory), + b3, ReLU, rounding, store.
// The chunks of the two blocks a warpgroup pair works on are interleaved in the ring, so both warpgroups draw
// from it at once.  Every output column keeps the per-layer kernel's operands, wgmma N (128) and K order, so the
// results are bit-identical to mlp_layer_kernel on the rows A, then on H, followed by a max over nsample.
constexpr int kSa2wBM = 64;
constexpr int kSa2wProWarps = 4;
constexpr int kSa2wLoaderWarp = kSa2wProWarps + kMlpMmaWarps;   // warp 12
constexpr int kSa2wThreads = (kSa2wLoaderWarp + 1) * 32;
constexpr int kSa2wMaxStages = 8;
constexpr int kSa2wMaxKc2 = 8;                             // layer-2 K chunks of the resident A tile (K <= 256)
constexpr uint32_t kSa2wChunk = kSa2wBM * 128u;            // one K chunk of the A or H tile: 64 rows x 32 tf32
constexpr uint32_t kSa2wStageBytes = 128u * 128u;          // one weight chunk: 128 output columns x 32 tf32

struct Sa2wArgs {
  MlpArgs a;            // PRO_SA_FACT producer fields, rows, out / ldo / col0 / round_out / pool; tmap, w, bias, k_pad, n_pad: layer 2
  alignas(64) CUtensorMap tmap3;
  const float *w3, *bias3;
  int k3_pad, n3_pad;   // k3_pad >= n_pad of layer 2; its columns past that are zero
};

struct Sa2wSmemCtl {
  uint64_t full[kSa2wMaxStages];   // the loader's arrive.expect_tx + the TMA bytes of the weight chunk
  uint64_t empty[kSa2wMaxStages];  // 4 arrivals: the warps of the warpgroup that consumed the chunk
  uint64_t a_full[kSa2wMaxKc2];    // 64 arrivals: the producer threads of K chunk kc of the A tile
  uint64_t a_empty;                // 8 arrivals: every MMA warp, once its layer-2 MMAs of the tile have retired
};

// shared-memory layout behind the 1024-byte aligned base (kernel and launcher use the same function):
// [A: k2_pad/32 chunks of 64 x 128 B][H: k3_pad/32 chunks of 64 x 128 B][weight ring: stages x 16 KB][barriers]
struct Sa2wSmem {
  uint32_t a, h, ring, ctl, bytes;   // offsets from the aligned base; bytes = dynamic size incl. alignment slack
};
static inline __host__ __device__ Sa2wSmem sa2w_smem(int k2_pad, int k3_pad, int stages) {
  Sa2wSmem s;
  s.a = 0;
  s.h = s.a + static_cast<uint32_t>(k2_pad / 32) * kSa2wChunk;
  s.ring = s.h + static_cast<uint32_t>(k3_pad / 32) * kSa2wChunk;
  s.ctl = s.ring + static_cast<uint32_t>(stages) * kSa2wStageBytes;
  s.bytes = 1024u + s.ctl + static_cast<uint32_t>(sizeof(Sa2wSmemCtl));
  return s;
}

// The weight chunks of one layer in ring order: the column blocks in pairs (2p, 2p+1), K chunks of the pair
// interleaved -- (2p, 0) (2p+1, 0) (2p, 1) (2p+1, 1) ..; chunk kc of block 2p + q is item kc * cnt + q of the pair.
__device__ __forceinline__ int sa2w_pair_blocks(int nb, int pp) { return nb - pp < 2 ? nb - pp : 2; }

// The loader warp's lane 0: the weight chunks of one layer (nb column blocks of 128, kcs K chunks, through `map`) by TMA
// into the ring in that order, each once its stage is free.  `it` counts the ring items across layers and tiles.
__device__ __forceinline__ void load_weight_blocks(int &it, const CUtensorMap *map, int nb, int kcs, uint32_t base,
                                                   uint32_t ring, int S, uint64_t *full, uint64_t *empty) {
  for (int pp = 0; pp < nb; pp += 2) {
    const int cnt = sa2w_pair_blocks(nb, pp);
    for (int kc = 0; kc < kcs; ++kc)
      for (int q = 0; q < cnt; ++q, ++it) {
        const int s = it % S;
        mbar_wait(&empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        mbar_expect_tx(&full[s], kSa2wStageBytes);   // rows past n_pad arrive as zeros and count too
        tma_load_2d(base + ring + static_cast<uint32_t>(s) * kSa2wStageBytes, map, kc * 32, (pp + q) * 128, &full[s]);
      }
  }
}

// One 64 x 128 block of a layer for the calling warpgroup: K chunks of `a_tile` (64 rows each) x the weight chunks
// of the ring into registers, each ring stage released once the MMAs that read it have retired -- except the last
// one with `keep_last`, which the caller releases (returned).  With `a_bars`, K chunk kc of the A tile is waited for
// first (layer 2; parity `a_par`).
__device__ __forceinline__ int sa2w_block(float (&d)[64], uint32_t a_tile, uint32_t ring, int S, int it0, int step, int kcs,
                                          uint64_t *full, uint64_t *empty, uint64_t *a_bars, unsigned a_par, bool keep_last,
                                          unsigned lane) {
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  int prev = -1;
  for (int kc = 0; kc < kcs; ++kc) {
    const int it = it0 + kc * step;
    const int s = it % S;
    if (a_bars) mbar_wait(&a_bars[kc], a_par);
    mbar_wait(&full[s], static_cast<unsigned>((it / S) & 1));
    fence_proxy_async_smem();
    const uint64_t adesc = smem_desc_sw128(a_tile + static_cast<uint32_t>(kc) * kSa2wChunk);
    const uint64_t bdesc = smem_desc_sw128(ring + static_cast<uint32_t>(s) * kSa2wStageBytes);
    wgmma_fence();
    wgmma_chunk_tf32<128>(d, adesc, bdesc, kc > 0);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    prev = s;
  }
  wgmma_wait<0>();
  acc_fence(d);
  if (lane == 0 && !keep_last) mbar_arrive(&empty[prev]);
  return prev;
}

__global__ void __launch_bounds__(kSa2wThreads, 1) mlp_sa_fact2w_kernel(const __grid_constant__ Sa2wArgs g) {
  const MlpArgs &a = g.a;
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const int kc2 = a.k_pad / 32, kc3 = g.k3_pad / 32;
  const int nb2 = (a.n_pad + 127) / 128, nb3 = (g.n3_pad + 127) / 128;
  const int S = a.stages;   // what the launcher's budget left (it computes the layout with the same function)
  const Sa2wSmem L = sa2w_smem(a.k_pad, g.k3_pad, S);
  Sa2wSmemCtl &ctl = *reinterpret_cast<Sa2wSmemCtl *>(mlp_smem_raw + (base - raw) + L.ctl);
  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int tiles = static_cast<int>((a.rows + kSa2wBM - 1) / kSa2wBM);   // the launcher checks the 32-bit counts

  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.full[s], 1);
      mbar_init(&ctl.empty[s], 4);
    }
    for (int kc = 0; kc < kc2; ++kc) mbar_init(&ctl.a_full[kc], 64);
    mbar_init(&ctl.a_empty, kMlpMmaWarps);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < kSa2wProWarps) {
    // ================= producers: warp w stages rows 32 (w & 1).. of the K chunks kc % 2 == w >> 1 ============
    const int rb = static_cast<int>(warp & 1u), kc_first = static_cast<int>(warp >> 1);
    const int sub = static_cast<int>(lane & 7u), r_first = 32 * rb + static_cast<int>(lane >> 3);
    int j = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++j) {
      const long long p_first = static_cast<long long>(tile) * kSa2wBM + r_first;
      RowState rs;
      rows_setup<PRO_SA_FACT>(a, p_first, rs);
      mbar_wait(&ctl.a_empty, static_cast<unsigned>((j & 1) ^ 1));   // the previous tile's layer 2 is done
      for (int kc = kc_first; kc < kc2; kc += 2) {
        stage_a_chunk<PRO_SA_FACT>(a, rs, r_first, sub, kc * 32, base + L.a + static_cast<uint32_t>(kc) * kSa2wChunk,
                                   true);
        fence_proxy_async_smem();
        mbar_arrive(&ctl.a_full[kc]);
      }
    }
  } else if (warp == kSa2wLoaderWarp) {
    // ================= loader: every weight chunk of every tile, in ring order ===============================
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x)
        for (int layer = 0; layer < 2; ++layer)
          load_weight_blocks(it, layer ? &g.tmap3 : &a.tmap, layer ? nb3 : nb2, layer ? kc3 : kc2, base, L.ring, S, ctl.full,
                             ctl.empty);
    }
  } else {
    // ================= MMA + epilogue: warpgroup wg, warp w4 of it holds rows 16 w4 .. +15 of the tile ======
    const unsigned mw = warp - kSa2wProWarps, wg = mw >> 2, w4 = mw & 3u;
    const int frag_row = static_cast<int>(16 * w4 + (lane >> 2));
    const int pair_bar = 2 + static_cast<int>(wg * 2 + (w4 >> 1));
    const int n2 = a.n_pad;
    int it_base = 0;
    float d[64];
    int j = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++j) {
      const long long p0 = static_cast<long long>(tile) * kSa2wBM;
      // ---- layer 2 -> H tile
      bool synced = false;
      for (int pp = 0; pp < nb2; pp += 2) {
        const int cnt = sa2w_pair_blocks(nb2, pp);
        if (static_cast<int>(wg) < cnt) {
          const int nb = pp + static_cast<int>(wg);
          // the bias of the lane's 32 columns, loaded before the block's MMAs so that they hide the loads' latency.
          // The producers' gathers stream through L1, so these come from L2; loaded one pair per stored pair after
          // the MMAs (as the break below forces), they held the tensor cores idle through 16 L2 round trips per block
          float b2v[32];
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int c = 128 * nb + 8 * jj + 2 * static_cast<int>(lane & 3u);
            b2v[2 * jj] = c < n2 ? __ldg(a.bias + c) : 0.f;
            b2v[2 * jj + 1] = c + 1 < n2 ? __ldg(a.bias + c + 1) : 0.f;
          }
          sa2w_block(d, base + L.a, base + L.ring, S, it_base + static_cast<int>(wg), cnt, kc2, ctl.full, ctl.empty, ctl.a_full,
                     static_cast<unsigned>(j & 1), false, lane);
          // both warpgroups have finished the previous tile's layer 3 (its reads of H)
          if (!synced) named_bar_sync(1, 2 * 128);
          synced = true;
          // H[row, c] = tf32(relu(acc + b2[c])) for the block's columns c < k3_pad; columns n2.. are layer 3's K padding
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int c = 128 * nb + 8 * jj + 2 * static_cast<int>(lane & 3u);
            if (c >= g.k3_pad) break;
            const bool on0 = c < n2, on1 = c + 1 < n2;
            const float b0 = b2v[2 * jj], b1 = b2v[2 * jj + 1];
            const uint32_t off = static_cast<uint32_t>(c >> 5) * kSa2wChunk + static_cast<uint32_t>(frag_row) * 128u +
                                 ((static_cast<uint32_t>(((c & 31) >> 2) ^ (frag_row & 7))) << 4) + (c & 3) * 4u;
            asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(base + L.h + off),
                         "f"(on0 ? to_tf32(fmaxf(d[4 * jj] + b0, 0.f)) : 0.f), "f"(on1 ? to_tf32(fmaxf(d[4 * jj + 1] + b1, 0.f)) : 0.f)
                         : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(base + L.h + off + 8u * 128u),
                         "f"(on0 ? to_tf32(fmaxf(d[4 * jj + 2] + b0, 0.f)) : 0.f),
                         "f"(on1 ? to_tf32(fmaxf(d[4 * jj + 3] + b1, 0.f)) : 0.f)
                         : "memory");
          }
        }
        it_base += kc2 * cnt;
      }
      if (lane == 0) mbar_arrive(&ctl.a_empty);   // this warp's layer-2 MMAs have retired: the A tile may be refilled
      if (!synced) named_bar_sync(1, 2 * 128);
      fence_proxy_async_smem();   // generic-proxy stores of H -> visible to the tensor core
      named_bar_sync(1, 2 * 128); // every block of H is written
      // ---- layer 3 from the H tile, pooled over the centres of the tile
      for (int pp = 0; pp < nb3; pp += 2) {
        const int cnt = sa2w_pair_blocks(nb3, pp);
        if (static_cast<int>(wg) < cnt) {
          const int nb = pp + static_cast<int>(wg);
          // the bias of the four columns this lane may store, loaded before the MMAs as in layer 2; the column of
          // p[i] after the butterfly: io = i + 16 b4 + 8 b3 + 4 b2 (lane bits 4, 3, 2), column 8 (io >> 1) + 2 (lane & 3) + (io & 1)
          const unsigned b4 = (lane >> 4) & 1u, b3 = (lane >> 3) & 1u, b2 = (lane >> 2) & 1u;
          float b3v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int io = i + (b4 ? 16 : 0) + (b3 ? 8 : 0) + (b2 ? 4 : 0);
            const int col = 128 * nb + 8 * (io >> 1) + 2 * static_cast<int>(lane & 3u) + (io & 1);
            b3v[i] = col < g.n3_pad ? __ldg(g.bias3 + col) : 0.f;
          }
          const int last = sa2w_block(d, base + L.h, base + L.ring, S, it_base + static_cast<int>(wg), cnt, kc3, ctl.full, ctl.empty, nullptr, 0u,
                                      true, lane);
          // max over the warp's 16 rows: the lane's two rows, then a transposing butterfly over lane bits 4, 3, 2
          // (lanes that differ there hold the same columns); p[2j + e] is column 8j + 2 (lane & 3) + e
          float p[32];
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            p[2 * jj] = fmaxf(d[4 * jj], d[4 * jj + 2]);
            p[2 * jj + 1] = fmaxf(d[4 * jj + 1], d[4 * jj + 3]);
          }
          rowmax_level<16, 16>(p, lane);
          rowmax_level<8, 8>(p, lane);
          rowmax_level<4, 4>(p, lane);
          // a 32-row centre: the odd warp of each pair hands its 16-row maxima to the even one through the block's
          // last weight stage -- only this warpgroup read it, its MMAs have retired, and the loader refills it only
          // after all four warps have released it below
          bool owner = true;
          long long grow = (p0 + 16 * w4) / 16;
          if (a.pool == 32) {
            const uint32_t xc = base + L.ring + static_cast<uint32_t>(last) * kSa2wStageBytes + (w4 >> 1) * 512u;
            if (w4 & 1u) {
#pragma unroll
              for (int i = 0; i < 4; ++i)
                asm volatile("st.shared.f32 [%0], %1;" ::"r"(xc + (lane * 4 + i) * 4u), "f"(p[i]) : "memory");
              fence_proxy_async_smem();   // these generic stores before the stage's next TMA write
              named_bar_sync(pair_bar, 64);
              owner = false;
            } else {
              named_bar_sync(pair_bar, 64);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                float q;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(q) : "r"(xc + (lane * 4 + i) * 4u) : "memory");
                p[i] = fmaxf(p[i], q);
              }
            }
            grow = (p0 + 32 * (w4 >> 1)) / 32;
          }
          __syncwarp();   // every lane's exchange loads / stores before the release
          if (lane == 0) mbar_arrive(&ctl.empty[last]);
          // the group's rows exist entirely or not at all (rows % pool == 0)
          if (owner && grow * a.pool < a.rows) {
            float *o = a.out + grow * a.ldo + a.col0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int io = i + (b4 ? 16 : 0) + (b3 ? 8 : 0) + (b2 ? 4 : 0);
              const int col = 128 * nb + 8 * (io >> 1) + 2 * static_cast<int>(lane & 3u) + (io & 1);
              if (col < g.n3_pad) {
                float r = fmaxf(p[i] + b3v[i], 0.f);
                if (a.round_out) r = to_tf32(r);
                o[col] = r;
              }
            }
          }
        }
        it_base += kc3 * cnt;
      }
    }
  }
}

// ring stages pvn3d_mlp_sa_fact2w runs a scale with; 0: the scale is not covered (nsample other than 16 / 32, a last
// layer of at most 128 columns -- pvn3d_mlp_sa_fact2's -- more than 8 layer-2 K chunks, a layer-3 K beyond the
// 128-column blocks of layer 2, or A + H tiles + three weight stages beyond the shared memory of a block)
int sa2w_stages(int k2_pad, int n2_pad, int k3_pad, int n3_pad, int ns) {
  // every H column layer 3 reads is written by a layer-2 block each tile: k3_pad within the 128-column blocks of layer 2
  if ((ns != 16 && ns != 32) || n3_pad <= 128 || k2_pad / 32 > kSa2wMaxKc2 || k3_pad > 128 * ceil_div(n2_pad, 128)) return 0;
  const uint32_t fixed = sa2w_smem(k2_pad, k3_pad, 0).bytes;
  if (fixed >= static_cast<uint32_t>(kMlpSmemMax)) return 0;
  const int stages = std::min<int>(kSa2wMaxStages, static_cast<int>((kMlpSmemMax - fixed) / kSa2wStageBytes));
  return stages >= 3 ? stages : 0;   // one stage per warpgroup in use and one in flight
}

int launch_sa_fact2w(Sa2wArgs &g, int stages, cudaStream_t st) {
  MlpArgs &a = g.a;
  if (a.rows <= 0) return PVN3D_OK;
  a.stages = stages;
  const size_t smem = sa2w_smem(a.k_pad, g.k3_pad, stages).bytes;
  const long long tiles = (a.rows + kSa2wBM - 1) / kSa2wBM;
  const long long chunks = static_cast<long long>(ceil_div(a.n_pad, 128)) * (a.k_pad / 32) +
                           static_cast<long long>(ceil_div(g.n3_pad, 128)) * (g.k3_pad / 32);
  if (tiles * chunks > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;   // the kernel counts weight chunks in 32 bits
  if (!weight_tensor_map(&a.tmap, a.w, a.k_pad, a.n_pad, 128) || !weight_tensor_map(&g.tmap3, g.w3, g.k3_pad, g.n3_pad, 128))
    return PVN3D_ERR_UNSUPPORTED;
  return launch_persistent<mlp_sa_fact2w_kernel>(g, tiles, kSa2wThreads, smem, a.reserve_sms, st, "mlp_sa_fact2w_kernel");
}

// =====================================================================================================
// Both layers of an FP module whose first layer reads the interpolated known descriptors and the skip columns (FP2-FP4),
// in ONE persistent kernel.
//
// As separate layer launches the TF32-rounded layer-1 activations H would go to HBM and come back once per layer-2
// column block (33-67 MB per module and 32-frame batch).  Per 64-row tile:
//   producers (warps 0-3)   stage A = [tf32(sum_t w_t known[idx_t]) | tf32(skip) | 0] in 64 x 32 K chunks through a ring
//                           (fp2_stage_chunk: row state in shared memory, not 48 registers); each chunk is read by BOTH
//                           warpgroups, so A is produced once per pair of layer-1 column blocks (once for 256 columns,
//                           twice for 512), running ahead across passes and tiles;
//   loader    (warp 12)     streams 32-column K chunks of W1 and W2 (128 output columns each) by TMA through a second
//                           ring, in the order the warpgroups consume them;
//   MMA       (warps 4-11)  both warpgroups work on the same 64 rows; warpgroup wg takes the column blocks nb % 2 == wg
//                           of each layer.  Layer 1: wgmma N = 128 over the A chunks, then tf32(relu(acc + b1)) into
//                           the block's columns of a K-major SWIZZLE_128B H tile; layer 2: the same from the H tile,
//                           relu(acc + b2) [rounded with ROUND_OUT] stored point-major, 32-byte row segments per quad.
// A thread never holds more than one 64 x 128 fragment.  Every output element keeps the per-layer kernel's operands,
// wgmma N (128), K order and epilogue arithmetic: bit-identical to mlp_layer_kernel on A (ROUND_OUT), then on H.
constexpr int kFp2BM = 64;
constexpr int kFp2ProWarps = 4;   // two pairs, a pair stages one 64-row A chunk (more warps: under 128 registers, spills)
constexpr int kFp2Pairs = kFp2ProWarps / 2;
constexpr int kFp2LoaderWarp = kFp2ProWarps + kMlpMmaWarps;      // warp 12
constexpr int kFp2Threads = (kFp2LoaderWarp + 1) * 32;
constexpr int kFp2MaxStages = 8;
constexpr uint32_t kFp2AStageBytes = kFp2BM * 128u;              // one A chunk, and one K chunk of the H tile: 64 rows x 32 tf32
constexpr uint32_t kFp2WStageBytes = 128u * 128u;                // one weight chunk: 128 output columns x 32 tf32

struct Fp2Args {
  MlpArgs a;            // PRO_FP_INTERP producer fields, rows, out / ldo / col0 / round_out; tmap, w, bias, k_pad, n_pad: layer 1
  alignas(64) CUtensorMap tmap2;
  const float *w2, *bias2;
  int k2_pad, n2_pad;   // k2_pad == n_pad of layer 1
  int a_stages, w_stages;
};

struct Fp2SmemCtl {
  uint64_t a_full[kFp2MaxStages];   // 64 arrivals: the producer threads of the pair that staged the chunk
  uint64_t a_empty[kFp2MaxStages];  // 8 arrivals: every MMA warp, once its MMAs that read the chunk have retired
  uint64_t w_full[kFp2MaxStages];   // the loader's arrive.expect_tx + the TMA bytes of the weight chunk
  uint64_t w_empty[kFp2MaxStages];  // 4 arrivals: the warps of the warpgroup that consumed the chunk
};

// shared-memory layout behind the 1024-byte aligned base (kernel, launcher and pvn3d_mlp_fp2_supported use the same
// function): [H: k2_pad/32 chunks of 64 x 128 B][A ring: a_stages x 8 KB][weight ring: w_stages x 16 KB]
// [row states: 32 B per row of each producer warp][barriers]
struct Fp2Smem {
  uint32_t h, aring, wring, rows, ctl, bytes;   // offsets from the aligned base; bytes = dynamic size incl. alignment slack
};
static inline __host__ __device__ Fp2Smem fp2_smem(int k2_pad, int a_stages, int w_stages) {
  Fp2Smem s;
  s.h = 0;
  s.aring = s.h + static_cast<uint32_t>(k2_pad / 32) * kFp2AStageBytes;
  s.wring = s.aring + static_cast<uint32_t>(a_stages) * kFp2AStageBytes;
  s.rows = s.wring + static_cast<uint32_t>(w_stages) * kFp2WStageBytes;
  s.ctl = s.rows + kFp2ProWarps * 32u * 32u;
  s.bytes = 1024u + s.ctl + static_cast<uint32_t>(sizeof(Fp2SmemCtl));
  return s;
}

// Row state of a producer thread's 8 rows (rows_setup<PRO_FP_INTERP>) in shared memory instead of 48 registers, 32 B
// per row: {g1, g2, g3, -} {w1, w2, w3, live}.  Row j of the thread is at `rst` + 128 j (its warp's rows rg + 4 j).
__device__ __forceinline__ void fp2_rows_store(const RowState &rs, uint32_t rst, unsigned sub) {
  if (sub != 0) return;   // the 8 lanes of a row hold the same state
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    asm volatile("st.shared.v4.s32 [%0], {%1,%2,%3,%4};" ::"r"(rst + 128u * j), "r"(rs.g1[j]), "r"(rs.g2[j]), "r"(rs.g3[j]), "r"(0)
                 : "memory");
    sts128(rst + 128u * j + 16u, rs.w1[j], rs.w2[j], rs.w3[j], ((rs.live >> j) & 1u) ? 1.f : 0.f);
  }
}
__device__ __forceinline__ int4 lds128i(uint32_t addr) {
  int4 v;
  asm volatile("ld.shared.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// three_interpolate of columns k .. k+3 of known_feat for the producer's 8 rows, from their row state in shared memory
// (fp2_rows_store): fma(p3,w3, fma(p1,w1, p2*w2)) as pn2_ops.cu contracts it, dead rows zero, into the swizzled operand
// tile at `sa`.  ROUND: TF32-rounded, as an operand is staged; otherwise unrounded.
template <bool ROUND>
__device__ __forceinline__ void interp_rows(const MlpArgs &a, int k, uint32_t rst, int r_first, int sub, uint32_t sa) {
  const float *kf = a.known_feat + k;
#pragma unroll
  for (int h = 0; h < 2; ++h) {  // two halves: 12 LDG.128 in flight each
    float4 p1[4], p2[4], p3[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int4 gi = lds128i(rst + 128u * (h * 4 + jj));
      p1[jj] = ldg128(kf + static_cast<size_t>(gi.x) * a.c2);
      p2[jj] = ldg128(kf + static_cast<size_t>(gi.y) * a.c2);
      p3[jj] = ldg128(kf + static_cast<size_t>(gi.z) * a.c2);
    }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = h * 4 + jj;
      const float4 w = lds128(rst + 128u * j + 16u);
      float4 v;
      v.x = __fmaf_rn(p3[jj].x, w.z, __fmaf_rn(p1[jj].x, w.x, __fmul_rn(p2[jj].x, w.y)));
      v.y = __fmaf_rn(p3[jj].y, w.z, __fmaf_rn(p1[jj].y, w.x, __fmul_rn(p2[jj].y, w.y)));
      v.z = __fmaf_rn(p3[jj].z, w.z, __fmaf_rn(p1[jj].z, w.x, __fmul_rn(p2[jj].z, w.y)));
      v.w = __fmaf_rn(p3[jj].w, w.z, __fmaf_rn(p1[jj].w, w.x, __fmul_rn(p2[jj].w, w.y)));
      if (w.w == 0.f) v = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (ROUND) sts_tf32(sa + sw128_off(r_first + 4 * j, sub), v);
      else sts128(sa + sw128_off(r_first + 4 * j, sub), v.x, v.y, v.z, v.w);
    }
  }
}

// K chunk k0 / 32 of the producer's 8 rows of A = [interpolated known | skip | 0], row state from shared memory
// (fp2_rows_store), TF32 rounding, dead rows zero
__device__ __forceinline__ void fp2_stage_chunk(const MlpArgs &a, uint32_t rst, long long p_first, int r_first, int sub,
                                                int k0, uint32_t sa, bool vec_ok) {
  const int k = k0 + 4 * sub;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (vec_ok && k + 4 <= a.c2) {
    interp_rows<true>(a, k, rst, r_first, sub, sa);
    return;
  }
  const bool skip_vec = (a.c2 % 4 == 0) && (a.lds % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.skip) & 15u) == 0);
  if (skip_vec && k >= a.c2 && k - a.c2 + 4 <= a.c1) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      v[j] = lds128(rst + 128u * j + 16u).w != 0.f ? ldg128(a.skip + (p_first + 4 * j) * a.lds + (k - a.c2)) : zero;
#pragma unroll
    for (int j = 0; j < 8; ++j) sts_tf32(sa + sw128_off(r_first + 4 * j, sub), v[j]);
    return;
  }
  if (k >= a.c2 + a.c1) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sts128(sa + sw128_off(r_first + 4 * j, sub), 0.f, 0.f, 0.f, 0.f);
    return;
  }
  // generic path (a chunk that straddles the interpolated / skip / padding boundary, unaligned rows): per element
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int4 gi = lds128i(rst + 128u * j);
    const float4 w = lds128(rst + 128u * j + 16u);
    const bool live = w.w != 0.f;
    const long long p = p_first + 4 * j;
    float vv[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int kk = k + e;
      const bool isk = live && kk < a.c2;
      const int d = kk - a.c2;
      const bool iss = live && d >= 0 && d < a.c1;
      const float *kf = a.known_feat + (isk ? kk : 0);
      const float p1 = isk ? __ldg(kf + static_cast<size_t>(gi.x) * a.c2) : 0.f;
      const float p2 = isk ? __ldg(kf + static_cast<size_t>(gi.y) * a.c2) : 0.f;
      const float p3 = isk ? __ldg(kf + static_cast<size_t>(gi.z) * a.c2) : 0.f;
      const float sk = iss ? __ldg(a.skip + p * a.lds + (iss ? d : 0)) : 0.f;
      vv[e] = isk ? __fmaf_rn(p3, w.z, __fmaf_rn(p1, w.x, __fmul_rn(p2, w.y))) : sk;
    }
    sts_tf32(sa + sw128_off(r_first + 4 * j, sub), make_float4(vv[0], vv[1], vv[2], vv[3]));
  }
}

// One 64 x 128 block of layer 1 for the calling warpgroup: the kc1 A chunks of the ring (items ita0..) x its weight
// chunks (items itw0, itw0 + 2, ..) into registers; each stage is released once the MMAs that read it have retired.
__device__ __forceinline__ void fp2_layer1_block(float (&d)[64], uint32_t aring, uint32_t wring, int SA, int SW, int ita0,
                                                 int itw0, int kc1, Fp2SmemCtl &ctl, unsigned lane) {
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  int pa = -1, pw = -1;
  for (int kc = 0; kc < kc1; ++kc) {
    const int ita = ita0 + kc, itw = itw0 + 2 * kc;
    const int sa = ita % SA, sw = itw % SW;
    mbar_wait(&ctl.a_full[sa], static_cast<unsigned>((ita / SA) & 1));
    mbar_wait(&ctl.w_full[sw], static_cast<unsigned>((itw / SW) & 1));
    fence_proxy_async_smem();
    const uint64_t adesc = smem_desc_sw128(aring + static_cast<uint32_t>(sa) * kFp2AStageBytes);
    const uint64_t bdesc = smem_desc_sw128(wring + static_cast<uint32_t>(sw) * kFp2WStageBytes);
    wgmma_fence();
    wgmma_chunk_tf32<128>(d, adesc, bdesc, kc > 0);
    wgmma_commit();
    if (pa >= 0) {
      wgmma_wait<1>();
      if (lane == 0) {
        mbar_arrive(&ctl.a_empty[pa]);
        mbar_arrive(&ctl.w_empty[pw]);
      }
    }
    pa = sa;
    pw = sw;
  }
  wgmma_wait<0>();
  acc_fence(d);
  if (lane == 0) {
    mbar_arrive(&ctl.a_empty[pa]);
    mbar_arrive(&ctl.w_empty[pw]);
  }
}

__global__ void __launch_bounds__(kFp2Threads, 1) mlp_fp2_kernel(const __grid_constant__ Fp2Args g) {
  const MlpArgs &a = g.a;
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const int kc1 = a.k_pad / 32, kc2 = g.k2_pad / 32;
  const int nb1 = a.n_pad / 128, nb2 = g.n2_pad / 128;   // nb1 = 2 or 4: every layer-1 pass has a block per warpgroup
  const int SA = g.a_stages, SW = g.w_stages;
  const Fp2Smem L = fp2_smem(g.k2_pad, SA, SW);
  Fp2SmemCtl &ctl = *reinterpret_cast<Fp2SmemCtl *>(mlp_smem_raw + (base - raw) + L.ctl);
  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int tiles = static_cast<int>((a.rows + kFp2BM - 1) / kFp2BM);   // the launcher checks the 32-bit counts

  if (t == 0) {
    for (int s = 0; s < SA; ++s) {
      mbar_init(&ctl.a_full[s], 64);
      mbar_init(&ctl.a_empty[s], kMlpMmaWarps);
    }
    for (int s = 0; s < SW; ++s) {
      mbar_init(&ctl.w_full[s], 1);
      mbar_init(&ctl.w_empty[s], 4);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < kFp2ProWarps) {
    // ================= producers: pair q = warp / 2 stages the A items it % 2 == q, warp w rows 32 (w & 1).. ======
    const unsigned pair = warp >> 1;
    const int sub = static_cast<int>(lane & 7u), r_first = 32 * static_cast<int>(warp & 1u) + static_cast<int>(lane >> 3);
    const bool vec_ok = (a.c2 % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.known_feat) & 15u) == 0);
    const int per_tile = (nb1 / 2) * kc1;   // A items per tile: one pass over K per pair of layer-1 blocks
    const uint32_t rst = base + L.rows + warp * 1024u + (lane >> 3) * 32u;
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const long long p_first = static_cast<long long>(tile) * kFp2BM + r_first;
      {
        RowState rs;
        rows_setup<PRO_FP_INTERP>(a, p_first, rs);
        __syncwarp();   // every lane is done with the previous tile's row state
        fp2_rows_store(rs, rst, static_cast<unsigned>(sub));
        __syncwarp();
      }
      for (int i = 0; i < per_tile; ++i, ++it) {
        if (static_cast<unsigned>(it % kFp2Pairs) != pair) continue;
        const int s = it % SA;
        mbar_wait(&ctl.a_empty[s], static_cast<unsigned>(((it / SA) & 1) ^ 1));
        const int kc = i % kc1;
        fp2_stage_chunk(a, rst, p_first, r_first, sub, kc * 32, base + L.aring + static_cast<uint32_t>(s) * kFp2AStageBytes, vec_ok);
        fence_proxy_async_smem();
        mbar_arrive(&ctl.a_full[s]);
      }
    }
  } else if (warp == kFp2LoaderWarp) {
    // ================= loader: every weight chunk of every tile, in ring order ===============================
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x)
        for (int layer = 0; layer < 2; ++layer)
          load_weight_blocks(it, layer ? &g.tmap2 : &a.tmap, layer ? nb2 : nb1, layer ? kc2 : kc1, base, L.wring, SW,
                             ctl.w_full, ctl.w_empty);
    }
  } else {
    // ================= MMA + epilogues: warpgroup wg, warp w4 of it holds rows 16 w4 .. +15 of the tile ======
    const unsigned mw = warp - kFp2ProWarps, wg = mw >> 2, w4 = mw & 3u;
    const int frag_row = static_cast<int>(16 * w4 + (lane >> 2));
    const uint32_t h_s = base + L.h;
    int ita = 0, itw = 0;
    float d[64];
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const long long p0 = static_cast<long long>(tile) * kFp2BM;
      // ---- layer 1 -> H tile, one pass over the A chunks per pair of column blocks
      for (int pp = 0; pp < nb1; pp += 2) {
        const int nb = pp + static_cast<int>(wg);
        fp2_layer1_block(d, base + L.aring, base + L.wring, SA, SW, ita, itw + static_cast<int>(wg), kc1, ctl, lane);
        ita += kc1;
        itw += 2 * kc1;
        // both warpgroups have finished the previous tile's layer 2 (its reads of H)
        if (pp == 0) named_bar_sync(1, 2 * 128);
        // H[row, c] = tf32(relu(acc + b1[c])): the epilogue of mlp_layer_kernel with RELU | ROUND_OUT
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int c = 128 * nb + 8 * jj + 2 * static_cast<int>(lane & 3u);
          const float b0 = __ldg(a.bias + c), b1 = __ldg(a.bias + c + 1);
          const uint32_t off = static_cast<uint32_t>(c >> 5) * kFp2AStageBytes + static_cast<uint32_t>(frag_row) * 128u +
                               ((static_cast<uint32_t>(((c & 31) >> 2) ^ (frag_row & 7))) << 4) + (c & 3) * 4u;
          asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(h_s + off), "f"(to_tf32(fmaxf(d[4 * jj] + b0, 0.f))),
                       "f"(to_tf32(fmaxf(d[4 * jj + 1] + b1, 0.f)))
                       : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(h_s + off + 8u * 128u), "f"(to_tf32(fmaxf(d[4 * jj + 2] + b0, 0.f))),
                       "f"(to_tf32(fmaxf(d[4 * jj + 3] + b1, 0.f)))
                       : "memory");
        }
      }
      fence_proxy_async_smem();   // generic-proxy stores of H -> visible to the tensor core
      named_bar_sync(1, 2 * 128); // every block of H is written
      // ---- layer 2 from the H tile: out = relu(acc + b2) [tf32], the epilogue of pvn3d_mlp_dense with RELU
      const long long r0 = p0 + frag_row;
      for (int pp = 0; pp < nb2; pp += 2) {
        const int cnt = sa2w_pair_blocks(nb2, pp);
        if (static_cast<int>(wg) < cnt) {
          const int nb = pp + static_cast<int>(wg);
          sa2w_block(d, h_s, base + L.wring, SW, itw + static_cast<int>(wg), cnt, kc2, ctl.w_full, ctl.w_empty, nullptr, 0u,
                     false, lane);
          // a quad of lanes writes 32 contiguous bytes of a row: whole sectors
          float *o = a.out + r0 * a.ldo + a.col0 + 128 * nb + 2 * static_cast<int>(lane & 3u);
          const bool on0 = r0 < a.rows, on1 = r0 + 8 < a.rows;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int c = 128 * nb + 8 * jj + 2 * static_cast<int>(lane & 3u);
            const float b0 = __ldg(g.bias2 + c), b1 = __ldg(g.bias2 + c + 1);
            float2 v0 = make_float2(fmaxf(d[4 * jj] + b0, 0.f), fmaxf(d[4 * jj + 1] + b1, 0.f));
            float2 v1 = make_float2(fmaxf(d[4 * jj + 2] + b0, 0.f), fmaxf(d[4 * jj + 3] + b1, 0.f));
            if (a.round_out) {
              v0.x = to_tf32(v0.x); v0.y = to_tf32(v0.y); v1.x = to_tf32(v1.x); v1.y = to_tf32(v1.y);
            }
            if (on0) *reinterpret_cast<float2 *>(o + 8 * jj) = v0;
            if (on1) *reinterpret_cast<float2 *>(o + 8 * static_cast<size_t>(a.ldo) + 8 * jj) = v1;
          }
        }
        itw += kc2 * cnt;
      }
    }
  }
}

// pvn3d_mlp_fp2's ring stages for a module (A ring, weight ring); false: the module is not covered -- a first layer of
// other than 256 or 512 columns, a second layer not a multiple of 128 columns, a layer-2 K other than the layer-1
// width, or H + three A stages + four weight stages beyond the shared memory of a block
bool fp2_stages(int k1_pad, int n1_pad, int k2_pad, int n2_pad, int *a_stages, int *w_stages) {
  if ((n1_pad != 256 && n1_pad != 512) || n2_pad <= 0 || n2_pad % 128 || k2_pad != n1_pad || k1_pad <= 0 || k1_pad % 32)
    return false;
  const uint32_t fixed = fp2_smem(k2_pad, 0, 0).bytes;
  const uint32_t least = 3u * kFp2AStageBytes + 4u * kFp2WStageBytes;
  if (fixed + least > static_cast<uint32_t>(kMlpSmemMax)) return false;
  // at least four weight stages -- with three, each warpgroup has one chunk of look-ahead and the ring's round trip
  // stalls it (N1 = 512 beside the 128 KB H tile: 3 A + 4 W stages, not 5 A + 3 W) -- then the A ring, then the rest
  const uint32_t avail = static_cast<uint32_t>(kMlpSmemMax) - fixed;
  const int sa = std::min<int>(kFp2MaxStages, static_cast<int>((avail - 4u * kFp2WStageBytes) / kFp2AStageBytes));
  const int sw = std::min<int>(kFp2MaxStages, static_cast<int>((avail - static_cast<uint32_t>(sa) * kFp2AStageBytes) / kFp2WStageBytes));
  *a_stages = sa;
  *w_stages = sw;
  return true;
}

int launch_fp2(Fp2Args &g, cudaStream_t st) {
  MlpArgs &a = g.a;
  if (a.rows <= 0) return PVN3D_OK;
  const size_t smem = fp2_smem(g.k2_pad, g.a_stages, g.w_stages).bytes;
  const long long tiles = (a.rows + kFp2BM - 1) / kFp2BM;
  const long long a_items = static_cast<long long>(a.n_pad / 256) * (a.k_pad / 32);
  const long long w_items = 2 * a_items + static_cast<long long>(g.n2_pad / 128) * (g.k2_pad / 32);
  if (tiles * w_items > 0x7fffffffll || tiles * a_items > 0x7fffffffll)
    return PVN3D_ERR_UNSUPPORTED;   // the kernel counts ring items in 32 bits
  if (!weight_tensor_map(&a.tmap, a.w, a.k_pad, a.n_pad, 128) || !weight_tensor_map(&g.tmap2, g.w2, g.k2_pad, g.n2_pad, 128))
    return PVN3D_ERR_UNSUPPORTED;
  return launch_persistent<mlp_fp2_kernel>(g, tiles, kFp2Threads, smem, a.reserve_sms, st, "mlp_fp2_kernel");
}

// =====================================================================================================
// The skip term and the second layer of a FACTORED FP module whose skip is the SA1 factor table (FP1), in ONE
// persistent kernel.
//
// As separate launches (S = W1s . table + b1, then layer 2 on relu(interpolated P + S)) S would go to HBM and
// straight back: 201 + 201 MB per 32-frame batch of 12288 points.  Here it never leaves the SM.  Per 64-row tile:
//   loader    (warp 16)     brings W_s and W2 into shared memory once (TMA), then the tile's 32-column table rows by
//                           TMA (SWIZZLE_128B: the wgmma layout) into a ring slot;
//   producers (warps 0-7)   warp w gathers K chunk w / 2 of rows 32 (w & 1).. : sum_t w_t P[idx_t] (fp32, unrounded)
//                           into the slot's K-major SWIZZLE_128B operand tile, row state in shared memory as
//                           mlp_fp2_kernel keeps it;
//   MMA       (warps 8-15)  warpgroup wg takes the slots it % 2 == wg: S = table . W_s^T (wgmma m64n128k8, the four K
//                           steps of the 32 columns) into registers, then in place over its fragment of the operand
//                           tile tf32(relu(interp + (S + b1))) (dead rows zero), fence.proxy.async, layer 2 from the
//                           tile (W2 resident, K 0..127), the slot released, relu(acc + b2) stored channel-major
//                           [b][128][n_unknown] from the fragment: the 8 rows of a lane quad are 8 consecutive points,
//                           whole 32-byte sectors of one channel.
// Every output element keeps the operands, wgmma shape, K order and epilogue arithmetic of mlp_layer_kernel for S and
// for layer 2 on the rows relu(interp + S): bit-identical to those point-major rows, transposed.
// Where the layer-2 output goes (the kernel's template parameter):
//   FPF2_OUT_CN    [b][128][n_unknown] channel-major, streaming stores: the layout Pointnet2MSG.forward returns,
//                  written from the fragment with no transposing pass;
//   FPF2_OUT_ROWS  relu(acc + b2) rounded to TF32, point-major into columns col0 .. col0+127 of rows ldo apart: a lane
//                  quad writes each 32-byte row segment (whole sectors), as mlp_fp2_kernel does.  The heads' table.
//   FPF2_OUT_ROWS_BF16  the same rows rounded to bf16 (cvt.rn: nearest even) instead of TF32, ldo and col0 in bf16
//                  elements: the heads' table at precision "bf16".  A lane quad writes 16 contiguous bytes of a row.
enum { FPF2_OUT_CN = 0, FPF2_OUT_ROWS = 1, FPF2_OUT_ROWS_BF16 = 2 };
constexpr int kFpf2BM = 64;
constexpr int kFpf2ProWarps = 8;
constexpr int kFpf2LoaderWarp = kFpf2ProWarps + kMlpMmaWarps;   // warp 16
constexpr int kFpf2Threads = (kFpf2LoaderWarp + 1) * 32;
constexpr int kFpf2MaxStages = 4;
constexpr uint32_t kFpf2AChunk = kFpf2BM * 128u;                 // one K chunk of the operand tile: 64 rows x 32 fp32
constexpr uint32_t kFpf2ABytes = 4u * kFpf2AChunk;               // the operand tile: 64 rows x K 128
constexpr uint32_t kFpf2TBytes = kFpf2BM * 128u;                 // the table rows of a tile: 64 x 32 fp32

struct FpFact2Args {
  MlpArgs a;   // PRO_FP_INTERP row fields (known_feat = P, c2 = 128, nn_idx, nn_w, n_unknown, m_known, rows), out; tmap: table
  alignas(64) CUtensorMap tmap_s, tmap_w2;
  const float *bias_s, *bias2;
};

struct FpFact2SmemCtl {
  uint64_t t_full[kFpf2MaxStages];   // the loader's arrive.expect_tx + the TMA bytes of the slot's table rows
  uint64_t a_full[kFpf2MaxStages];   // 256 arrivals: every producer thread, once its part of the operand tile is stored
  uint64_t empty[kFpf2MaxStages];    // 4 arrivals: the warps of the warpgroup that consumed the slot
  uint64_t w_full;                   // the loader's arrive.expect_tx + the TMA bytes of W_s and W2
};

// shared-memory layout behind the 1024-byte aligned base (kernel, launcher and pvn3d_mlp_fp_fact2_supported use the
// same function): [W2: 4 chunks of 128 x 128 B][W_s: 128 x 128 B][operand tiles: stages x 32 KB][table rows: stages x
// 8 KB][row states: 32 B per row of each producer warp][barriers]
struct FpFact2Smem {
  uint32_t w2, ws, a, t, rows, ctl, bytes;   // offsets from the aligned base; bytes = dynamic size incl. alignment slack
};
static inline __host__ __device__ FpFact2Smem fpf2_smem(int stages) {
  FpFact2Smem s;
  s.w2 = 0;
  s.ws = s.w2 + 4u * 128u * 128u;
  s.a = s.ws + 128u * 128u;
  s.t = s.a + static_cast<uint32_t>(stages) * kFpf2ABytes;
  s.rows = s.t + static_cast<uint32_t>(stages) * kFpf2TBytes;
  s.ctl = s.rows + kFpf2ProWarps * 32u * 32u;
  s.bytes = 1024u + s.ctl + static_cast<uint32_t>(sizeof(FpFact2SmemCtl));
  return s;
}
// ring slots pvn3d_mlp_fp_fact2 runs with (3: 209 KB); 0 if the layers are not covered (a skip layer other than K 32 ->
// 128, a second layer other than 128 -> 128)
int fpf2_stages(int ks_pad, int ns_pad, int k2_pad, int n2_pad) {
  if (ks_pad != 32 || ns_pad != 128 || k2_pad != 128 || n2_pad != 128) return 0;
  const uint32_t fixed = fpf2_smem(0).bytes;
  const int stages = std::min<int>(kFpf2MaxStages, static_cast<int>((kMlpSmemMax - fixed) / (kFpf2ABytes + kFpf2TBytes)));
  return stages >= 2 ? stages : 0;
}

template <int OUT>
__global__ void __launch_bounds__(kFpf2Threads, 1) mlp_fp_fact2_kernel(const __grid_constant__ FpFact2Args g) {
  const MlpArgs &a = g.a;
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const int S = a.stages;
  const FpFact2Smem L = fpf2_smem(S);
  FpFact2SmemCtl &ctl = *reinterpret_cast<FpFact2SmemCtl *>(mlp_smem_raw + (base - raw) + L.ctl);
  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int tiles = static_cast<int>((a.rows + kFpf2BM - 1) / kFpf2BM);   // the launcher checks tiles < 2^31

  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.t_full[s], 1);
      mbar_init(&ctl.a_full[s], kFpf2ProWarps * 32);
      mbar_init(&ctl.empty[s], 4);
    }
    mbar_init(&ctl.w_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < kFpf2ProWarps) {
    // ================= producers: warp w stages K chunk w / 2 of rows 32 (w & 1) .. +31 of every tile ============
    const int kc = static_cast<int>(warp >> 1);
    const int sub = static_cast<int>(lane & 7u), r_first = 32 * static_cast<int>(warp & 1u) + static_cast<int>(lane >> 3);
    const uint32_t rst = base + L.rows + warp * 1024u + (lane >> 3) * 32u;
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
      const int s = it % S;
      const long long p_first = static_cast<long long>(tile) * kFpf2BM + r_first;
      {
        RowState rs;
        rows_setup<PRO_FP_INTERP>(a, p_first, rs);
        __syncwarp();   // every lane is done with the previous tile's row state
        fp2_rows_store(rs, rst, static_cast<unsigned>(sub));
        __syncwarp();
      }
      mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
      // unrounded: the MMA warpgroup adds S, applies the ReLU and rounds
      interp_rows<false>(a, kc * 32 + 4 * sub, rst, r_first, sub, base + L.a + static_cast<uint32_t>(s) * kFpf2ABytes + kc * kFpf2AChunk);
      mbar_arrive(&ctl.a_full[s]);
    }
  } else if (warp == kFpf2LoaderWarp) {
    // ================= loader: the resident weights once, then every tile's table rows, in ring order ==========
    if (lane == 0) {
      mbar_expect_tx(&ctl.w_full, 5u * 128u * 128u);
      tma_load_2d(base + L.ws, &g.tmap_s, 0, 0, &ctl.w_full);
      for (int kc = 0; kc < 4; ++kc) tma_load_2d(base + L.w2 + kc * 128u * 128u, &g.tmap_w2, kc * 32, 0, &ctl.w_full);
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
        const int s = it % S;
        mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        mbar_expect_tx(&ctl.t_full[s], kFpf2TBytes);   // a ragged last tile: TMA fills the rows past the end with zeros
        tma_load_2d(base + L.t + static_cast<uint32_t>(s) * kFpf2TBytes, &a.tmap, 0, tile * kFpf2BM, &ctl.t_full[s]);
      }
    }
  } else {
    // ================= MMA + epilogue: warpgroup wg takes the slots it % 2 == wg, warp w4 rows 16 w4 .. +15 =======
    const unsigned mw = warp - kFpf2ProWarps, wg = mw >> 2, w4 = mw & 3u;
    const int frag_row = static_cast<int>(16 * w4 + (lane >> 2));
    const uint64_t ws_desc = smem_desc_sw128(base + L.ws);
    const long long n_unk = a.n_unknown;
    float d[64];
    mbar_wait(&ctl.w_full, 0u);
    int it = static_cast<int>(wg);
    for (int tile = blockIdx.x + static_cast<int>(wg) * gridDim.x; tile < tiles; tile += 2 * gridDim.x, it += 2) {
      const int s = it % S;
      const unsigned par = static_cast<unsigned>((it / S) & 1);
      const uint32_t a_s = base + L.a + static_cast<uint32_t>(s) * kFpf2ABytes;
      // ---- S = table . W_s^T: the MMA of pvn3d_mlp_dense (K 32: four k8 steps, zero columns included)
      mbar_wait(&ctl.t_full[s], par);
      {
        const uint64_t tdesc = smem_desc_sw128(base + L.t + static_cast<uint32_t>(s) * kFpf2TBytes);
        wgmma_fence();
        wgmma_chunk_tf32<128>(d, tdesc, ws_desc, false);
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(d);
      }
      // ---- the layer-2 operand in place: tf32(relu(interp + (S + b1))), one plain add, as the dense producer rounds
      const long long r0 = static_cast<long long>(tile) * kFpf2BM + frag_row;
      const bool on0 = r0 < a.rows, on1 = r0 + 8 < a.rows;
      mbar_wait(&ctl.a_full[s], par);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
        const float b0 = __ldg(g.bias_s + c), b1 = __ldg(g.bias_s + c + 1);
        const uint32_t off = frag_off(c, frag_row, kFpf2AChunk);
        float x0, x1, y0, y1;
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(x0), "=f"(x1) : "r"(a_s + off));
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(y0), "=f"(y1) : "r"(a_s + off + 8u * 128u));
        x0 = on0 ? to_tf32(fmaxf(x0 + (d[4 * j] + b0), 0.f)) : 0.f;
        x1 = on0 ? to_tf32(fmaxf(x1 + (d[4 * j + 1] + b1), 0.f)) : 0.f;
        y0 = on1 ? to_tf32(fmaxf(y0 + (d[4 * j + 2] + b0), 0.f)) : 0.f;
        y1 = on1 ? to_tf32(fmaxf(y1 + (d[4 * j + 3] + b1), 0.f)) : 0.f;
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a_s + off), "f"(x0), "f"(x1) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a_s + off + 8u * 128u), "f"(y0), "f"(y1) : "memory");
      }
      fence_proxy_async_smem();   // generic-proxy stores of the operand -> visible to the tensor core
      named_bar_sync(1 + static_cast<int>(wg), 128);
      // ---- layer 2: K 0..127 in order against the resident W2
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        const uint64_t adesc = smem_desc_sw128(a_s + static_cast<uint32_t>(kc) * kFpf2AChunk);
        const uint64_t bdesc = smem_desc_sw128(base + L.w2 + static_cast<uint32_t>(kc) * 128u * 128u);
        wgmma_chunk_tf32<128>(d, adesc, bdesc, kc > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(d);
      if (lane == 0) mbar_arrive(&ctl.empty[s]);   // the slot (operand tile and table rows) may be refilled
      if constexpr (OUT == FPF2_OUT_ROWS) {
        // ---- out[r][col0 + c] = tf32(relu(acc + b2[c])): a lane quad writes 32 contiguous bytes of a row
        float *o0 = a.out + (r0 * a.ldo + a.col0);
        float *o1 = o0 + 8 * static_cast<long long>(a.ldo);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
          const float2 bb = __ldg(reinterpret_cast<const float2 *>(g.bias2 + c));   // the launcher checks 8-byte alignment
          if (on0) stg64(o0 + c, to_tf32(fmaxf(d[4 * j] + bb.x, 0.f)), to_tf32(fmaxf(d[4 * j + 1] + bb.y, 0.f)));
          if (on1) stg64(o1 + c, to_tf32(fmaxf(d[4 * j + 2] + bb.x, 0.f)), to_tf32(fmaxf(d[4 * j + 3] + bb.y, 0.f)));
        }
      } else if constexpr (OUT == FPF2_OUT_ROWS_BF16) {
        // ---- out[r][col0 + c] = bf16(relu(acc + b2[c])): the arithmetic of FPF2_OUT_ROWS, one bf16x2 per lane and row
        uint16_t *o0 = reinterpret_cast<uint16_t *>(a.out) + (r0 * a.ldo + a.col0);
        uint16_t *o1 = o0 + 8 * static_cast<long long>(a.ldo);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
          const float2 bb = __ldg(reinterpret_cast<const float2 *>(g.bias2 + c));
          if (on0) stg32(o0 + c, pack_bf16x2(fmaxf(d[4 * j] + bb.x, 0.f), fmaxf(d[4 * j + 1] + bb.y, 0.f)));
          if (on1) stg32(o1 + c, pack_bf16x2(fmaxf(d[4 * j + 2] + bb.x, 0.f), fmaxf(d[4 * j + 3] + bb.y, 0.f)));
        }
      } else {
        // ---- out[b][c][i] = relu(acc + b2[c]): a lane quad's rows are 8 consecutive points of one channel
        const long long fb0 = r0 / n_unk, fb1 = (r0 + 8) / n_unk;
        float *o0 = a.out + fb0 * 128 * n_unk + (r0 - fb0 * n_unk);
        float *o1 = a.out + fb1 * 128 * n_unk + (r0 + 8 - fb1 * n_unk);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
          const float b0 = __ldg(g.bias2 + c), b1 = __ldg(g.bias2 + c + 1);
          if (on0) {
            stg_stream(o0 + c * n_unk, fmaxf(d[4 * j] + b0, 0.f));
            stg_stream(o0 + (c + 1) * n_unk, fmaxf(d[4 * j + 1] + b1, 0.f));
          }
          if (on1) {
            stg_stream(o1 + c * n_unk, fmaxf(d[4 * j + 2] + b0, 0.f));
            stg_stream(o1 + (c + 1) * n_unk, fmaxf(d[4 * j + 3] + b1, 0.f));
          }
        }
      }
    }
  }
}

template <int OUT>
int launch_fp_fact2(FpFact2Args &g, const float *table, const float *ws, const float *w2, cudaStream_t st) {
  MlpArgs &a = g.a;
  if (a.rows <= 0) return PVN3D_OK;
  const size_t smem = fpf2_smem(a.stages).bytes;
  const long long tiles = (a.rows + kFpf2BM - 1) / kFpf2BM;
  // the kernel counts tiles and ring items in 32 bits; TMA addresses table rows with a 32-bit coordinate
  if (tiles * kFpf2BM > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  if (!weight_tensor_map(&a.tmap, table, 32, static_cast<int>(a.rows), kFpf2BM) ||
      !weight_tensor_map(&g.tmap_s, ws, 32, 128, 128) || !weight_tensor_map(&g.tmap_w2, w2, 128, 128, 128))
    return PVN3D_ERR_UNSUPPORTED;
  return launch_persistent<mlp_fp_fact2_kernel<OUT>>(g, tiles, kFpf2Threads, smem, a.reserve_sms, st, "mlp_fp_fact2_kernel");
}

// =====================================================================================================
// The full-resolution tail of PVN3D's CNN evaluated ONLY at the sampled pixels, in ONE persistent kernel.
//
// Modified_PSPNet ends with up_3 = bilinear x2 (align_corners) -> Conv2d(64,64,3,pad 1) -> BatchNorm -> PReLU and
// final = Conv2d(64,128,1), both at H x W = 2h x 2w, and PVN3D.forward keeps N of the H*W embedding columns (4 % at
// 12288 of 480 x 640).  Up to the PReLU every step is linear per pixel, so row r = f * n + p of the heads' table is
//   out[r] = tf32(W2 . prelu(W1 . taps + b1) + b2),   taps[(3 (dy+1) + (dx+1)) * 64 + c] = up(x)[f][c][y+dy][x+dx]
// with (y, x) = divmod(choose[r], W), up() the align_corners bilinear sample of the half-resolution map (zero outside
// [0,H) x [0,W): the conv's padding applies to the up-sampled map) and W1 the 3x3 conv with the BN folded, K tap-major.
// Per 128-row tile:
//   loader    (warp 16)     brings W2 into shared memory once, then streams W1's 18 K chunks (64 x 32 fp32 = 8 KB, TMA,
//                           SWIZZLE_128B) into the ring slot of each chunk.  Streamed, not resident: W1 is 144 KB, which
//                           beside W2 (32 KB) and H would leave two A stages; the stream is 144 KB of L2 reads per 128
//                           rows, under the 1.1 MB the same rows gather, and leaves room for a six-deep ring;
//   producers (warps 0-7)   group q = warp / 4 stages the chunks it % 2 == q, warp w rows 32 (w & 3)..: K chunk kc is
//                           channels 32 (kc & 1).. of tap kc / 2, the bilinear combination of one contiguous 128-byte
//                           run of each of four source pixels of the channels-last map, rounded to TF32.  The source
//                           rows / columns and weights of a row's three tap rows and three tap columns are computed
//                           once per tile and kept in shared memory (16 words per row);
//   MMA       (warps 8-15)  warpgroup wg holds rows 64 wg.. : layer 1 (wgmma m64n64k8, 72 K steps) into registers,
//                           tf32(prelu(acc + b1)) into its rows of the K-major SWIZZLE_128B H tile, fence.proxy.async,
//                           layer 2 (m64n128k8, 8 K steps) against the resident W2, tf32(acc + b2) (OUT_BF16: rounded
//                           to bf16 instead) stored a lane quad per row segment as mlp_fp_fact2_kernel<FPF2_OUT_ROWS>.
// The bilinear index and weight are exact integer arithmetic: i0 = t (h-1) div (H-1), lambda = (t (h-1) mod (H-1)) /
// (H-1) correctly rounded (torch multiplies by an fp32 scale: the same sample to ~1e-7 * h in lambda).
// A choose index outside [0, H*W) gives a NaN row: its operand row is NaN and both layers carry it.
constexpr int kPspBM = 128;
constexpr int kPspProWarps = 8;
constexpr int kPspLoaderWarp = kPspProWarps + kMlpMmaWarps;   // warp 16
constexpr int kPspThreads = (kPspLoaderWarp + 1) * 32;
constexpr int kPspC = 64;                    // channels of the half-resolution map and of up_3
constexpr int kPspKc1 = 9 * kPspC / 32;      // K chunks of layer 1: two per tap
constexpr int kPspN2 = 128;                  // the embedding width
constexpr int kPspMaxStages = 6;
constexpr uint32_t kPspAStage = kPspBM * 128u;           // one K chunk of the operand tile: 128 rows x 32 fp32
constexpr uint32_t kPspWStage = kPspC * 128u;            // one K chunk of W1: 64 rows x 32 fp32
constexpr uint32_t kPspStage = kPspAStage + kPspWStage;
constexpr uint32_t kPspRowBytes = 64u;                   // row state, words: [0..2] (f h + i0) w of the tap rows dy = -1, 0, 1,
                                                         // [3..5] the same for i1, [6..8] lambda_y, [9..11] j0 of the tap
                                                         // columns, [12..14] lambda_x, [15] mask
constexpr unsigned kPspNanRow = 64u;                     // mask: bits 0-2 tap row inside the image, 3-5 tap column, 6 NaN row

struct PspTailArgs {
  alignas(64) CUtensorMap tmap_w1, tmap_w2;
  const float *x;            // [b][h][w][64] channels-last
  const long long *choose;   // [b][1][n]
  const float *bias1, *slope, *bias2;
  void *out;
  long long rows;            // b * n
  int n, h, w, ldo, col0, stages, reserve_sms;
};

struct PspTailSmemCtl {
  uint64_t full[kPspMaxStages];    // 128 producer threads + the loader's arrive.expect_tx + the TMA bytes of the W1 chunk
  uint64_t empty[kPspMaxStages];   // 8 arrivals: the MMA warps
  uint64_t w2_full;
};

// shared-memory layout behind the 1024-byte aligned base (kernel, launcher and pvn3d_psp_tail_supported use the same
// function): [W2: 2 chunks of 128 x 128 B][H: 2 chunks of 128 x 128 B][ring: stages x (16 KB A + 8 KB W1)][row states:
// 64 B per row of each producer warp][barriers]
struct PspTailSmem {
  uint32_t w2, h, ring, rows, ctl, bytes;   // offsets from the aligned base; bytes = dynamic size incl. alignment slack
};
static inline __host__ __device__ PspTailSmem psp_tail_smem(int stages) {
  PspTailSmem s;
  s.w2 = 0;
  s.h = s.w2 + 2u * kPspN2 * 128u;
  s.ring = s.h + 2u * kPspAStage;
  s.rows = s.ring + static_cast<uint32_t>(stages) * kPspStage;
  s.ctl = s.rows + kPspProWarps * 32u * kPspRowBytes;
  s.bytes = 1024u + s.ctl + static_cast<uint32_t>(sizeof(PspTailSmemCtl));
  return s;
}
// ring slots pvn3d_psp_tail_rows runs with (6: 225 KB); 0 if the layers are not 576 -> 64 and 64 -> 128
int psp_tail_stages(int k1_pad, int n1_pad, int k2_pad, int n2_pad) {
  if (k1_pad != 9 * kPspC || n1_pad != kPspC || k2_pad != kPspC || n2_pad != kPspN2) return 0;
  const uint32_t fixed = psp_tail_smem(0).bytes;
  const int stages = std::min<int>(kPspMaxStages, static_cast<int>((kMlpSmemMax - fixed) / kPspStage));
  return stages >= 3 ? stages : 0;
}

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// source index and weight of up-sampled coordinate t (0 <= t < 2 n_src) under align_corners: exact floor and remainder
__device__ __forceinline__ void psp_axis(int t, int n_src, int &i0, float &lambda) {
  const int den = 2 * n_src - 1, num = t * (n_src - 1);
  i0 = num / den;
  lambda = __fdiv_rn(static_cast<float>(num - i0 * den), static_cast<float>(den));
}

// the row state of point p (rows past the end: every tap dead, the operand row is zero)
__device__ __forceinline__ void psp_row_setup(const PspTailArgs &g, long long p, uint32_t dst) {
  int yo0[3] = {0, 0, 0}, yo1[3] = {0, 0, 0}, xo[3] = {0, 0, 0};
  float ly[3] = {0.f, 0.f, 0.f}, lx[3] = {0.f, 0.f, 0.f};
  unsigned mask = 0u;
  if (p < g.rows) {
    const long long c = __ldg(g.choose + p);
    const int H = 2 * g.h, W = 2 * g.w;
    if (c < 0 || c >= static_cast<long long>(H) * W) {
      mask = kPspNanRow;
    } else {
      const int f = static_cast<int>(p / g.n), y = static_cast<int>(c / W), x = static_cast<int>(c - static_cast<long long>(y) * W);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const int ty = y + d - 1, tx = x + d - 1;
        if (ty >= 0 && ty < H) {
          int i0;
          psp_axis(ty, g.h, i0, ly[d]);
          yo0[d] = (f * g.h + i0) * g.w;
          yo1[d] = (f * g.h + min(i0 + 1, g.h - 1)) * g.w;
          mask |= 1u << d;
        }
        if (tx >= 0 && tx < W) {
          psp_axis(tx, g.w, xo[d], lx[d]);
          mask |= 8u << d;
        }
      }
    }
  }
  sts128(dst, __int_as_float(yo0[0]), __int_as_float(yo0[1]), __int_as_float(yo0[2]), __int_as_float(yo1[0]));
  sts128(dst + 16u, __int_as_float(yo1[1]), __int_as_float(yo1[2]), ly[0], ly[1]);
  sts128(dst + 32u, ly[2], __int_as_float(xo[0]), __int_as_float(xo[1]), __int_as_float(xo[2]));
  sts128(dst + 48u, lx[0], lx[1], lx[2], __uint_as_float(mask));
}

// K chunk kc of the producer's 8 rows: tf32 of tap kc / 2, channels 32 (kc & 1) + 4 sub .. +3.  `rst` is the state of the
// thread's first row; its rows are 4 apart.
__device__ __forceinline__ void psp_stage_chunk(const PspTailArgs &g, uint32_t rst, int r_first, int sub, int kc, uint32_t sa) {
  const int tap = kc >> 1, dy = tap / 3, dx = tap - 3 * dy;
  const unsigned need = (1u << dy) | (8u << dx);
  const float *xc = g.x + (kc & 1) * 32 + 4 * sub;
  const float nan = __int_as_float(0x7fc00000);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {  // two halves: 16 LDG.128 in flight each
    float4 v00[4], v01[4], v10[4], v11[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const uint32_t rs = rst + 4u * kPspRowBytes * (hh * 4 + jj);
      v00[jj] = v01[jj] = v10[jj] = v11[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
      if ((lds32(rs + 60u) & need) == need) {
        const int y0 = static_cast<int>(lds32(rs + 4u * dy)), y1 = static_cast<int>(lds32(rs + 12u + 4u * dy));
        const int x0 = static_cast<int>(lds32(rs + 36u + 4u * dx)), x1 = min(x0 + 1, g.w - 1);
        v00[jj] = ldg128(xc + static_cast<size_t>(y0 + x0) * kPspC);
        v01[jj] = ldg128(xc + static_cast<size_t>(y0 + x1) * kPspC);
        v10[jj] = ldg128(xc + static_cast<size_t>(y1 + x0) * kPspC);
        v11[jj] = ldg128(xc + static_cast<size_t>(y1 + x1) * kPspC);
      }
    }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = hh * 4 + jj;
      const uint32_t rs = rst + 4u * kPspRowBytes * j;
      const float ly = __uint_as_float(lds32(rs + 24u + 4u * dy)), lx = __uint_as_float(lds32(rs + 48u + 4u * dx));
      const float my = 1.f - ly, mx = 1.f - lx;
      float4 v;
      v.x = __fmaf_rn(ly, __fmaf_rn(lx, v11[jj].x, mx * v10[jj].x), my * __fmaf_rn(lx, v01[jj].x, mx * v00[jj].x));
      v.y = __fmaf_rn(ly, __fmaf_rn(lx, v11[jj].y, mx * v10[jj].y), my * __fmaf_rn(lx, v01[jj].y, mx * v00[jj].y));
      v.z = __fmaf_rn(ly, __fmaf_rn(lx, v11[jj].z, mx * v10[jj].z), my * __fmaf_rn(lx, v01[jj].z, mx * v00[jj].z));
      v.w = __fmaf_rn(ly, __fmaf_rn(lx, v11[jj].w, mx * v10[jj].w), my * __fmaf_rn(lx, v01[jj].w, mx * v00[jj].w));
      if (lds32(rs + 60u) & kPspNanRow) v = make_float4(nan, nan, nan, nan);
      sts_tf32(sa + sw128_off(r_first + 4 * j, sub), v);
    }
  }
}

template <bool OUT_BF16>
__global__ void __launch_bounds__(kPspThreads, 1) psp_tail_kernel(const __grid_constant__ PspTailArgs g) {
  extern __shared__ unsigned char mlp_smem_raw[];
  const uint32_t raw = smem_u32(mlp_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B atoms are 8 rows x 128 B
  const int S = g.stages;
  const PspTailSmem L = psp_tail_smem(S);
  PspTailSmemCtl &ctl = *reinterpret_cast<PspTailSmemCtl *>(mlp_smem_raw + (base - raw) + L.ctl);
  const int t = threadIdx.x;
  const unsigned warp = t >> 5, lane = t & 31u;
  const int tiles = static_cast<int>((g.rows + kPspBM - 1) / kPspBM);   // the launcher checks the 32-bit counts

  if (t == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&ctl.full[s], 128 + 1);
      mbar_init(&ctl.empty[s], kMlpMmaWarps);
    }
    mbar_init(&ctl.w2_full, 1);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < kPspProWarps) {
    // ================= producers: group q = warp / 4 stages the items it % 2 == q, warp w rows 32 (w & 3).. ======
    const unsigned grp = warp >> 2;
    const int sub = static_cast<int>(lane & 7u), r_first = 32 * static_cast<int>(warp & 3u) + static_cast<int>(lane >> 3);
    const uint32_t rst_w = base + L.rows + warp * 32u * kPspRowBytes;
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      __syncwarp();   // every lane is done with the previous tile's row state
      psp_row_setup(g, static_cast<long long>(tile) * kPspBM + 32 * static_cast<int>(warp & 3u) + static_cast<int>(lane),
                    rst_w + lane * kPspRowBytes);
      __syncwarp();
      for (int kc = 0; kc < kPspKc1; ++kc, ++it) {
        if (static_cast<unsigned>(it & 1) != grp) continue;
        const int s = it % S;
        mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
        psp_stage_chunk(g, rst_w + (lane >> 3) * kPspRowBytes, r_first, sub, kc, base + L.ring + static_cast<uint32_t>(s) * kPspStage);
        fence_proxy_async_smem();
        mbar_arrive(&ctl.full[s]);
      }
    }
  } else if (warp == kPspLoaderWarp) {
    // ================= loader: W2 once, then the W1 chunk of every item, in ring order ==========================
    if (lane == 0) {
      mbar_expect_tx(&ctl.w2_full, 2u * kPspN2 * 128u);
      for (int kc = 0; kc < 2; ++kc) tma_load_2d(base + L.w2 + kc * kPspN2 * 128u, &g.tmap_w2, kc * 32, 0, &ctl.w2_full);
      int it = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x)
        for (int kc = 0; kc < kPspKc1; ++kc, ++it) {
          const int s = it % S;
          mbar_wait(&ctl.empty[s], static_cast<unsigned>(((it / S) & 1) ^ 1));
          mbar_expect_tx(&ctl.full[s], kPspWStage);
          tma_load_2d(base + L.ring + static_cast<uint32_t>(s) * kPspStage + kPspAStage, &g.tmap_w1, kc * 32, 0, &ctl.full[s]);
        }
    }
  } else {
    // ================= MMA + epilogues: warpgroup wg, warp w4 of it holds rows 64 wg + 16 w4 .. +15 of the tile ===
    const unsigned mw = warp - kPspProWarps, wg = mw >> 2, w4 = mw & 3u;
    const int frag_row = static_cast<int>(64 * wg + 16 * w4 + (lane >> 2));
    const uint32_t h_s = base + L.h;
    mbar_wait(&ctl.w2_full, 0u);
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      // ---- layer 1: the 18 K chunks of the ring into registers, each slot released once its MMAs have retired
      float d1[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d1[i] = 0.f;
      int prev = -1;
      for (int kc = 0; kc < kPspKc1; ++kc, ++it) {
        const int s = it % S;
        mbar_wait(&ctl.full[s], static_cast<unsigned>((it / S) & 1));
        fence_proxy_async_smem();
        const uint32_t slot = base + L.ring + static_cast<uint32_t>(s) * kPspStage;
        const uint64_t adesc = smem_desc_sw128(slot + wg * 64u * 128u), bdesc = smem_desc_sw128(slot + kPspAStage);
        wgmma_fence();
        wgmma_chunk_tf32<64>(d1, adesc, bdesc, kc > 0);
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&ctl.empty[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>();
      acc_fence(d1);
      if (lane == 0) mbar_arrive(&ctl.empty[prev]);
      // ---- H[row, c] = tf32(prelu(acc + b1[c])) into the warpgroup's rows, once its warps are past the previous
      //      tile's layer 2 (the reads of those rows)
      named_bar_sync(1 + static_cast<int>(wg), 128);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
        const float b0 = __ldg(g.bias1 + c), b1 = __ldg(g.bias1 + c + 1), s0 = __ldg(g.slope + c), s1 = __ldg(g.slope + c + 1);
        const uint32_t off = static_cast<uint32_t>(c >> 5) * kPspAStage + static_cast<uint32_t>(frag_row) * 128u +
                             ((static_cast<uint32_t>(((c & 31) >> 2) ^ (frag_row & 7))) << 4) + (c & 3) * 4u;
        float x0 = d1[4 * j] + b0, x1 = d1[4 * j + 1] + b1, y0 = d1[4 * j + 2] + b0, y1 = d1[4 * j + 3] + b1;
        x0 = x0 >= 0.f ? x0 : s0 * x0;
        x1 = x1 >= 0.f ? x1 : s1 * x1;
        y0 = y0 >= 0.f ? y0 : s0 * y0;
        y1 = y1 >= 0.f ? y1 : s1 * y1;
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(h_s + off), "f"(to_tf32(x0)), "f"(to_tf32(x1)) : "memory");
        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(h_s + off + 8u * 128u), "f"(to_tf32(y0)), "f"(to_tf32(y1)) : "memory");
      }
      fence_proxy_async_smem();   // generic-proxy stores of H -> visible to the tensor core
      named_bar_sync(1 + static_cast<int>(wg), 128);
      // ---- layer 2: K 0..63 in order against the resident W2
      float d[64];
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 2; ++kc) {
        const uint64_t adesc = smem_desc_sw128(h_s + static_cast<uint32_t>(kc) * kPspAStage + wg * 64u * 128u);
        const uint64_t bdesc = smem_desc_sw128(base + L.w2 + static_cast<uint32_t>(kc) * kPspN2 * 128u);
        wgmma_chunk_tf32<128>(d, adesc, bdesc, kc > 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(d);
      // ---- out[r][col0 + c] = tf32(acc + b2[c]) (final has no activation): a lane quad writes one row segment
      const long long r0 = static_cast<long long>(tile) * kPspBM + frag_row;
      const bool on0 = r0 < g.rows, on1 = r0 + 8 < g.rows;
      if constexpr (OUT_BF16) {
        uint16_t *o0 = static_cast<uint16_t *>(g.out) + (r0 * g.ldo + g.col0);
        uint16_t *o1 = o0 + 8 * static_cast<long long>(g.ldo);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
          const float2 bb = __ldg(reinterpret_cast<const float2 *>(g.bias2 + c));   // the launcher checks 8-byte alignment
          if (on0) stg32(o0 + c, pack_bf16x2(d[4 * j] + bb.x, d[4 * j + 1] + bb.y));
          if (on1) stg32(o1 + c, pack_bf16x2(d[4 * j + 2] + bb.x, d[4 * j + 3] + bb.y));
        }
      } else {
        float *o0 = static_cast<float *>(g.out) + (r0 * g.ldo + g.col0);
        float *o1 = o0 + 8 * static_cast<long long>(g.ldo);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = 8 * j + 2 * static_cast<int>(lane & 3u);
          const float2 bb = __ldg(reinterpret_cast<const float2 *>(g.bias2 + c));
          if (on0) stg64(o0 + c, to_tf32(d[4 * j] + bb.x), to_tf32(d[4 * j + 1] + bb.y));
          if (on1) stg64(o1 + c, to_tf32(d[4 * j + 2] + bb.x), to_tf32(d[4 * j + 3] + bb.y));
        }
      }
    }
  }
}

template <bool OUT_BF16>
int launch_psp_tail(PspTailArgs &g, const float *w1, const float *w2, cudaStream_t st) {
  if (g.rows <= 0) return PVN3D_OK;
  const size_t smem = psp_tail_smem(g.stages).bytes;
  const long long tiles = (g.rows + kPspBM - 1) / kPspBM;
  if (tiles * kPspKc1 > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;   // the kernel counts ring items in 32 bits
  if (!weight_tensor_map(&g.tmap_w1, w1, 9 * kPspC, kPspC, kPspC) || !weight_tensor_map(&g.tmap_w2, w2, kPspC, kPspN2, kPspN2))
    return PVN3D_ERR_UNSUPPORTED;
  return launch_persistent<psp_tail_kernel<OUT_BF16>>(g, tiles, kPspThreads, smem, g.reserve_sms, st, "psp_tail_kernel");
}

// ---- factored first layer of an SA scale -------------------------------------------------------------
// table row j = [ tf32(f_j) (C) | hi(x_j) (3) | lo(x_j) (3) | 0.. ]: x = hi + lo with hi = tf32(x), lo = tf32(x - hi),
// so that a TF32 GEMM against [W_f | W_x | W_x] evaluates W_x . x to ~2^-21 relative (the coordinates are
// ~1 m and their DIFFERENCES ~1 cm: a single TF32 rounding of x would cost 10 % of the difference)
__global__ void sa_factor_table_kernel(const float *__restrict__ xyz, const float *__restrict__ feat, int ldf,
                                       int c_feat, long long rows, int k_pad, float *__restrict__ out) {
  // one 16-byte group of a row per thread (k_pad / 4 threads per row): 128-byte stores, 4+ rows per warp
  const int qpr = k_pad >> 2;
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long p = g / qpr;
  if (p >= rows) return;
  const int c0 = static_cast<int>(g - p * qpr) * 4;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int c = c0 + e;
    float r = 0.f;
    if (c < c_feat) {
      r = to_tf32(__ldg(feat + p * ldf + c));
    } else if (c < c_feat + 6) {
      const int d = (c - c_feat) % 3;
      const float x = __ldg(xyz + p * 3 + d);
      const float hi = to_tf32(x);
      r = c < c_feat + 3 ? hi : to_tf32(x - hi);
    }
    v[e] = r;
  }
  *reinterpret_cast<float4 *>(out + p * k_pad + c0) = make_float4(v[0], v[1], v[2], v[3]);
}
// V[i, n] = sum_d Wx[n, d] * c_i[d] - bias[n]   (fp32 FMAs; Wx = the TF32-rounded xyz columns of W1)
__global__ void sa_centre_term_kernel(const float *__restrict__ centres, const float *__restrict__ wx,
                                      const float *__restrict__ bias, long long rows, int n_pad,
                                      float *__restrict__ out) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.y + threadIdx.y;
  if (p >= rows) return;
  const float cx = __ldg(centres + p * 3), cy = __ldg(centres + p * 3 + 1), cz = __ldg(centres + p * 3 + 2);
  for (int n = threadIdx.x; n < n_pad; n += blockDim.x) {
    const float w0 = __ldg(wx + n * 3), w1 = __ldg(wx + n * 3 + 1), w2 = __ldg(wx + n * 3 + 2);
    out[p * n_pad + n] = __fmaf_rn(w2, cz, __fmaf_rn(w1, cy, w0 * cx)) - __ldg(bias + n);
  }
}

// inverse-distance weights of PointnetFPModule.forward (pointnet2_modules.py:183-186) + 3-NN indices
__global__ void nn_weights_kernel(const float *__restrict__ dist2, long long rows,
                                  float *__restrict__ w) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= rows) return;
  const float r1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(dist2[p * 3 + 0]), 1e-8f));
  const float r2 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(dist2[p * 3 + 1]), 1e-8f));
  const float r3 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(dist2[p * 3 + 2]), 1e-8f));
  const float norm = __fadd_rn(__fadd_rn(r1, r2), r3);
  w[p * 3 + 0] = __fdiv_rn(r1, norm);
  w[p * 3 + 1] = __fdiv_rn(r2, norm);
  w[p * 3 + 2] = __fdiv_rn(r3, norm);
}

// ---- the CNN embedding at the sampled pixels, point-major (PVN3D.forward's torch.gather, pvn3d.py:288-292) ------------
// out[r][col0 + ch] = tf32(emb[f][ch][choose[r]]) for the rows r = f * n + p.  A CTA takes kGatherPts consecutive rows:
// lane i of every warp reads one channel of point i (the datasets' ascending `choose` puts neighbouring pixels in the
// same sectors), the values are transposed through shared memory and every row leaves in whole 16-byte groups.  An
// index outside [0, hw) writes a row of NaN: the C ABI never aborts.
constexpr int kGatherPts = 32;
constexpr int kGatherThreads = 256;
constexpr int kGatherMaxC = 256;

__global__ void __launch_bounds__(kGatherThreads) gather_pixel_rows_kernel(const float *__restrict__ emb, int c, long long hw,
                                                                           const long long *__restrict__ choose, int n,
                                                                           long long rows, float *__restrict__ out, int ldo,
                                                                           int col0) {
  __shared__ __align__(16) float tile[kGatherPts * (kGatherMaxC + 4)];   // [point][channel], rows 16-byte aligned
  const int ld = c + 4;
  const int lane = static_cast<int>(threadIdx.x & 31u), warp = static_cast<int>(threadIdx.x >> 5);
  const long long r0 = static_cast<long long>(blockIdx.x) * kGatherPts;
  const long long r = r0 + lane;
  const float *src = nullptr;
  if (r < rows) {
    const long long idx = __ldg(choose + r);
    if (idx >= 0 && idx < hw) src = emb + (r / n) * c * hw + idx;
  }
#pragma unroll 4
  for (int ch = warp; ch < c; ch += kGatherThreads / 32)
    tile[lane * ld + ch] = src ? to_tf32(__ldg(src + ch * hw)) : __int_as_float(0x7fc00000);
  __syncthreads();
  const int q4 = c >> 2;
  for (int i = static_cast<int>(threadIdx.x); i < kGatherPts * q4; i += kGatherThreads) {
    const int pt = i / q4, q = i - pt * q4;
    if (r0 + pt < rows)
      *reinterpret_cast<float4 *>(out + (r0 + pt) * ldo + col0 + 4 * q) = *reinterpret_cast<const float4 *>(tile + pt * ld + 4 * q);
  }
}

// the same rows in bf16 (the heads' table at precision "bf16"): out[r][col0 + ch] = bf16(emb[f][ch][choose[r]]), from an
// fp32 embedding (round to nearest even, as torch's .to(bfloat16)) or a bf16 one (copied).  Rows leave in 16-byte groups
// of 8 channels; an index outside [0, hw) writes a row of NaN.
__device__ __forceinline__ uint16_t bf16_bits(float x) { return static_cast<uint16_t>(pack_bf16x2(x, 0.f) & 0xffffu); }
__device__ __forceinline__ uint16_t bf16_bits(uint16_t x) { return x; }

template <typename T>
__global__ void __launch_bounds__(kGatherThreads) gather_pixel_rows_bf16_kernel(const T *__restrict__ emb, int c, long long hw,
                                                                                const long long *__restrict__ choose, int n,
                                                                                long long rows, uint16_t *__restrict__ out,
                                                                                int ldo, int col0) {
  __shared__ __align__(16) uint16_t tile[kGatherPts * (kGatherMaxC + 8)];   // [point][channel], rows 16-byte aligned
  const int ld = c + 8;
  const int lane = static_cast<int>(threadIdx.x & 31u), warp = static_cast<int>(threadIdx.x >> 5);
  const long long r0 = static_cast<long long>(blockIdx.x) * kGatherPts;
  const long long r = r0 + lane;
  const T *src = nullptr;
  if (r < rows) {
    const long long idx = __ldg(choose + r);
    if (idx >= 0 && idx < hw) src = emb + (r / n) * c * hw + idx;
  }
#pragma unroll 4
  for (int ch = warp; ch < c; ch += kGatherThreads / 32)
    tile[lane * ld + ch] = src ? bf16_bits(__ldg(src + ch * hw)) : static_cast<uint16_t>(0x7fc0u);
  __syncthreads();
  const int q8 = c >> 3;
  for (int i = static_cast<int>(threadIdx.x); i < kGatherPts * q8; i += kGatherThreads) {
    const int pt = i / q8, q = i - pt * q8;
    if (r0 + pt < rows)
      *reinterpret_cast<uint4 *>(out + (r0 + pt) * ldo + col0 + 8 * q) = *reinterpret_cast<const uint4 *>(tile + pt * ld + 8 * q);
  }
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

// the shapes a pair of layers must have, `first` feeding `second`: K a positive multiple of 32, N one of 16, and the
// second layer's K covering the first one's N
static bool layer_pair_ok(const pvn3d_mlp_layer_t *first, const pvn3d_mlp_layer_t *second) {
  return first && second && first->k_pad > 0 && first->k_pad % 32 == 0 && first->n_pad > 0 && first->n_pad % 16 == 0 &&
         second->k_pad >= first->n_pad && second->k_pad % 32 == 0 && second->n_pad > 0 && second->n_pad % 16 == 0;
}
// both pointers of a layer set, w 16-byte aligned (it is read 16 bytes at a time)
static bool layer_ptrs_ok(const pvn3d_mlp_layer_t *l) {
  return l->w && l->bias && !(reinterpret_cast<uintptr_t>(l->w) & 15u);
}

// the operand checks and kernel arguments of a layer on relu(U[idx] - V), the second of a factored SA scale
// (pvn3d_mlp_sa_fact2, pvn3d_mlp_sa_fact2w): PVN3D_ERR_INVALID_ARG for a bad operand, then
// PVN3D_ERR_UNSUPPORTED for sizes beyond the kernels' 32-bit row arithmetic
static int sa_fact_args(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m, int ns,
                        const pvn3d_mlp_layer_t &layer, int flags, float *out, int ldo, int col0, MlpArgs &a) {
  if (!u || !v || !idx || !layer.w || !layer.bias || !out || b < 0 || n <= 0 || m < 0 || ns <= 0 || c_valid <= 0 ||
      c_valid % 4 || ldu < c_valid || ldu % 4 || layer.k_pad < c_valid || ldo % 4 || col0 % 4 ||
      (reinterpret_cast<uintptr_t>(u) & 15u) || (reinterpret_cast<uintptr_t>(v) & 15u))
    return PVN3D_ERR_INVALID_ARG;
  if (static_cast<long long>(m) * ns > 0x3fffffffll || static_cast<long long>(b) * n > 0x7fffffffll ||
      static_cast<long long>(b) * m > 0x7fffffffll)
    return PVN3D_ERR_UNSUPPORTED;
  a.w = layer.w; a.bias = layer.bias; a.k_pad = layer.k_pad; a.n_pad = layer.n_pad;
  a.rows = static_cast<long long>(b) * m * ns;
  a.feat = u; a.new_xyz = v; a.ldf = ldu; a.c_feat = c_valid; a.idx = idx;
  a.n = n; a.m = m; a.ns = ns;
  a.out = out; a.ldo = ldo; a.col0 = col0;
  a.relu = flags & PVN3D_MLP_RELU; a.round_out = (flags & PVN3D_MLP_ROUND_OUT) ? 1 : 0;
  a.reserve_sms = (flags >> 8) & 0xff;
  return PVN3D_OK;
}

// the same for a layer on [interpolated known descriptors | skip], the first of an FP module (pvn3d_mlp_fp2)
static int fp_interp_args(const float *known_feat_pm, int c2, const int *nn_idx, const float *nn_w, const float *skip_pm,
                          int lds, int c1, int b, int n_unknown, int m_known, const pvn3d_mlp_layer_t &layer, int flags,
                          float *out, int ldo, int col0, MlpArgs &a) {
  if (!known_feat_pm || !nn_idx || !nn_w || !layer.w || !layer.bias || !out || b < 0 || n_unknown < 0 || m_known <= 0 ||
      c2 <= 0 || c1 < 0 || (c1 > 0 && (!skip_pm || lds < c1)) || layer.k_pad < c2 + c1 || ldo % 4 || col0 % 4)
    return PVN3D_ERR_INVALID_ARG;
  if (static_cast<long long>(b) * m_known > 0x7fffffffll || n_unknown > 0x3fffffff) return PVN3D_ERR_UNSUPPORTED;
  a.w = layer.w; a.bias = layer.bias; a.k_pad = layer.k_pad; a.n_pad = layer.n_pad;
  a.rows = static_cast<long long>(b) * n_unknown;
  a.known_feat = known_feat_pm; a.c2 = c2; a.nn_idx = nn_idx; a.nn_w = nn_w; a.skip = skip_pm;
  a.lds = lds; a.c1 = c1; a.n_unknown = n_unknown; a.m_known = m_known;
  a.out = out; a.ldo = ldo; a.col0 = col0;
  a.relu = flags & PVN3D_MLP_RELU; a.round_out = (flags & PVN3D_MLP_ROUND_OUT) ? 1 : 0;
  a.reserve_sms = (flags >> 8) & 0xff;
  return PVN3D_OK;
}

// the argument checks and kernel arguments the three TF32 dense entry points share: PVN3D_ERR_INVALID_ARG for a bad
// operand, before any CUDA call
static int dense_args(const float *a, int lda, int a_cols, long long rows, const float *w, const float *bias, int k_pad,
                      int n_pad, int flags, float *out, int ldo, int col0, MlpArgs &m) {
  if (!a || !w || !bias || !out || lda < a_cols || a_cols < 0 || a_cols % 4 || rows < 0 || ldo % 4 || col0 % 4)
    return PVN3D_ERR_INVALID_ARG;
  m.w = w; m.bias = bias; m.rows = rows; m.k_pad = k_pad; m.n_pad = n_pad;
  m.a = a; m.lda = lda; m.a_cols = a_cols;
  m.out = out; m.ldo = ldo; m.col0 = col0;
  m.relu = flags & PVN3D_MLP_RELU; m.round_out = (flags & PVN3D_MLP_ROUND_OUT) ? 1 : 0;
  m.a_tf32 = (flags & PVN3D_MLP_A_TF32) ? 1 : 0;
  m.reserve_sms = (flags >> 8) & 0xff;
  return PVN3D_OK;
}

extern "C" int pvn3d_mlp_dense(const float *a, int lda, int a_cols, long long rows, const float *w, const float *bias,
                               int k_pad, int n_pad, int flags, float *out, int ldo, int col0, pvn3d_stream_t stream) {
  MlpArgs m{};
  const int rc = dense_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, out, ldo, col0, m);
  return rc != PVN3D_OK ? rc : launch_mlp<EPI_STORE>(m, as_stream(stream));
}

extern "C" int pvn3d_three_nn_weights(const float *dist2, long long rows, float *weight,
                                      pvn3d_stream_t stream) {
  if (!dist2 || !weight || rows < 0) return PVN3D_ERR_INVALID_ARG;
  if (rows == 0) return PVN3D_OK;
  nn_weights_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, as_stream(stream)>>>(
      dist2, rows, weight);
  return check_launch("nn_weights_kernel");
}

extern "C" int pvn3d_sa_factor_table(const float *xyz, const float *feat_pm, int ldf, int c_feat, long long rows,
                                     int k_pad, float *out, pvn3d_stream_t stream) {
  if (!xyz || !out || rows < 0 || c_feat < 0 || (c_feat > 0 && (!feat_pm || ldf < c_feat)) || k_pad < c_feat + 6 ||
      k_pad % 32)
    return PVN3D_ERR_INVALID_ARG;
  if (rows == 0) return PVN3D_OK;
  const long long groups = rows * (k_pad / 4);
  if ((groups + 255) / 256 > 0x7fffffffll || (reinterpret_cast<uintptr_t>(out) & 15u)) return PVN3D_ERR_UNSUPPORTED;
  sa_factor_table_kernel<<<static_cast<unsigned>((groups + 255) / 256), 256, 0, as_stream(stream)>>>(xyz, feat_pm, ldf, c_feat,
                                                                                                    rows, k_pad, out);
  return check_launch("sa_factor_table_kernel");
}

extern "C" int pvn3d_sa_centre_term(const float *centres, const float *wx, const float *bias, long long rows,
                                    int n_pad, float *out, pvn3d_stream_t stream) {
  if (!centres || !wx || !bias || !out || rows < 0 || n_pad <= 0 || n_pad % 4) return PVN3D_ERR_INVALID_ARG;
  if (rows == 0) return PVN3D_OK;
  const dim3 block(32, 8);
  sa_centre_term_kernel<<<static_cast<unsigned>((rows + 7) / 8), block, 0, as_stream(stream)>>>(centres, wx, bias, rows,
                                                                                               n_pad, out);
  return check_launch("sa_centre_term_kernel");
}

// the argument checks and kernel arguments pvn3d_mlp_sa_fact2 (G = Sa2Args) and pvn3d_mlp_sa_fact2w (Sa2wArgs) share
template <typename G>
static int sa_fact2_args(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n, int m, int ns,
                         const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int flags, int pool, float *out,
                         int ldo, int col0, G &g) {
  if (!layer_pair_ok(layer2, layer3) || !layer_ptrs_ok(layer2) || !layer_ptrs_ok(layer3) || pool != ns)
    return PVN3D_ERR_INVALID_ARG;
  const int rc = sa_fact_args(u, v, ldu, c_valid, idx, b, n, m, ns, *layer2, flags, out, ldo, col0, g.a);
  if (rc != PVN3D_OK) return rc;
  g.a.relu = 1;
  g.a.pool = ns;
  g.w3 = layer3->w; g.bias3 = layer3->bias; g.k3_pad = layer3->k_pad; g.n3_pad = layer3->n_pad;
  return PVN3D_OK;
}

extern "C" int pvn3d_mlp_sa_fact2(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n,
                                  int m, int ns, const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3,
                                  int flags, int pool, float *out, int ldo, int col0, pvn3d_stream_t stream) {
  Sa2Args g{};
  const int rc = sa_fact2_args(u, v, ldu, c_valid, idx, b, n, m, ns, layer2, layer3, flags, pool, out, ldo, col0, g);
  if (rc != PVN3D_OK) return rc;
  const int stages = sa2_stages(layer2->k_pad, layer2->n_pad, layer3->k_pad, layer3->n_pad, ns);
  if (!stages) return PVN3D_ERR_UNSUPPORTED;
  switch (mma_n(layer2->n_pad)) {
    case 16: return launch_sa_fact2_n3<16>(g, stages, as_stream(stream));
    case 32: return launch_sa_fact2_n3<32>(g, stages, as_stream(stream));
    case 64: return launch_sa_fact2_n3<64>(g, stages, as_stream(stream));
    default: return launch_sa_fact2_n3<128>(g, stages, as_stream(stream));
  }
}

extern "C" int pvn3d_mlp_sa_fact2_supported(const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int ns) {
  if (!layer_pair_ok(layer2, layer3)) return 0;
  return sa2_stages(layer2->k_pad, layer2->n_pad, layer3->k_pad, layer3->n_pad, ns) ? 1 : 0;
}

extern "C" int pvn3d_mlp_sa_fact2w(const float *u, const float *v, int ldu, int c_valid, const int *idx, int b, int n,
                                   int m, int ns, const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3,
                                   int flags, int pool, float *out, int ldo, int col0, pvn3d_stream_t stream) {
  Sa2wArgs g{};
  const int rc = sa_fact2_args(u, v, ldu, c_valid, idx, b, n, m, ns, layer2, layer3, flags, pool, out, ldo, col0, g);
  if (rc != PVN3D_OK) return rc;
  const int stages = sa2w_stages(layer2->k_pad, layer2->n_pad, layer3->k_pad, layer3->n_pad, ns);
  if (!stages) return PVN3D_ERR_UNSUPPORTED;
  return launch_sa_fact2w(g, stages, as_stream(stream));
}

extern "C" int pvn3d_mlp_sa_fact2w_supported(const pvn3d_mlp_layer_t *layer2, const pvn3d_mlp_layer_t *layer3, int ns) {
  if (!layer_pair_ok(layer2, layer3)) return 0;
  return sa2w_stages(layer2->k_pad, layer2->n_pad, layer3->k_pad, layer3->n_pad, ns) ? 1 : 0;
}

extern "C" int pvn3d_mlp_fp2(const float *known_feat_pm, int c2, const int *nn_idx, const float *nn_w, const float *skip_pm,
                             int lds, int c1, int b, int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer1,
                             const pvn3d_mlp_layer_t *layer2, int flags, float *out, int ldo, int col0, pvn3d_stream_t stream) {
  if (!layer_pair_ok(layer1, layer2) || !layer_ptrs_ok(layer1) || !layer_ptrs_ok(layer2)) return PVN3D_ERR_INVALID_ARG;
  Fp2Args g{};
  const int rc = fp_interp_args(known_feat_pm, c2, nn_idx, nn_w, skip_pm, lds, c1, b, n_unknown, m_known, *layer1, flags,
                                out, ldo, col0, g.a);
  if (rc != PVN3D_OK) return rc;
  if (!fp2_stages(layer1->k_pad, layer1->n_pad, layer2->k_pad, layer2->n_pad, &g.a_stages, &g.w_stages))
    return PVN3D_ERR_UNSUPPORTED;
  g.a.relu = 1;
  g.w2 = layer2->w; g.bias2 = layer2->bias; g.k2_pad = layer2->k_pad; g.n2_pad = layer2->n_pad;
  return launch_fp2(g, as_stream(stream));
}

extern "C" int pvn3d_mlp_fp2_supported(const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2) {
  if (!layer_pair_ok(layer1, layer2)) return 0;
  int a_stages = 0, w_stages = 0;
  return fp2_stages(layer1->k_pad, layer1->n_pad, layer2->k_pad, layer2->n_pad, &a_stages, &w_stages) ? 1 : 0;
}

// the argument checks and kernel arguments pvn3d_mlp_fp_fact2 and pvn3d_mlp_fp_fact2_rows share
static int fp_fact2_args(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b, int n_unknown,
                         int m_known, const pvn3d_mlp_layer_t *layer_s, const pvn3d_mlp_layer_t *layer2, int flags,
                         float *out, FpFact2Args &g) {
  if (!p || !table || !nn_idx || !nn_w || !layer_s || !layer2 || !layer_s->w || !layer_s->bias || !layer2->w ||
      !layer2->bias || !out || b < 0 || n_unknown < 0 || m_known <= 0 || (flags & ~0xff00) ||
      (reinterpret_cast<uintptr_t>(p) & 15u) || (reinterpret_cast<uintptr_t>(table) & 15u) ||
      (reinterpret_cast<uintptr_t>(layer_s->w) & 15u) || (reinterpret_cast<uintptr_t>(layer2->w) & 15u))
    return PVN3D_ERR_INVALID_ARG;
  const int stages = fpf2_stages(layer_s->k_pad, layer_s->n_pad, layer2->k_pad, layer2->n_pad);
  if (!stages) return PVN3D_ERR_UNSUPPORTED;
  if (static_cast<long long>(b) * m_known > 0x7fffffffll || n_unknown > 0x3fffffff) return PVN3D_ERR_UNSUPPORTED;
  MlpArgs &a = g.a;
  a.rows = static_cast<long long>(b) * n_unknown;
  a.known_feat = p; a.c2 = layer_s->n_pad; a.nn_idx = nn_idx; a.nn_w = nn_w;
  a.n_unknown = n_unknown; a.m_known = m_known;
  a.out = out; a.stages = stages;
  a.reserve_sms = (flags >> 8) & 0xff;
  g.bias_s = layer_s->bias; g.bias2 = layer2->bias;
  return PVN3D_OK;
}

extern "C" int pvn3d_mlp_fp_fact2(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b,
                                  int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer_s,
                                  const pvn3d_mlp_layer_t *layer2, int flags, float *out, pvn3d_stream_t stream) {
  FpFact2Args g{};
  const int rc = fp_fact2_args(p, table, nn_idx, nn_w, b, n_unknown, m_known, layer_s, layer2, flags, out, g);
  if (rc != PVN3D_OK) return rc;
  return launch_fp_fact2<FPF2_OUT_CN>(g, table, layer_s->w, layer2->w, as_stream(stream));
}

extern "C" int pvn3d_mlp_fp_fact2_rows(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b,
                                       int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer_s,
                                       const pvn3d_mlp_layer_t *layer2, int flags, float *out, int ldo, int col0,
                                       pvn3d_stream_t stream) {
  if (ldo % 4 || col0 < 0 || col0 % 4 || static_cast<long long>(col0) + 128 > ldo || (reinterpret_cast<uintptr_t>(out) & 15u) ||
      (layer2 && (reinterpret_cast<uintptr_t>(layer2->bias) & 7u)))
    return PVN3D_ERR_INVALID_ARG;
  FpFact2Args g{};
  const int rc = fp_fact2_args(p, table, nn_idx, nn_w, b, n_unknown, m_known, layer_s, layer2, flags, out, g);
  if (rc != PVN3D_OK) return rc;
  g.a.ldo = ldo;
  g.a.col0 = col0;
  return launch_fp_fact2<FPF2_OUT_ROWS>(g, table, layer_s->w, layer2->w, as_stream(stream));
}

extern "C" int pvn3d_gather_pixel_rows(const float *emb, int b, int c, long long hw, const long long *choose, int n,
                                       float *out, int ldo, int col0, pvn3d_stream_t stream) {
  if (!emb || !choose || !out || b < 0 || n < 0 || c <= 0 || c % 4 || hw <= 0 || ldo % 4 || col0 < 0 || col0 % 4 ||
      static_cast<long long>(col0) + c > ldo || (reinterpret_cast<uintptr_t>(emb) & 3u) ||
      (reinterpret_cast<uintptr_t>(choose) & 7u) || (reinterpret_cast<uintptr_t>(out) & 15u))
    return PVN3D_ERR_INVALID_ARG;
  const long long rows = static_cast<long long>(b) * n;
  if (rows > 0x7fffffffll || c > kGatherMaxC) return PVN3D_ERR_UNSUPPORTED;
  if (rows == 0) return PVN3D_OK;
  const unsigned grid = static_cast<unsigned>((rows + kGatherPts - 1) / kGatherPts);
  gather_pixel_rows_kernel<<<grid, kGatherThreads, 0, as_stream(stream)>>>(emb, c, hw, choose, n, rows, out, ldo, col0);
  return check_launch("gather_pixel_rows_kernel");
}

extern "C" int pvn3d_mlp_fp_fact2_supported(const pvn3d_mlp_layer_t *layer_s, const pvn3d_mlp_layer_t *layer2) {
  if (!layer_s || !layer2) return 0;
  return fpf2_stages(layer_s->k_pad, layer_s->n_pad, layer2->k_pad, layer2->n_pad) ? 1 : 0;
}

extern "C" int pvn3d_mlp_dense_frame_bias(const float *a, int lda, int a_cols, long long rows, int rows_per_frame,
                                          const float *w, const float *bias, int k_pad, int n_pad, int flags,
                                          float *out, int ldo, int col0, pvn3d_stream_t stream) {
  if (rows_per_frame <= 0 || rows_per_frame % kMlpBM || rows % rows_per_frame) return PVN3D_ERR_INVALID_ARG;
  MlpArgs m{};
  const int rc = dense_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, out, ldo, col0, m);
  if (rc != PVN3D_OK) return rc;
  m.bias_npb = rows_per_frame;
  return launch_mlp<EPI_STORE>(m, as_stream(stream));
}

extern "C" int pvn3d_mlp_dense_sum32(const float *a, int lda, int a_cols, long long rows, const float *w,
                                     const float *bias, int k_pad, int n_pad, int flags, float *out, int ldo,
                                     int col0, pvn3d_stream_t stream) {
  MlpArgs m{};
  const int rc = dense_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, out, ldo, col0, m);
  if (rc != PVN3D_OK) return rc;
  m.relu = 1; m.round_out = 0;   // sums of relu(row), stored unrounded
  m.pool = 32;
  return launch_mlp<EPI_SUMPOOL>(m, as_stream(stream));
}

// ---- BF16 forms (FusedHeads at precision "bf16") ------------------------------------------------------------------------
// the argument checks and kernel arguments the three bf16 dense entry points share: PVN3D_ERR_INVALID_ARG for a bad
// operand or a flag outside `allowed` (and the reserved-SM byte), before any CUDA call
static int dense_bf16_args(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, const pvn3d_bf16_t *w,
                           const float *bias, int k_pad, int n_pad, int flags, int allowed, const void *out, int ldo, int col0,
                           MlpArgs &m) {
  if (!a || !w || !bias || !out || a_cols < 0 || lda < a_cols || lda % 8 || a_cols % 8 || rows < 0 || k_pad <= 0 ||
      k_pad % 64 || n_pad <= 0 || n_pad % 16 || ldo % 4 || col0 < 0 || col0 % 4 ||
      static_cast<long long>(col0) + n_pad > ldo || (flags & ~(allowed | 0xff00)) ||
      (reinterpret_cast<uintptr_t>(a) & 15u) || (reinterpret_cast<uintptr_t>(w) & 15u) ||
      (reinterpret_cast<uintptr_t>(out) & 15u))
    return PVN3D_ERR_INVALID_ARG;
  m.w = reinterpret_cast<const float *>(w); m.bias = bias; m.rows = rows; m.k_pad = k_pad; m.n_pad = n_pad;
  m.a = reinterpret_cast<const float *>(a); m.lda = lda; m.a_cols = a_cols;
  m.out = static_cast<float *>(const_cast<void *>(out)); m.ldo = ldo; m.col0 = col0;
  m.relu = (flags & PVN3D_MLP_RELU) ? 1 : 0;
  m.reserve_sms = (flags >> 8) & 0xff;
  return PVN3D_OK;
}

extern "C" int pvn3d_mlp_dense_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, const pvn3d_bf16_t *w,
                                    const float *bias, int k_pad, int n_pad, int flags, void *out, int ldo, int col0,
                                    pvn3d_stream_t stream) {
  MlpArgs m{};
  const int rc = dense_bf16_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, PVN3D_MLP_RELU | PVN3D_MLP_OUT_BF16,
                                 out, ldo, col0, m);
  if (rc != PVN3D_OK) return rc;
  if (flags & PVN3D_MLP_OUT_BF16) return launch_mlp_bf16<EPI_STORE, true>(m, as_stream(stream));
  return launch_mlp_bf16<EPI_STORE, false>(m, as_stream(stream));
}

extern "C" int pvn3d_mlp_dense_frame_bias_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows,
                                               int rows_per_frame, const pvn3d_bf16_t *w, const float *bias, int k_pad,
                                               int n_pad, int flags, void *out, int ldo, int col0, pvn3d_stream_t stream) {
  if (rows_per_frame <= 0 || rows_per_frame % kMlpBM || rows % rows_per_frame) return PVN3D_ERR_INVALID_ARG;
  MlpArgs m{};
  const int rc = dense_bf16_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, PVN3D_MLP_RELU | PVN3D_MLP_OUT_BF16,
                                 out, ldo, col0, m);
  if (rc != PVN3D_OK) return rc;
  m.bias_npb = rows_per_frame;
  if (flags & PVN3D_MLP_OUT_BF16) return launch_mlp_bf16<EPI_STORE, true>(m, as_stream(stream));
  return launch_mlp_bf16<EPI_STORE, false>(m, as_stream(stream));
}

extern "C" int pvn3d_mlp_dense_sum32_bf16(const pvn3d_bf16_t *a, int lda, int a_cols, long long rows, const pvn3d_bf16_t *w,
                                          const float *bias, int k_pad, int n_pad, int flags, float *out, int ldo, int col0,
                                          pvn3d_stream_t stream) {
  MlpArgs m{};
  const int rc = dense_bf16_args(a, lda, a_cols, rows, w, bias, k_pad, n_pad, flags, PVN3D_MLP_RELU, out, ldo, col0, m);
  if (rc != PVN3D_OK) return rc;
  m.relu = 1;
  m.pool = 32;
  return launch_mlp_bf16<EPI_SUMPOOL, false>(m, as_stream(stream));
}

extern "C" int pvn3d_mlp_fp_fact2_rows_bf16(const float *p, const float *table, const int *nn_idx, const float *nn_w, int b,
                                            int n_unknown, int m_known, const pvn3d_mlp_layer_t *layer_s,
                                            const pvn3d_mlp_layer_t *layer2, int flags, pvn3d_bf16_t *out, int ldo, int col0,
                                            pvn3d_stream_t stream) {
  if (ldo % 8 || col0 < 0 || col0 % 8 || static_cast<long long>(col0) + 128 > ldo || (reinterpret_cast<uintptr_t>(out) & 15u) ||
      (layer2 && (reinterpret_cast<uintptr_t>(layer2->bias) & 7u)))
    return PVN3D_ERR_INVALID_ARG;
  FpFact2Args g{};
  const int rc = fp_fact2_args(p, table, nn_idx, nn_w, b, n_unknown, m_known, layer_s, layer2, flags,
                               reinterpret_cast<float *>(out), g);
  if (rc != PVN3D_OK) return rc;
  g.a.ldo = ldo;
  g.a.col0 = col0;
  return launch_fp_fact2<FPF2_OUT_ROWS_BF16>(g, table, layer_s->w, layer2->w, as_stream(stream));
}

extern "C" int pvn3d_gather_pixel_rows_bf16(const void *emb, int emb_bf16, int b, int c, long long hw,
                                            const long long *choose, int n, pvn3d_bf16_t *out, int ldo, int col0,
                                            pvn3d_stream_t stream) {
  if (!emb || !choose || !out || (emb_bf16 != 0 && emb_bf16 != 1) || b < 0 || n < 0 || c <= 0 || c % 8 || hw <= 0 ||
      ldo % 8 || col0 < 0 || col0 % 8 || static_cast<long long>(col0) + c > ldo ||
      (reinterpret_cast<uintptr_t>(emb) & (emb_bf16 ? 1u : 3u)) || (reinterpret_cast<uintptr_t>(choose) & 7u) ||
      (reinterpret_cast<uintptr_t>(out) & 15u))
    return PVN3D_ERR_INVALID_ARG;
  const long long rows = static_cast<long long>(b) * n;
  if (rows > 0x7fffffffll || c > kGatherMaxC) return PVN3D_ERR_UNSUPPORTED;
  if (rows == 0) return PVN3D_OK;
  const unsigned grid = static_cast<unsigned>((rows + kGatherPts - 1) / kGatherPts);
  if (emb_bf16)
    gather_pixel_rows_bf16_kernel<uint16_t><<<grid, kGatherThreads, 0, as_stream(stream)>>>(
        static_cast<const uint16_t *>(emb), c, hw, choose, n, rows, out, ldo, col0);
  else
    gather_pixel_rows_bf16_kernel<float><<<grid, kGatherThreads, 0, as_stream(stream)>>>(
        static_cast<const float *>(emb), c, hw, choose, n, rows, out, ldo, col0);
  return check_launch("gather_pixel_rows_bf16_kernel");
}

// ---- the CNN tail at the sampled pixels (psp_tail_kernel) -----------------------------------------------------------
// the argument checks and kernel arguments pvn3d_psp_tail_rows and pvn3d_psp_tail_rows_bf16 share; `align` = elements of
// the output type per 16 bytes
static int psp_tail_args(const float *x, int b, int h, int w, const long long *choose, int n, const pvn3d_mlp_layer_t *layer1,
                         const pvn3d_mlp_layer_t *layer2, const float *slope, int flags, void *out, int ldo, int col0,
                         int align, PspTailArgs &g) {
  if (!x || !choose || !layer1 || !layer2 || !slope || !out || !layer_ptrs_ok(layer1) || !layer_ptrs_ok(layer2) || b < 0 ||
      n < 0 || h < 2 || w < 2 || (flags & ~0xff00) || ldo % align || col0 < 0 || col0 % align ||
      static_cast<long long>(col0) + kPspN2 > ldo || (reinterpret_cast<uintptr_t>(x) & 15u) ||
      (reinterpret_cast<uintptr_t>(choose) & 7u) || (reinterpret_cast<uintptr_t>(out) & 15u) ||
      (reinterpret_cast<uintptr_t>(layer2->bias) & 7u))
    return PVN3D_ERR_INVALID_ARG;
  g.stages = psp_tail_stages(layer1->k_pad, layer1->n_pad, layer2->k_pad, layer2->n_pad);
  if (!g.stages) return PVN3D_ERR_UNSUPPORTED;
  // the kernel addresses source pixels and rows with 32-bit integers, and t (h - 1) of a tap coordinate t < 2 h
  if (h > 0x7fff || w > 0x7fff || static_cast<long long>(b) * h * w > 0x7fffffffll ||
      static_cast<long long>(b) * n > 0x7fffffffll)
    return PVN3D_ERR_UNSUPPORTED;
  g.x = x; g.choose = choose; g.bias1 = layer1->bias; g.slope = slope; g.bias2 = layer2->bias;
  g.out = out; g.rows = static_cast<long long>(b) * n;
  g.n = n; g.h = h; g.w = w; g.ldo = ldo; g.col0 = col0;
  g.reserve_sms = (flags >> 8) & 0xff;
  return PVN3D_OK;
}

extern "C" int pvn3d_psp_tail_rows(const float *x, int b, int h, int w, const long long *choose, int n,
                                   const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2, const float *slope,
                                   int flags, float *out, int ldo, int col0, pvn3d_stream_t stream) {
  PspTailArgs g{};
  const int rc = psp_tail_args(x, b, h, w, choose, n, layer1, layer2, slope, flags, out, ldo, col0, 4, g);
  if (rc != PVN3D_OK) return rc;
  return launch_psp_tail<false>(g, layer1->w, layer2->w, as_stream(stream));
}

extern "C" int pvn3d_psp_tail_rows_bf16(const float *x, int b, int h, int w, const long long *choose, int n,
                                        const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2,
                                        const float *slope, int flags, pvn3d_bf16_t *out, int ldo, int col0,
                                        pvn3d_stream_t stream) {
  PspTailArgs g{};
  const int rc = psp_tail_args(x, b, h, w, choose, n, layer1, layer2, slope, flags, out, ldo, col0, 8, g);
  if (rc != PVN3D_OK) return rc;
  return launch_psp_tail<true>(g, layer1->w, layer2->w, as_stream(stream));
}

extern "C" int pvn3d_psp_tail_supported(const pvn3d_mlp_layer_t *layer1, const pvn3d_mlp_layer_t *layer2) {
  if (!layer1 || !layer2) return 0;
  return psp_tail_stages(layer1->k_pad, layer1->n_pad, layer2->k_pad, layer2->n_pad) ? 1 : 0;
}
