// query_group.cu -- fused ball-query + grouping for sm_90a (the HBM-bound kernel of the path).
//
// Replaces the five launches + two copies the reference spends per scale in
// QueryAndGroup.forward (pvn3d/lib/pointnet2_utils/pointnet2_utils.py:311-321):
//     ball_query -> transpose(xyz) -> group_points(xyz) -> subtract centre -> group_points(feats)
//     -> torch.cat
// with ONE kernel that writes idx[B,M,S] and the concatenated tensor out[B,3+C,M,S] directly --
// optionally for the TWO radii of a multi-scale-grouping level at once (same centres, same cloud:
// every squared distance is computed once and compared against both radii).
//
// Two kernels per launch (plus two tiny pre-passes):
//   pre-pass   bounding box of every 128-point block of the cloud; scan order of the centres (bucketed
//              by y, so that the CW centres a warp scans for together are neighbours).
//   scan       (ball_scan_kernel, 8 warps x CW centres per CTA, little shared memory -> 5+ CTAs/SM)
//              each warp walks the cloud ON ITS OWN -- no tile staging, no CTA barriers -- balloting 32
//              points per step against its CW centres (hits are appended in index order: the
//              reference's first-nsample rule by construction) and skipping every block whose box is
//              out of reach of the box of its centres.  Exact pruning: free on shuffled clouds, removes
//              ~90 % of the scan on raster-ordered ones (the reference's samplers keep raster order).
//              The next step's points are loaded while the current ones are tested.  Result: idx[B,M,S]
//              (the caller's buffer, or stream-ordered scratch when only the grouped tensor is wanted).
//   group      (group_write_kernel, 768 consecutive output slots of one scale per CTA, 3 CTAs/SM)
//              descriptors are read POINT-MAJOR (feat_pm[B,N,ldf]).  A warp owns 32 consecutive slots:
//              cp.async pulls 32 channels of four neighbours per instruction (8 lanes = one fully used
//              128-byte run) into one of two private shared-memory tiles while the previous tile is
//              written out as 16-byte stores -- 8 lanes cover one 128-byte line of a channel row, a
//              warp instruction four rows -- after a 4x4 register transpose.  Every output byte is
//              written once, in runs of 3 KB per channel and CTA; every gathered sector is fully used.
// Algorithmic HBM bytes per launch and scale (DESIGN.md section 4):
//   B * [ 12 N + 12 M + 4 C N  (reads)  +  4 M S + 4 (3+C) M S  (writes) ].
#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kQgThreads = 256;
constexpr int kQgWarps = 8;
constexpr int kQgMaxBlocks = 1024;  // bounding-box blocks per cloud (24 KB of shared memory at most)
constexpr int kQgMaxSlots = 2048;   // scan: slots (centres x nsample, both scales) per CTA
constexpr int kQgGroupSlots = 768;  // group: consecutive output slots of one scale per CTA (75 KB of
                                    // shared memory with the transpose tiles: three CTAs per SM)
constexpr int kQgTrStride = 36;     // floats per row of a per-warp [32 slots][32 channels] tile
constexpr int kQgTrFloats = 32 * kQgTrStride;  // one tile; every warp owns two (double buffering)
static_assert(2 * kQgTrFloats >= 32 * 33, "scalar fallback transposes through the same buffer");

struct QgScale {
  float radius;
  int ns;
  int *idx;    // [B,M,ns] or null
  float *out;  // [B,3+C,M,ns] or null (idx-only launch)
};
struct QgArgs {
  const float *xyz, *new_xyz, *feat;
  int ldf, n, m, c;
  int blk;  // points per bounding-box block (multiple of 32; at most 896 blocks + their super boxes)
  const float *boxes;  // [B][nblk][6] from qg_boxes_kernel
  int group_slots;     // output slots per CTA of group_write_kernel (<= kQgGroupSlots, multiple of 32)
  const int *perm;     // [B][M] centres in scan order (sorted by y) from qg_sort_centres_kernel
  QgScale s[2];
};

struct QgGroupSmem {
  static constexpr size_t rows_bytes = kQgGroupSlots * sizeof(int);                        // 3072
  static constexpr size_t tr_bytes = kQgWarps * 2 * kQgTrFloats * sizeof(float);           // 73728
  static constexpr size_t total = rows_bytes + tr_bytes;
};

__device__ __forceinline__ void qg_append(unsigned hits, int &cnt, int &first, int ns, int *row,
                                          int kbase, unsigned lane) {
  if (cnt == 0) first = kbase + __ffs(hits) - 1;
  const int slot = cnt + __popc(hits & lanemask_lt());
  if (((hits >> lane) & 1u) && slot < ns) row[slot] = kbase + static_cast<int>(lane);
  cnt += __popc(hits);
}

__device__ __forceinline__ void cp_async16(void *dst_smem, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// write one scale's slots of this CTA: xyz difference channels + descriptor channels
// write the CTA's slots [slot0, slot0 + nslots) of one scale (slot = centre * ns + neighbour):
// xyz difference channels + descriptor channels.  rows[s] = index of the neighbour in the cloud.
__device__ __forceinline__ void qg_write_scale(const QgArgs &a, const QgScale &sc, int b, int slot0,
                                               int nslots, const int *rows, float *s_tr) {
  const int t = threadIdx.x;
  const unsigned lane = lane_id(), warp = t >> 5;
  const int ns = sc.ns, c = a.c;
  const size_t plane = static_cast<size_t>(a.m) * ns;
  const size_t slot_base = static_cast<size_t>(slot0);
  const float *cloud = a.xyz + static_cast<size_t>(b) * a.n * 3;
  float *out_b = sc.out + static_cast<size_t>(b) * (3 + c) * plane + slot_base;

  for (int s = t; s < nslots; s += kQgThreads) {
    const int p = rows[s];
    // grouped_xyz - new_xyz  (pointnet2_utils.py:313-314)
    const float *ctr = a.new_xyz + (static_cast<size_t>(b) * a.m + (slot0 + s) / ns) * 3;
    const float *pt = cloud + static_cast<size_t>(p) * 3;
    stg_stream(out_b + 0 * plane + s, __ldg(pt + 0) - __ldg(ctr + 0));
    stg_stream(out_b + 1 * plane + s, __ldg(pt + 1) - __ldg(ctr + 1));
    stg_stream(out_b + 2 * plane + s, __ldg(pt + 2) - __ldg(ctr + 2));
  }
  if (c == 0) return;
  const float *feat_b = a.feat + static_cast<size_t>(b) * a.n * a.ldf;
  float *out_f = out_b + 3 * plane;
  const bool vec = (c % 4 == 0) && (a.ldf % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.feat) & 15u) == 0) &&
                   (plane % 4 == 0) && (slot_base % 4 == 0) && (nslots % 4 == 0) &&
                   ((reinterpret_cast<uintptr_t>(sc.out) & 15u) == 0);
  float *tr = s_tr + warp * (2 * kQgTrFloats);
  const int ngroups = (nslots + 31) / 32;
  if (vec) {
    // Work items of this warp: (group g of 32 slots, chunk of 32 channels).  The neighbour rows of
    // item i+1 are fetched with cp.async (16 B per lane, 8 lanes = one 128-byte run of a row, four
    // rows per instruction) into the other buffer while item i is transposed and stored.
    const int nchunks = (c + 31) / 32;
    const int my_groups = (ngroups > static_cast<int>(warp)) ? (ngroups - static_cast<int>(warp) + kQgWarps - 1) / kQgWarps : 0;
    const int items = my_groups * nchunks;
    const int sub = lane >> 3, chunk = lane & 7;  // gather: neighbour sub-row, 16-byte chunk
    const int m8 = lane >> 2, k4 = lane & 3;      // store: slots 4*m8.., channel quad
    auto issue = [&](int item, float *buf) {
      const int g0 = (static_cast<int>(warp) + (item / nchunks) * kQgWarps) * 32;
      const int c0 = (item % nchunks) * 32;
      const int glive = min(32, nslots - g0);
      const int quads = min(8, (c - c0) / 4);
      if (chunk < quads) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int q = 4 * i + sub;
          if (q < glive)
            cp_async16(buf + q * kQgTrStride + 4 * chunk,
                       feat_b + static_cast<size_t>(rows[g0 + q]) * a.ldf + c0 + 4 * chunk);
        }
      }
      cp_async_commit();
    };
    if (items > 0) issue(0, tr);
    for (int item = 0; item < items; ++item) {
      float *buf = tr + (item & 1) * kQgTrFloats;
      if (item + 1 < items) {
        issue(item + 1, tr + ((item + 1) & 1) * kQgTrFloats);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncwarp();
      const int g0 = (static_cast<int>(warp) + (item / nchunks) * kQgWarps) * 32;
      const int c0 = (item % nchunks) * 32;
      const int glive = min(32, nslots - g0);  // multiple of 4 (nslots % 4 == 0)
      const int quads = min(8, (c - c0) / 4);
      if (4 * m8 < glive) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int quad = 4 * j + k4;
          if (quad < quads) {
            const float4 v0 = *reinterpret_cast<const float4 *>(buf + (4 * m8 + 0) * kQgTrStride + 4 * quad);
            const float4 v1 = *reinterpret_cast<const float4 *>(buf + (4 * m8 + 1) * kQgTrStride + 4 * quad);
            const float4 v2 = *reinterpret_cast<const float4 *>(buf + (4 * m8 + 2) * kQgTrStride + 4 * quad);
            const float4 v3 = *reinterpret_cast<const float4 *>(buf + (4 * m8 + 3) * kQgTrStride + 4 * quad);
            float *dst = out_f + static_cast<size_t>(c0 + 4 * quad) * plane + g0 + 4 * m8;
            stg_stream4(dst + 0 * plane, make_float4(v0.x, v1.x, v2.x, v3.x));
            stg_stream4(dst + 1 * plane, make_float4(v0.y, v1.y, v2.y, v3.y));
            stg_stream4(dst + 2 * plane, make_float4(v0.z, v1.z, v2.z, v3.z));
            stg_stream4(dst + 3 * plane, make_float4(v0.w, v1.w, v2.w, v3.w));
          }
        }
      }
      __syncwarp();  // buffer (item & 1) is refilled two items later
    }
    return;
  }
  if (c <= 16) {
    // few channels (level 1: rgb + normal): every slot walks its own short row
    for (int s = t; s < nslots; s += kQgThreads) {
      const float *row = feat_b + static_cast<size_t>(rows[s]) * a.ldf;
      for (int ch = 0; ch < c; ++ch) stg_stream(out_f + ch * plane + s, __ldg(row + ch));
    }
    return;
  }
  // generic rows (odd channel counts / unaligned strides): scalar 32x32 transposes
  for (int g = warp; g < ngroups; g += kQgWarps) {  // warp-uniform
    const int g0 = g * 32;
    const int glive = min(32, nslots - g0);
    const int p = (static_cast<int>(lane) < glive) ? rows[g0 + lane] : 0;
    for (int c0 = 0; c0 < c; c0 += 32) {
      const int cw = min(32, c - c0);
      __syncwarp();
      for (int q = 0; q < 32; ++q) {
        const int pq = __shfl_sync(0xffffffffu, p, q);
        float v = 0.f;
        if (static_cast<int>(lane) < cw && q < glive)
          v = __ldg(feat_b + static_cast<size_t>(pq) * a.ldf + c0 + lane);
        tr[lane * 33 + q] = v;
      }
      __syncwarp();
      if (static_cast<int>(lane) < glive) {
        float *dst = out_f + static_cast<size_t>(c0) * plane + g0 + lane;
        for (int cc = 0; cc < cw; ++cc) stg_stream(dst + cc * plane, tr[cc * 33 + lane]);
      }
    }
  }
}

// Bounding boxes of every block of `blk` consecutive points (one warp per block) -- computed once per
// cloud, not once per CTA.
__global__ void qg_boxes_kernel(const float *__restrict__ xyz, int n, int blk, int nblk,
                                float *__restrict__ boxes) {
  const int b = blockIdx.y;
  const unsigned lane = lane_id();
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= nblk) return;
  const float *cloud = xyz + static_cast<size_t>(b) * n * 3;
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  const int k_end = min((g + 1) * blk, n);
  for (int k = g * blk + static_cast<int>(lane); k < k_end; k += 32) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float v = __ldg(cloud + static_cast<size_t>(k) * 3 + d);
      lo[d] = fminf(lo[d], v);
      hi[d] = fmaxf(hi[d], v);
      if (!(v == v)) { lo[d] = -3.0e38f; hi[d] = 3.0e38f; }  // NaN coordinate: never skip this block
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if (lane == 0) {
    float *o = boxes + (static_cast<size_t>(b) * nblk + g) * 6;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      o[d] = lo[d];
      o[3 + d] = hi[d];
    }
  }
}
// Scan order of the centres of one cloud: bucketed by y (1024 buckets between the smallest and the
// largest y; the order inside a bucket is whatever the atomics give).  FPS hands the centres out
// scattered all over the cloud; the CW centres a warp scans for together must be NEIGHBOURS for the
// union of their balls to stay as small as one ball (and the blocks of a raster-ordered cloud are
// thin in y).  ANY order gives the same output, so a counting sort is enough.  One CTA per cloud.
constexpr int kQgSortMax = 1 << 20;
constexpr int kQgBuckets = 1024;
__global__ void __launch_bounds__(1024) qg_sort_centres_kernel(const float *__restrict__ new_xyz, int m,
                                                               int *__restrict__ perm) {
  __shared__ int s_cnt[kQgBuckets];
  __shared__ float s_lo[32], s_hi[32];
  __shared__ int s_warp[32];
  const int b = blockIdx.x, t = threadIdx.x;
  const unsigned lane = lane_id(), warp = t >> 5;
  const float *ys = new_xyz + static_cast<size_t>(b) * m * 3 + 1;
  float lo = 3.0e38f, hi = -3.0e38f;
  for (int i = t; i < m; i += 1024) {
    const float y = ys[static_cast<size_t>(i) * 3];
    if (fabsf(y) < 3.0e38f) {  // finite
      lo = fminf(lo, y);
      hi = fmaxf(hi, y);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
  s_cnt[t] = 0;
  __syncthreads();
  lo = s_lo[0]; hi = s_hi[0];
  for (int w = 1; w < 32; ++w) { lo = fminf(lo, s_lo[w]); hi = fmaxf(hi, s_hi[w]); }
  const float scale = hi > lo ? static_cast<float>(kQgBuckets) / (hi - lo) : 0.f;
  auto bucket = [&](float y) {
    if (!(fabsf(y) < 3.0e38f)) return kQgBuckets - 1;  // NaN / inf: last bucket
    const int k = static_cast<int>((y - lo) * scale);
    return max(0, min(kQgBuckets - 1, k));
  };
  for (int i = t; i < m; i += 1024) atomicAdd(&s_cnt[bucket(ys[static_cast<size_t>(i) * 3])], 1);
  __syncthreads();
  // exclusive scan of the 1024 counts (one per thread)
  const int mine = s_cnt[t];
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (static_cast<int>(lane) >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int base = 0;
  for (int w = 0; w < static_cast<int>(warp); ++w) base += s_warp[w];
  __syncthreads();
  s_cnt[t] = base + incl - mine;  // first output position of bucket t
  __syncthreads();
  for (int i = t; i < m; i += 1024) {
    const int pos = atomicAdd(&s_cnt[bucket(ys[static_cast<size_t>(i) * 3])], 1);
    perm[static_cast<size_t>(b) * m + pos] = i;
  }
}
__global__ void qg_identity_perm_kernel(int m, int *__restrict__ perm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) perm[static_cast<size_t>(blockIdx.y) * m + i] = i;
}

// squared distance between two axis-aligned boxes (0 when they overlap); b[0..2] = lo, b[3..5] = hi
__device__ __forceinline__ float qg_box_dist2(const float (&u)[6], const float *b) {
  const float ex = fmaxf(fmaxf(b[0] - u[3], u[0] - b[3]), 0.f);
  const float ey = fmaxf(fmaxf(b[1] - u[4], u[1] - b[4]), 0.f);
  const float ez = fmaxf(fmaxf(b[2] - u[5], u[2] - b[5]), 0.f);
  return ex * ex + ey * ey + ez * ez;
}

template <int CW, bool DUAL>
__global__ void __launch_bounds__(kQgThreads, 4) ball_scan_kernel(QgArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int *s_rows = reinterpret_cast<int *>(smem_raw);                                      // [kQgMaxSlots]
  float *s_box = reinterpret_cast<float *>(smem_raw + kQgMaxSlots * sizeof(int));       // [nblk][6]
  __shared__ int s_cent[32];  // local centre (scan slot) -> centre index in the cloud

  constexpr int TJ = kQgWarps * CW;
  const int b = blockIdx.y;
  const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
  const float *cloud = a.xyz + static_cast<size_t>(b) * a.n * 3;
  const int jc0 = blockIdx.x * TJ;
  const int live_centres = min(TJ, a.m - jc0);
  const int nsa = a.s[0].ns, nsb = DUAL ? a.s[1].ns : 0;
  const float r2a = __fmul_rn(a.s[0].radius, a.s[0].radius);  // ball_query_gpu.cu:22
  const float r2b = DUAL ? __fmul_rn(a.s[1].radius, a.s[1].radius) : 0.f;
  // a block can be skipped when even its bounding box is out of reach of the larger radius; the bound
  // is inflated so that fp32 rounding of the box distance can never hide a true hit
  const float r2max = fmaxf(r2a, r2b);
  const bool a_is_max = !DUAL || !(r2a < r2b);
  const float r2skip = r2max * 1.0001f + 1e-12f;
  int *rows_a = s_rows;             // [TJ][nsa]
  int *rows_b = s_rows + TJ * nsa;  // [TJ][nsb]

  // ---- bounding boxes of the cloud's blocks (a.blk points each) -------------------------------------
  const int blk = a.blk, nblk = (a.n + blk - 1) / blk;
  {
    const float *src = a.boxes + static_cast<size_t>(b) * nblk * 6;
    for (int e = threadIdx.x; e < nblk * 6; e += kQgThreads) s_box[e] = __ldg(src + e);
  }
  // the CTA's centres: TJ consecutive entries of the cloud's y-sorted centre list
  if (threadIdx.x < TJ)
    s_cent[threadIdx.x] = (static_cast<int>(threadIdx.x) < live_centres)
                              ? __ldg(a.perm + static_cast<size_t>(b) * a.m + jc0 + threadIdx.x)
                              : 0;
  __syncthreads();
  // ---------------- phase 1: warp w scans for the centres in scan slots w*CW .. w*CW+CW-1 ------------
  // No tile staging, no CTA barriers: every warp walks the cloud on its own (L1/L2-resident, 384
  // contiguous bytes per step) and only where the box tests say a neighbour can be.
  float cx[CW], cy[CW], cz[CW];
  int cnta[CW], firsta[CW], cntb[CW], firstb[CW], lcs[CW];
  float ub[6] = {3.0e38f, 3.0e38f, 3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f};  // box of the warp's centres
  bool warp_open = false;
#pragma unroll
  for (int q = 0; q < CW; ++q) {
    const int lc = static_cast<int>(warp) * CW + q;
    lcs[q] = lc;
    const bool live = lc < live_centres;
    const float *p = a.new_xyz + (static_cast<size_t>(b) * a.m + (live ? s_cent[lc] : 0)) * 3;
    cx[q] = p[0];
    cy[q] = p[1];
    cz[q] = p[2];
    cnta[q] = live ? 0 : nsa;  // dead centres count as full
    cntb[q] = live ? 0 : nsb;
    firsta[q] = firstb[q] = 0;
    if (live) {
      warp_open = true;
      ub[0] = fminf(ub[0], cx[q]); ub[1] = fminf(ub[1], cy[q]); ub[2] = fminf(ub[2], cz[q]);
      ub[3] = fmaxf(ub[3], cx[q]); ub[4] = fmaxf(ub[4], cy[q]); ub[5] = fmaxf(ub[5], cz[q]);
      if (!(cx[q] == cx[q]) || !(cy[q] == cy[q]) || !(cz[q] == cz[q])) {  // NaN centre: no pruning
        ub[0] = ub[1] = ub[2] = -3.0e38f;
        ub[3] = ub[4] = ub[5] = 3.0e38f;
      }
    }
  }
  for (int gb = 0; gb < nblk && warp_open; gb += 32) {
    // 32 box tests at once (lane l: block gb + l), then only the blocks that can hold a neighbour
    const int gl = gb + static_cast<int>(lane);
    unsigned cand = __ballot_sync(0xffffffffu, gl < nblk && !(qg_box_dist2(ub, s_box + gl * 6) > r2skip));
    while (cand && warp_open) {
      const int g = gb + __ffs(cand) - 1;
      cand &= cand - 1;
      const int k_end = min((g + 1) * blk, a.n);
      int off = g * blk;
      bool in = off + static_cast<int>(lane) < k_end;
      const float *pt = cloud + static_cast<size_t>(in ? off + static_cast<int>(lane) : off) * 3;
      float x = __ldg(pt), y = __ldg(pt + 1), z = __ldg(pt + 2);
      for (; off < k_end; off += 32) {
        // the next 32 points are on their way while these are tested
        const int noff = off + 32;
        bool nin = false;
        float nx = 0.f, ny = 0.f, nz = 0.f;
        if (noff < k_end) {
          nin = noff + static_cast<int>(lane) < k_end;
          const float *np = cloud + static_cast<size_t>(nin ? noff + static_cast<int>(lane) : noff) * 3;
          nx = __ldg(np); ny = __ldg(np + 1); nz = __ldg(np + 2);
        }
#pragma unroll
        for (int q = 0; q < CW; ++q) {
          const float d2 = ref_sqdist(cx[q] - x, cy[q] - y, cz[q] - z);
          // one ballot against the larger radius decides the common no-neighbour step (and is that
          // radius' hit mask)
          const unsigned any = __ballot_sync(0xffffffffu, in && d2 < r2max);
          if (any) {
            const unsigned ha = a_is_max ? any : __ballot_sync(0xffffffffu, in && d2 < r2a);
            const unsigned hb = !DUAL ? 0u : (a_is_max ? __ballot_sync(0xffffffffu, in && d2 < r2b) : any);
            if (ha && cnta[q] < nsa)
              qg_append(ha, cnta[q], firsta[q], nsa, rows_a + lcs[q] * nsa, off, lane);
            if (DUAL && hb && cntb[q] < nsb)
              qg_append(hb, cntb[q], firstb[q], nsb, rows_b + lcs[q] * nsb, off, lane);
          }
        }
        x = nx; y = ny; z = nz; in = nin;
      }
      bool open = false;
#pragma unroll
      for (int q = 0; q < CW; ++q) open |= (cnta[q] < nsa) || (DUAL && cntb[q] < nsb);
      warp_open = open;  // every ball of this warp is full: nothing further can be appended
    }
  }
  // pad the rows (slots >= cnt repeat the first hit; 0 for an empty ball: torch::zeros,
  // ball_query.cpp:19) and hand them out: idx[b][centre][0:ns]
  __syncwarp();
#pragma unroll
  for (int q = 0; q < CW; ++q) {
    const int lc = lcs[q];
    if (lc < live_centres) {
      const size_t cent = static_cast<size_t>(b) * a.m + s_cent[lc];
      for (int s = static_cast<int>(lane); s < nsa; s += 32)
        a.s[0].idx[cent * nsa + s] = s < cnta[q] ? rows_a[lc * nsa + s] : firsta[q];
      if (DUAL)
        for (int s = static_cast<int>(lane); s < nsb; s += 32)
          a.s[1].idx[cent * nsb + s] = s < cntb[q] ? rows_b[lc * nsb + s] : firstb[q];
    }
  }
}

// grid (ceil(M*ns / kQgGroupSlots), B, scales): the grouped tensor of one scale from its idx
__global__ void __launch_bounds__(kQgThreads, 3) group_write_kernel(QgArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int *s_rows = reinterpret_cast<int *>(smem_raw);
  float *s_tr = reinterpret_cast<float *>(smem_raw + QgGroupSmem::rows_bytes);
  const QgScale &sc = a.s[blockIdx.z];
  if (!sc.out) return;
  const int b = blockIdx.y;
  const long long total = static_cast<long long>(a.m) * sc.ns;
  const long long slot0 = static_cast<long long>(blockIdx.x) * a.group_slots;
  if (slot0 >= total) return;
  const int nslots = static_cast<int>(min(static_cast<long long>(a.group_slots), total - slot0));
  const int *src = sc.idx + static_cast<size_t>(b) * total + slot0;
  for (int s = threadIdx.x; s < nslots; s += kQgThreads) s_rows[s] = __ldg(src + s);
  __syncthreads();
  qg_write_scale(a, sc, b, static_cast<int>(slot0), nslots, s_rows, s_tr);
}

template <int CW, bool DUAL>
int qg_launch(const QgArgs &a, int b, cudaStream_t st) {
  const int nblk = ceil_div(a.n, a.blk);
  const size_t smem = kQgMaxSlots * sizeof(int) + static_cast<size_t>(nblk) * 6 * sizeof(float);
  dim3 grid(ceil_div(a.m, kQgWarps * CW), b);
  ball_scan_kernel<CW, DUAL><<<grid, kQgThreads, smem, st>>>(a);
  return check_launch("ball_scan_kernel");
}

int qg_launch_group(QgArgs &a, int b, bool dual, cudaStream_t st) {
  if (!a.s[0].out && !(dual && a.s[1].out)) return PVN3D_OK;
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once,
                        cudaFuncSetAttribute(group_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)QgGroupSmem::total),
                        "group_write smem attr");
  const int ns_max = std::max(a.s[0].ns, dual ? a.s[1].ns : 0);
  // slots per CTA: the full 768 when that still gives every SM its three CTAs twice over, else less
  const long long all_slots = static_cast<long long>(b) * a.m * (a.s[0].ns + (dual ? a.s[1].ns : 0));
  const long long want_ctas = 6ll * std::max(1, sm_count());
  a.group_slots = kQgGroupSlots;
  while (a.group_slots > 256 && all_slots / a.group_slots < want_ctas) a.group_slots -= 128;
  const long long groups = (static_cast<long long>(a.m) * ns_max + a.group_slots - 1) / a.group_slots;
  if (groups > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  dim3 grid(static_cast<unsigned>(groups), b, dual ? 2 : 1);
  group_write_kernel<<<grid, kQgThreads, QgGroupSmem::total, st>>>(a);
  return check_launch("group_write_kernel");
}

int qg_dispatch_launch(QgArgs &a, int b, bool dual, cudaStream_t st);

int qg_dispatch(QgArgs &a, int b, bool dual, cudaStream_t st) {
  a.blk = 128;  // (32-point boxes prune better but cost more than they save: 330 vs 270 us at level 1)
  while (ceil_div(a.n, a.blk) > kQgMaxBlocks) a.blk *= 2;  // box table lives in 24 KB of shared memory
  const int nblk = ceil_div(a.n, a.blk);
  int rc0 = keep_async_pool_warm();
  if (rc0 != PVN3D_OK) return rc0;
  // stream-ordered scratch: boxes [B][nblk][6] floats (2.3 KB per 12288-pt cloud), scan order [B][M],
  // and idx [B][M][ns] of every scale whose idx the caller did not ask for
  const size_t box_bytes = align_up(sizeof(float) * 6 * static_cast<size_t>(b) * nblk, 256);
  const size_t perm_bytes = align_up(sizeof(int) * static_cast<size_t>(b) * a.m, 256);
  size_t idx_bytes[2] = {0, 0};
  for (int i = 0; i < (dual ? 2 : 1); ++i)
    if (!a.s[i].idx) idx_bytes[i] = align_up(sizeof(int) * static_cast<size_t>(b) * a.m * a.s[i].ns, 256);
  unsigned char *scratch = nullptr;
  PVN3D_CUDA_TRY(cudaMallocAsync(&scratch, box_bytes + perm_bytes + idx_bytes[0] + idx_bytes[1], st),
                 "query_group scratch");
  float *boxes = reinterpret_cast<float *>(scratch);
  int *perm = reinterpret_cast<int *>(scratch + box_bytes);
  if (idx_bytes[0]) a.s[0].idx = reinterpret_cast<int *>(scratch + box_bytes + perm_bytes);
  if (idx_bytes[1]) a.s[1].idx = reinterpret_cast<int *>(scratch + box_bytes + perm_bytes + idx_bytes[0]);
  qg_boxes_kernel<<<dim3(ceil_div(nblk, 8), b), 256, 0, st>>>(a.xyz, a.n, a.blk, nblk, boxes);
  int rc = check_launch("qg_boxes_kernel");
  if (rc == PVN3D_OK) {
    if (a.m <= kQgSortMax) {
      qg_sort_centres_kernel<<<b, 1024, 0, st>>>(a.new_xyz, a.m, perm);
      rc = check_launch("qg_sort_centres_kernel");
    } else {
      qg_identity_perm_kernel<<<dim3(ceil_div(a.m, 256), b), 256, 0, st>>>(a.m, perm);
      rc = check_launch("qg_identity_perm_kernel");
    }
  }
  a.boxes = boxes;
  a.perm = perm;
  if (rc == PVN3D_OK) rc = qg_dispatch_launch(a, b, dual, st);
  if (rc == PVN3D_OK) rc = qg_launch_group(a, b, dual, st);
  cudaFreeAsync(scratch, st);
  return rc;
}

int qg_dispatch_launch(QgArgs &a, int b, bool dual, cudaStream_t st) {
  const int ns_tot = a.s[0].ns + (dual ? a.s[1].ns : 0);
  // centres per warp: as many as fit the row buffer; big clouds amortise the scan over 4 centres
  int cw = 4;
  if (a.n < 2048) cw = 2;
  if (a.n < 1024) cw = 1;
  while (cw > 1 && kQgWarps * cw * ns_tot > kQgMaxSlots) cw >>= 1;
  if (kQgWarps * cw * ns_tot > kQgMaxSlots) return PVN3D_ERR_UNSUPPORTED;
  if (dual) {
    if (cw == 4) return qg_launch<4, true>(a, b, st);
    if (cw == 2) return qg_launch<2, true>(a, b, st);
    return qg_launch<1, true>(a, b, st);
  }
  if (cw == 4) return qg_launch<4, false>(a, b, st);
  if (cw == 2) return qg_launch<2, false>(a, b, st);
  return qg_launch<1, false>(a, b, st);
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_query_and_group(const float *xyz, const float *new_xyz, const float *feat_pm,
                                     int ldf, int b, int n, int m, int c, float radius,
                                     int nsample, int *idx, float *out, pvn3d_stream_t stream) {
  if (!xyz || !new_xyz || !out || b < 0 || n <= 0 || m < 0 || c < 0 || nsample < 0)
    return PVN3D_ERR_INVALID_ARG;
  if (c > 0 && (!feat_pm || ldf < c)) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || m == 0 || nsample == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  QgArgs a{};
  a.xyz = xyz; a.new_xyz = new_xyz; a.feat = feat_pm; a.ldf = ldf; a.n = n; a.m = m; a.c = c;
  a.s[0] = QgScale{radius, nsample, idx, out};
  return qg_dispatch(a, b, false, as_stream(stream));
}

extern "C" int pvn3d_query_and_group2(const float *xyz, const float *new_xyz, const float *feat_pm,
                                      int ldf, int b, int n, int m, int c, float radius0,
                                      int nsample0, int *idx0, float *out0, float radius1,
                                      int nsample1, int *idx1, float *out1, pvn3d_stream_t stream) {
  if (!xyz || !new_xyz || b < 0 || n <= 0 || m < 0 || c < 0 || nsample0 <= 0 || nsample1 <= 0)
    return PVN3D_ERR_INVALID_ARG;
  if ((!idx0 && !out0) || (!idx1 && !out1)) return PVN3D_ERR_INVALID_ARG;
  if (c > 0 && (out0 || out1) && (!feat_pm || ldf < c)) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || m == 0) return PVN3D_OK;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  QgArgs a{};
  a.xyz = xyz; a.new_xyz = new_xyz; a.feat = feat_pm; a.ldf = ldf; a.n = n; a.m = m; a.c = c;
  a.s[0] = QgScale{radius0, nsample0, idx0, out0};
  a.s[1] = QgScale{radius1, nsample1, idx1, out1};
  return qg_dispatch(a, b, true, as_stream(stream));
}
