// train.cu -- PVN3D's training targets and losses on device:
//
//   train_targets  the regression targets get_item builds from the sampled cloud (reference
//                  pvn3d/datasets/ycb/ycb_dataset.py:241-278, linemod_dataset.py:275-310): every slot's keypoints and
//                  centre moved by its float64 meta pose, and each point's offsets to the keypoints / centre of the
//                  slot whose class is the point's label.  One pass over the points; the frame's slot table
//                  (float64) and the label -> slot map sit in shared memory, the K*3 + 3 floats of a tile of points
//                  are stored coalesced.
//   train_loss     model_fn's three terms (train_ycb_pvn3d.py:172-184): FocalLoss(gamma) on the segmentation logits
//                  and OFLoss on the keypoint and centre offsets (lib/loss.py), forward and backward.  The forward is
//                  two launches (per-block partials of all terms in one grid, then one block that combines them in a
//                  fixed order); the backward is one launch.  No float atomics anywhere: two calls give the same bits.
#include <math.h>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kTgtThreads = 256;           // points per block of train_targets_kernel
constexpr int kTgtMaxSmem = 48 * 1024;
constexpr int kTgtMaxClasses = 4096;
constexpr int kLossTile = 128;             // logits rows / points per block of the loss kernels (one per thread)
constexpr int kLossWarps = kLossTile / 32;
constexpr int kLossMaxClasses = 128;
constexpr int kLossMaxKp = 48;
constexpr int kLossMaxSmem = 96 * 1024;
constexpr int kFinThreads = 256;

// ---------------------------------------------------------------------------------------------------------------
// targets
// ---------------------------------------------------------------------------------------------------------------

// numpy's `np.dot(p, r.T) + t` for one float32 point p and a float64 pose: p is promoted, three products summed left
// to right, then the translation (no contraction, so the float64 value does not depend on the compiler).
__device__ __forceinline__ double rt_row(const double *rt, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, rt[0]), __dmul_rn(y, rt[1])), __dmul_rn(z, rt[2])), rt[3]);
}

// grid (ceil(n / kTgtThreads), b).  Shared: pts[s][(k+1)*3] f64 (k keypoints, then the centre), map[n_cls] i32,
// slot[kTgtThreads] i32.
__global__ void __launch_bounds__(kTgtThreads)
    train_targets_kernel(const float *__restrict__ pcld, const int *__restrict__ labels, const int *__restrict__ cls_ids,
                         const double *__restrict__ rts, int n, int s, const float *__restrict__ kp_table,
                         const float *__restrict__ ctr_table, int n_cls, int k, float *__restrict__ kp_targ,
                         float *__restrict__ ctr_targ, float *__restrict__ kp3ds, float *__restrict__ ctr3ds) {
  extern __shared__ double s_pts[];
  const int b = blockIdx.y;
  const int kc = (k + 1) * 3;
  int *s_map = reinterpret_cast<int *>(s_pts + static_cast<size_t>(s) * kc);
  int *s_slot = s_map + n_cls;
  const int *ids = cls_ids + static_cast<size_t>(b) * s;

  for (int c = threadIdx.x; c < n_cls; c += blockDim.x) s_map[c] = -1;
  for (int e = threadIdx.x; e < s * (k + 1); e += blockDim.x) {
    const int slot = e / (k + 1), j = e - slot * (k + 1);
    const int c = ids[slot];
    double o0 = 0.0, o1 = 0.0, o2 = 0.0;
    if (c >= 1 && c < n_cls) {  // any other id is an empty slot: zeros, and the tables are never read
      const float *src = j < k ? kp_table + (static_cast<size_t>(c) * k + j) * 3 : ctr_table + static_cast<size_t>(c) * 3;
      const double x = src[0], y = src[1], z = src[2];
      const double *rt = rts + (static_cast<size_t>(b) * s + slot) * 12;
      o0 = rt_row(rt, x, y, z);
      o1 = rt_row(rt + 4, x, y, z);
      o2 = rt_row(rt + 8, x, y, z);
    }
    double *d = s_pts + static_cast<size_t>(slot) * kc + j * 3;
    d[0] = o0;
    d[1] = o1;
    d[2] = o2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int slot = 0; slot < s; ++slot) {  // in meta order: a class listed twice keeps its LAST slot, as the
      const int c = ids[slot];               // reference loop overwrites
      if (c >= 1 && c < n_cls) s_map[c] = slot;
    }
  }
  if (blockIdx.x == 0) {
    for (int e = threadIdx.x; e < s * kc; e += blockDim.x) {
      const int slot = e / kc, r = e - slot * kc;
      const float v = __double2float_rn(s_pts[e]);
      if (r < k * 3)
        kp3ds[(static_cast<size_t>(b) * s + slot) * k * 3 + r] = v;
      else
        ctr3ds[(static_cast<size_t>(b) * s + slot) * 3 + (r - k * 3)] = v;
    }
  }
  __syncthreads();
  const int p0 = blockIdx.x * kTgtThreads;
  const int np = min(kTgtThreads, n - p0);
  const size_t row0 = static_cast<size_t>(b) * n + p0;
  if (static_cast<int>(threadIdx.x) < np) {
    const int l = labels[row0 + threadIdx.x];
    s_slot[threadIdx.x] = (l >= 0 && l < n_cls) ? s_map[l] : -1;
  }
  __syncthreads();
  const float *cld = pcld + row0 * 3;
  const int k3 = k * 3;
  float *kout = kp_targ + row0 * k3;
  for (int e = threadIdx.x; e < np * k3; e += blockDim.x) {
    const int p = e / k3, r = e - p * k3;  // r = keypoint * 3 + axis
    const int slot = s_slot[p];
    float v = 0.f;
    if (slot >= 0) v = __double2float_rn(__dsub_rn(static_cast<double>(cld[p * 3 + r % 3]), s_pts[slot * kc + r]));
    kout[e] = v;
  }
  float *cout = ctr_targ + row0 * 3;
  for (int e = threadIdx.x; e < np * 3; e += blockDim.x) {
    const int p = e / 3, r = e - p * 3;
    const int slot = s_slot[p];
    float v = 0.f;
    if (slot >= 0) v = __double2float_rn(__dsub_rn(static_cast<double>(cld[e]), s_pts[slot * kc + k3 + r]));
    cout[e] = v;
  }
}

size_t targets_smem(int s, int k, int n_cls) {
  return static_cast<size_t>(s) * (k + 1) * 3 * sizeof(double) + static_cast<size_t>(n_cls + kTgtThreads) * sizeof(int);
}

// ---------------------------------------------------------------------------------------------------------------
// losses
// ---------------------------------------------------------------------------------------------------------------

// Where each block of the loss grids works: blocks [0, seg_blocks) take kLossTile logits rows each, then
// kp_blocks = b * tiles blocks the keypoint offsets, then as many the centre offsets (tiles = ceil(n / kLossTile)).
struct LossPlan {
  pvn3d_loss_args_t a;
  long long seg_blocks;
  int tiles, kp_blocks, ctr_blocks;
  // workspace (byte offsets)
  size_t off_m, off_den, off_seg_sum, off_seg_hit, off_kp, off_kp_cnt, off_ctr, off_ctr_cnt, off_vals, bytes;
};

__host__ __device__ inline size_t al(size_t x) { return (x + 255) / 256 * 256; }

// (1 - pt)^gamma as torch.pow gives it for the reference's `(1-pt)**self.gamma`: 0^0 = 1, x^2 = x*x
__device__ __forceinline__ float focal_factor(float x, float gamma) {
  if (gamma == 0.f) return 1.f;
  if (gamma == 1.f) return x;
  if (gamma == 2.f) return x * x;
  return powf(x, gamma);
}

__device__ __forceinline__ size_t seg_addr(long long row, int j, int n_cls, int inner) {
  // [rows, n_cls] when inner == 1; [rows / inner, n_cls, inner] (FocalLoss's N,C,H,W input) otherwise
  return (static_cast<size_t>(row / inner) * n_cls + j) * inner + static_cast<size_t>(row % inner);
}

// The logits of rows r0 .. r0+nr-1 into s[j * (kLossTile + 1) + r] (one row per thread afterwards, conflict-free).
__device__ void stage_seg(float *s, const float *seg, long long r0, int nr, int n_cls, int inner) {
  if (inner == 1) {
    const float *src = seg + static_cast<size_t>(r0) * n_cls;
    for (int e = threadIdx.x; e < nr * n_cls; e += blockDim.x) {
      const int r = e / n_cls, j = e - r * n_cls;
      s[j * (kLossTile + 1) + r] = src[e];
    }
  } else {
    for (int e = threadIdx.x; e < nr * n_cls; e += blockDim.x) {
      const int j = e / nr, r = e - j * nr;
      s[j * (kLossTile + 1) + r] = seg[seg_addr(r0 + r, j, n_cls, inner)];
    }
  }
}

struct RowStats {
  float mx, sum, logpt;
  int arg;
};

// log_softmax's max and sum of exp, the target's log-probability (NaN for a target outside [0, C)) and the first
// maximal index (torch.max / pvn3d_seg_argmax: strict '>', a leading NaN is replaced by the first number)
__device__ __forceinline__ RowStats row_stats(const float *s, int r, int n_cls, long long t) {
  RowStats o;
  o.mx = s[r];
  o.arg = 0;
  for (int j = 1; j < n_cls; ++j) {
    const float v = s[j * (kLossTile + 1) + r];
    if (v > o.mx || (o.mx != o.mx && v == v)) {
      o.mx = v;
      o.arg = j;
    }
  }
  float sum = 0.f;
  for (int j = 0; j < n_cls; ++j) sum += expf(s[j * (kLossTile + 1) + r] - o.mx);
  o.sum = sum;
  o.logpt = (t >= 0 && t < n_cls) ? (s[static_cast<int>(t) * (kLossTile + 1) + r] - o.mx) - logf(sum) : __int_as_float(0x7fc00000);
  return o;
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ bool row_in(const pvn3d_loss_args_t &a, long long row) {
  return a.ok == nullptr || a.ok[row / a.n] != 0;
}

// Stage the [np, K, 3] offset targets of tile `tile` of frame b and the tile's weights (labels > 0); returns np.
__device__ int stage_of(float *s_t, float *s_w, const float *targ, const long long *labels, int b, int n, int kk,
                        int tile) {
  const int p0 = tile * kLossTile;
  const int np = min(kLossTile, n - p0);
  const float *src = targ + (static_cast<size_t>(b) * n + p0) * kk * 3;
  for (int e = threadIdx.x; e < np * kk * 3; e += blockDim.x) s_t[e] = src[e];
  if (static_cast<int>(threadIdx.x) < np)
    s_w[threadIdx.x] = labels[static_cast<size_t>(b) * n + p0 + threadIdx.x] > 0 ? 1.f : 0.f;  // labels > 1e-8
  __syncthreads();
  return np;
}

__global__ void __launch_bounds__(kLossTile)
    train_loss_partials_kernel(const __grid_constant__ LossPlan pl, unsigned char *__restrict__ ws) {
  extern __shared__ float s_dyn[];
  __shared__ float s_red[kLossWarps * kLossMaxKp];
  __shared__ int s_cnt[kLossWarps];
  const pvn3d_loss_args_t &a = pl.a;
  const int warp = threadIdx.x >> 5;
  long long blk = blockIdx.x;
  if (blk < pl.seg_blocks) {
    const long long r0 = blk * kLossTile;
    const int nr = static_cast<int>(min(static_cast<long long>(kLossTile), a.seg_rows - r0));
    stage_seg(s_dyn, a.seg, r0, nr, a.n_cls, a.seg_inner);
    __syncthreads();
    float loss = 0.f;
    int hit = 0;
    const int r = threadIdx.x;
    if (r < nr && row_in(a, r0 + r)) {
      const long long t = a.seg_target[r0 + r];
      const RowStats st = row_stats(s_dyn, r, a.n_cls, t);
      const float pt = expf(st.logpt);  // detached in the reference: Variable(logpt.data.exp())
      loss = -focal_factor(1.f - pt, a.gamma) * st.logpt;
      hit = st.arg == t;
    }
    loss = warp_sum(loss);
    hit = warp_sum_i(hit);
    if ((threadIdx.x & 31) == 0) {
      s_red[warp] = loss;
      s_cnt[warp] = hit;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float v = 0.f;
      int h = 0;
      for (int w = 0; w < kLossWarps; ++w) {
        v += s_red[w];
        h += s_cnt[w];
      }
      reinterpret_cast<float *>(ws + pl.off_seg_sum)[blk] = v;
      reinterpret_cast<int *>(ws + pl.off_seg_hit)[blk] = h;
    }
    return;
  }
  blk -= pl.seg_blocks;
  const bool kp = blk < pl.kp_blocks;
  if (!kp) blk -= pl.kp_blocks;
  const int kk = kp ? a.n_kp : a.n_ctr;
  const float *pred = kp ? a.kp_pred : a.ctr_pred;
  const int b = static_cast<int>(blk / pl.tiles), tile = static_cast<int>(blk % pl.tiles);
  float *s_t = s_dyn;
  float *s_w = s_dyn + kLossTile * kk * 3;
  const int np = stage_of(s_t, s_w, kp ? a.kp_targ : a.ctr_targ, a.labels, b, a.n, kk, tile);
  const int p0 = tile * kLossTile;
  for (int k = 0; k < kk; ++k) {
    const float *pk = pred + ((static_cast<size_t>(b) * kk + k) * a.n + p0) * 3;
    float acc = 0.f;
    for (int e = threadIdx.x; e < np * 3; e += blockDim.x) {
      const int p = e / 3, c = e - p * 3;
      acc += s_w[p] * fabsf(pk[e] - s_t[(p * kk + k) * 3 + c]);  // w * |diff|: a NaN diff stays NaN at w = 0
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_red[warp * kLossMaxKp + k] = acc;
  }
  int cnt = 0;
  if (static_cast<int>(threadIdx.x) < np) cnt = s_w[threadIdx.x] != 0.f;
  cnt = warp_sum_i(cnt);
  if ((threadIdx.x & 31) == 0) s_cnt[warp] = cnt;
  __syncthreads();
  float *part = reinterpret_cast<float *>(ws + (kp ? pl.off_kp : pl.off_ctr)) + blk * kk;
  for (int k = threadIdx.x; k < kk; k += blockDim.x) {
    float v = 0.f;
    for (int w = 0; w < kLossWarps; ++w) v += s_red[w * kLossMaxKp + k];
    part[k] = v;
  }
  if (threadIdx.x == 0) {
    int c = 0;
    for (int w = 0; w < kLossWarps; ++w) c += s_cnt[w];
    reinterpret_cast<int *>(ws + (kp ? pl.off_kp_cnt : pl.off_ctr_cnt))[blk] = c;
  }
}

// One block: every sum over blocks in a fixed order (float64), then the per-(frame, keypoint) OF terms, the focal
// mean, the weighted total and the accuracy.  Keeps the focal divisor and the OF denominators for the backward.
__global__ void __launch_bounds__(kFinThreads)
    train_loss_finish_kernel(const __grid_constant__ LossPlan pl, unsigned char *__restrict__ ws, float *kp_loss,
                             float *ctr_loss, float *loss, float *parts, float *acc) {
  __shared__ double s_d[kFinThreads];
  __shared__ long long s_h[kFinThreads];
  const pvn3d_loss_args_t &a = pl.a;
  float *m_out = reinterpret_cast<float *>(ws + pl.off_m);
  float *den = reinterpret_cast<float *>(ws + pl.off_den);
  float *vals = reinterpret_cast<float *>(ws + pl.off_vals);
  float focal = 0.f, accv = 0.f;
  if (pl.seg_blocks > 0) {
    const float *ps = reinterpret_cast<const float *>(ws + pl.off_seg_sum);
    const int *ph = reinterpret_cast<const int *>(ws + pl.off_seg_hit);
    double v = 0.0;
    long long h = 0;
    for (long long i = threadIdx.x; i < pl.seg_blocks; i += blockDim.x) {
      v += ps[i];
      h += ph[i];
    }
    s_d[threadIdx.x] = v;
    s_h[threadIdx.x] = h;
    __syncthreads();
    for (int st = kFinThreads / 2; st > 0; st >>= 1) {
      if (static_cast<int>(threadIdx.x) < st) {
        s_d[threadIdx.x] += s_d[threadIdx.x + st];
        s_h[threadIdx.x] += s_h[threadIdx.x + st];
      }
      __syncthreads();
    }
    long long m = a.seg_rows;
    if (a.ok) {
      int nok = 0;
      for (int f = 0; f < a.b; ++f) nok += a.ok[f] != 0;
      m = static_cast<long long>(nok) * a.n;
    }
    const float mf = static_cast<float>(m);
    const float sum = static_cast<float>(s_d[0]);
    if (!a.seg_mean)
      focal = sum;
    else if (m > 0)
      focal = sum / mf;
    else
      focal = a.ok ? 0.f : __int_as_float(0x7fc00000);   // no ok frame: nothing to learn from
    accv = m > 0 ? static_cast<float>(static_cast<double>(s_h[0]) / static_cast<double>(m)) : 0.f;
    if (threadIdx.x == 0) m_out[0] = a.seg_mean ? mf : -1.f;   // -1: sum, no divisor
  }
  // OF terms: in_loss[b,k] = sum_{n,c} w |diff| / (sum_n w + 1e-3), both sums in float32 as lib/loss.py's
  for (int term = 0; term < 2; ++term) {
    const int kk = term == 0 ? a.n_kp : a.n_ctr;
    const int blocks = term == 0 ? pl.kp_blocks : pl.ctr_blocks;
    if (blocks == 0) continue;
    const float *part = reinterpret_cast<const float *>(ws + (term == 0 ? pl.off_kp : pl.off_ctr));
    const int *pc = reinterpret_cast<const int *>(ws + (term == 0 ? pl.off_kp_cnt : pl.off_ctr_cnt));
    float *out = term == 0 ? kp_loss : ctr_loss;
    for (int i = threadIdx.x; i < a.b * kk; i += blockDim.x) {
      const int b = i / kk, k = i - b * kk;
      double s = 0.0;
      int c = 0;
      for (int t = 0; t < pl.tiles; ++t) {
        s += part[(static_cast<size_t>(b) * pl.tiles + t) * kk + k];
        c += pc[b * pl.tiles + t];
      }
      const float d = __fadd_rn(static_cast<float>(c), 1e-3f);
      const float v = __fdiv_rn(static_cast<float>(s), d);
      if (out) out[i] = v;
      vals[term * a.b * kLossMaxKp + i] = v;
      if (k == 0 && term == 0) den[b] = d;
      if (k == 0 && term == 1 && pl.kp_blocks == 0) den[b] = d;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sk = 0.f, sc = 0.f;
    for (int i = 0; i < a.b * a.n_kp && pl.kp_blocks; ++i) sk += vals[i];
    for (int i = 0; i < a.b * a.n_ctr && pl.ctr_blocks; ++i) sc += vals[a.b * kLossMaxKp + i];
    if (loss) loss[0] = a.w_seg * focal + a.w_kp * sk + a.w_ctr * sc;
    if (parts) {
      parts[0] = focal;
      parts[1] = sk;
      parts[2] = sc;
    }
    if (acc) acc[0] = accv;
  }
}

struct GradIn {
  const float *g_loss, *g_parts, *g_kp;
};

__global__ void __launch_bounds__(kLossTile)
    train_loss_backward_kernel(const __grid_constant__ LossPlan pl, GradIn g, const unsigned char *__restrict__ ws,
                               float *__restrict__ d_seg, float *__restrict__ d_kp, float *__restrict__ d_ctr) {
  extern __shared__ float s_dyn[];
  const pvn3d_loss_args_t &a = pl.a;
  const float gl = g.g_loss ? g.g_loss[0] : 0.f;
  long long blk = blockIdx.x;
  if (blk < pl.seg_blocks) {
    const long long r0 = blk * kLossTile;
    const int nr = static_cast<int>(min(static_cast<long long>(kLossTile), a.seg_rows - r0));
    stage_seg(s_dyn, a.seg, r0, nr, a.n_cls, a.seg_inner);
    __syncthreads();
    const float m = reinterpret_cast<const float *>(ws + pl.off_m)[0];
    const float gf = a.w_seg * gl + (g.g_parts ? g.g_parts[0] : 0.f);
    // d loss / d z_j = -(g / M) (1 - pt)^gamma (delta_jt - p_j): pt is a constant (detached in the reference)
    const float scale = m < 0.f ? gf : (m > 0.f ? gf / m : 0.f);
    const int r = threadIdx.x;
    if (r < nr) {
      if (!row_in(a, r0 + r)) {
        for (int j = 0; j < a.n_cls; ++j) s_dyn[j * (kLossTile + 1) + r] = 0.f;
      } else {
        const long long t = a.seg_target[r0 + r];
        const RowStats st = row_stats(s_dyn, r, a.n_cls, t);
        const float pt = expf(st.logpt);
        const float gg = scale * -focal_factor(1.f - pt, a.gamma);   // gradient of logpt (NaN row stays NaN)
        const float lse = logf(st.sum);
        for (int j = 0; j < a.n_cls; ++j) {
          float &z = s_dyn[j * (kLossTile + 1) + r];
          const float p = expf((z - st.mx) - lse);                   // exp(log_softmax)
          z = __fmaf_rn(-p, gg, j == t ? gg : 0.f);                  // log_softmax backward: g_j - p_j sum(g)
        }
      }
    }
    __syncthreads();
    if (a.seg_inner == 1) {
      float *dst = d_seg + static_cast<size_t>(r0) * a.n_cls;
      for (int e = threadIdx.x; e < nr * a.n_cls; e += blockDim.x) {
        const int rr = e / a.n_cls, j = e - rr * a.n_cls;
        dst[e] = s_dyn[j * (kLossTile + 1) + rr];
      }
    } else {
      for (int e = threadIdx.x; e < nr * a.n_cls; e += blockDim.x) {
        const int j = e / nr, rr = e - j * nr;
        d_seg[seg_addr(r0 + rr, j, a.n_cls, a.seg_inner)] = s_dyn[j * (kLossTile + 1) + rr];
      }
    }
    return;
  }
  blk -= pl.seg_blocks;
  const bool kp = blk < pl.kp_blocks;
  if (!kp) blk -= pl.kp_blocks;
  const int kk = kp ? a.n_kp : a.n_ctr;
  const float *pred = kp ? a.kp_pred : a.ctr_pred;
  float *grad = kp ? d_kp : d_ctr;
  const int b = static_cast<int>(blk / pl.tiles), tile = static_cast<int>(blk % pl.tiles);
  float *s_t = s_dyn;
  float *s_w = s_dyn + kLossTile * kk * 3;
  const int np = stage_of(s_t, s_w, kp ? a.kp_targ : a.ctr_targ, a.labels, b, a.n, kk, tile);
  const int p0 = tile * kLossTile;
  const float den = reinterpret_cast<const float *>(ws + pl.off_den)[b];
  const float gw = (kp ? a.w_kp : a.w_ctr) * gl + (g.g_parts ? g.g_parts[kp ? 1 : 2] : 0.f);
  for (int k = 0; k < kk; ++k) {
    const float gk = gw + (kp && g.g_kp ? g.g_kp[b * kk + k] : 0.f);
    const float q = __fdiv_rn(gk, den);  // d(S / den) / dS
    const size_t base = ((static_cast<size_t>(b) * kk + k) * a.n + p0) * 3;
    for (int e = threadIdx.x; e < np * 3; e += blockDim.x) {
      const int p = e / 3, c = e - p * 3;
      const float d = pred[base + e] - s_t[(p * kk + k) * 3 + c];
      const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);   // torch.abs's backward: sign(0) = sign(NaN) = 0
      grad[base + e] = (q * s_w[p]) * sg;
    }
  }
}

int loss_plan(const pvn3d_loss_args_t *a, LossPlan *pl, size_t *smem) {
  if (!a) return PVN3D_ERR_INVALID_ARG;
  *pl = LossPlan{};
  pl->a = *a;
  const bool seg = a->seg != nullptr, kp = a->kp_pred != nullptr, ctr = a->ctr_pred != nullptr;
  if (!seg && !kp && !ctr) return PVN3D_ERR_INVALID_ARG;
  size_t need = 0;
  if (seg) {
    if (!a->seg_target || a->seg_rows < 1 || a->n_cls < 1 || a->seg_inner < 1 || a->seg_rows % a->seg_inner != 0 ||
        !(a->gamma >= 0.f) || isinf(a->gamma))
      return PVN3D_ERR_INVALID_ARG;
    if (a->n_cls > kLossMaxClasses) return PVN3D_ERR_UNSUPPORTED;
    pl->seg_blocks = (a->seg_rows + kLossTile - 1) / kLossTile;
    need = static_cast<size_t>(a->n_cls) * (kLossTile + 1) * sizeof(float);
  } else {
    pl->a.seg_target = nullptr;
  }
  if (kp || ctr || a->ok) {
    if (a->b < 1 || a->n < 1) return PVN3D_ERR_INVALID_ARG;
  }
  if (a->ok && (!seg || a->seg_rows != static_cast<long long>(a->b) * a->n)) return PVN3D_ERR_INVALID_ARG;
  if (kp || ctr) {
    if (!a->labels) return PVN3D_ERR_INVALID_ARG;
    pl->tiles = (a->n + kLossTile - 1) / kLossTile;
    if (static_cast<long long>(a->b) * pl->tiles > 0x3fffffff) return PVN3D_ERR_UNSUPPORTED;
  }
  if (kp) {
    if (!a->kp_targ || a->n_kp < 1) return PVN3D_ERR_INVALID_ARG;
    if (a->n_kp > kLossMaxKp) return PVN3D_ERR_UNSUPPORTED;
    pl->kp_blocks = a->b * pl->tiles;
    need = max(need, static_cast<size_t>(kLossTile) * (a->n_kp * 3 + 1) * sizeof(float));
  } else {
    pl->a.n_kp = 0;
  }
  if (ctr) {
    if (!a->ctr_targ || a->n_ctr < 1) return PVN3D_ERR_INVALID_ARG;
    if (a->n_ctr > kLossMaxKp) return PVN3D_ERR_UNSUPPORTED;
    pl->ctr_blocks = a->b * pl->tiles;
    need = max(need, static_cast<size_t>(kLossTile) * (a->n_ctr * 3 + 1) * sizeof(float));
  } else {
    pl->a.n_ctr = 0;
  }
  if (pl->seg_blocks + pl->kp_blocks + pl->ctr_blocks > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  const int bb = (kp || ctr) ? a->b : 1;
  size_t o = 0;
  pl->off_m = o;
  o = al(o + sizeof(float));
  pl->off_den = o;
  o = al(o + sizeof(float) * bb);
  pl->off_seg_sum = o;
  o = al(o + sizeof(float) * pl->seg_blocks);
  pl->off_seg_hit = o;
  o = al(o + sizeof(int) * pl->seg_blocks);
  pl->off_kp = o;
  o = al(o + sizeof(float) * pl->kp_blocks * pl->a.n_kp);
  pl->off_kp_cnt = o;
  o = al(o + sizeof(int) * pl->kp_blocks);
  pl->off_ctr = o;
  o = al(o + sizeof(float) * pl->ctr_blocks * pl->a.n_ctr);
  pl->off_ctr_cnt = o;
  o = al(o + sizeof(int) * pl->ctr_blocks);
  pl->off_vals = o;
  o = al(o + sizeof(float) * 2 * bb * kLossMaxKp);
  pl->bytes = o;
  *smem = need;
  return PVN3D_OK;
}

// Opt in on every device's first call, whatever this call's footprint: the partials kernel also holds static shared
// memory (s_red, s_cnt), and the launch limit without the opt-in is 48 KB for static and dynamic together, so a
// dynamic size just under 48 KB (the focal tile at C = 94, 95) would otherwise be refused.
int loss_smem_setup() {
  static PerDeviceOnce once;
  PVN3D_ONCE_PER_DEVICE(once,
                        cudaFuncSetAttribute(train_loss_partials_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kLossMaxSmem),
                        "train_loss_partials smem");
  static PerDeviceOnce once_b;
  PVN3D_ONCE_PER_DEVICE(once_b,
                        cudaFuncSetAttribute(train_loss_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kLossMaxSmem),
                        "train_loss_backward smem");
  return PVN3D_OK;
}

int loss_workspace_check(const LossPlan &pl, const void *ws, size_t ws_bytes) {
  if (!ws) return PVN3D_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(ws) & 255u) return PVN3D_ERR_INVALID_ARG;
  if (ws_bytes < pl.bytes) return PVN3D_ERR_WORKSPACE;
  return PVN3D_OK;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_train_targets(const float *pcld, const int *labels, const int *cls_ids, const double *rts, int b,
                                   int n, int s, const float *kp_table, const float *ctr_table, int n_cls, int k,
                                   float *kp_targ, float *ctr_targ, float *kp3ds, float *ctr3ds,
                                   pvn3d_stream_t stream) {
  if (!pcld || !labels || !cls_ids || !rts || !kp_table || !ctr_table || !kp_targ || !ctr_targ || !kp3ds || !ctr3ds ||
      b < 1 || n < 1 || s < 1 || n_cls < 1 || k < 1)
    return PVN3D_ERR_INVALID_ARG;
  if (b > 65535 || n_cls > kTgtMaxClasses || targets_smem(s, k, n_cls) > kTgtMaxSmem ||
      static_cast<long long>(kTgtThreads) * k * 3 > 0x7fffffffll)
    return PVN3D_ERR_UNSUPPORTED;
  const dim3 grid(static_cast<unsigned>(ceil_div(n, kTgtThreads)), static_cast<unsigned>(b));
  train_targets_kernel<<<grid, kTgtThreads, targets_smem(s, k, n_cls), as_stream(stream)>>>(
      pcld, labels, cls_ids, rts, n, s, kp_table, ctr_table, n_cls, k, kp_targ, ctr_targ, kp3ds, ctr3ds);
  return check_launch("train_targets_kernel");
}

extern "C" size_t pvn3d_train_loss_workspace_bytes(const pvn3d_loss_args_t *args) {
  LossPlan pl;
  size_t smem = 0;
  if (loss_plan(args, &pl, &smem) != PVN3D_OK) return 0;
  return pl.bytes;
}

extern "C" int pvn3d_train_loss_forward(const pvn3d_loss_args_t *args, float *loss, float *parts, float *kp_loss,
                                        float *ctr_loss, float *acc, void *workspace, size_t workspace_bytes,
                                        pvn3d_stream_t stream) {
  LossPlan pl;
  size_t smem = 0;
  int rc = loss_plan(args, &pl, &smem);
  if (rc != PVN3D_OK) return rc;
  if ((rc = loss_workspace_check(pl, workspace, workspace_bytes)) != PVN3D_OK) return rc;
  if ((rc = loss_smem_setup()) != PVN3D_OK) return rc;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  const unsigned grid = static_cast<unsigned>(pl.seg_blocks + pl.kp_blocks + pl.ctr_blocks);
  train_loss_partials_kernel<<<grid, kLossTile, smem, as_stream(stream)>>>(pl, ws);
  if ((rc = check_launch("train_loss_partials_kernel")) != PVN3D_OK) return rc;
  train_loss_finish_kernel<<<1, kFinThreads, 0, as_stream(stream)>>>(pl, ws, kp_loss, ctr_loss, loss, parts, acc);
  return check_launch("train_loss_finish_kernel");
}

extern "C" int pvn3d_train_loss_backward(const pvn3d_loss_args_t *args, const float *g_loss, const float *g_parts,
                                         const float *g_kp, float *d_seg, float *d_kp, float *d_ctr,
                                         const void *workspace, size_t workspace_bytes, pvn3d_stream_t stream) {
  LossPlan pl;
  size_t smem = 0;
  int rc = loss_plan(args, &pl, &smem);
  if (rc != PVN3D_OK) return rc;
  if ((rc = loss_workspace_check(pl, workspace, workspace_bytes)) != PVN3D_OK) return rc;
  if ((pl.seg_blocks && !d_seg) || (pl.kp_blocks && !d_kp) || (pl.ctr_blocks && !d_ctr) || (!g_loss && !g_parts && !g_kp))
    return PVN3D_ERR_INVALID_ARG;
  if ((rc = loss_smem_setup()) != PVN3D_OK) return rc;
  const unsigned grid = static_cast<unsigned>(pl.seg_blocks + pl.kp_blocks + pl.ctr_blocks);
  train_loss_backward_kernel<<<grid, kLossTile, smem, as_stream(stream)>>>(
      pl, GradIn{g_loss, g_parts, g_kp}, static_cast<const unsigned char *>(workspace), d_seg, d_kp, d_ctr);
  return check_launch("train_loss_backward_kernel");
}
