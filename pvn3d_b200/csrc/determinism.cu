// determinism.cu -- fixed-order backward kernels for torch.use_deterministic_algorithms(True).
//
// The PointNet++ grad ops of pn2_ops.cu scatter with float atomicAdd, and torch has no deterministic CUDA backward
// for adaptive average pooling or bilinear upsampling: in both cases the order of the float additions onto an element
// depends on the schedule.  Every kernel here instead writes each output element exactly once, as the float32 sum
// of its contributions starting from +0.0 and adding one term at a time in a fixed ascending order, so the bits do not
// depend on the schedule, the stream or the device.
//
//   * gather / group / three_interpolate grad: a per-batch inverse index (a stable radix sort of (frame, point) keys
//     carrying the slot number), the start of every point's run, then one gather-sum thread per output point that
//     walks its run in ascending slot order for a block of channels.
//   * adaptive_avg_pool2d / upsample_bilinear2d backward: one thread per input element, which enumerates the output
//     elements whose window (bin or four taps) holds it, in ascending output index.
// The sums and PSP kernels are templated on the element type of the gradients (half_io.cuh): a 16-bit form reads
// 16-bit terms, runs the same float32 sum in the same order and rounds each output element once.
#include "common.cuh"
#include "half_io.cuh"

namespace pvn3d {
namespace {

enum { kGradGather = 0, kGradInterp = 1 };   // contribution of a slot: grad_out[., slot] or grad_out[., slot/3] * w
constexpr int kSumThreads = 256;
constexpr int kSumChannels = 4;               // channels summed per pass over a point's run

// key of slot p (frame f = p / slots): f * n + idx for an index in [0, n), else the trash key b * n
template <typename Key>
__global__ void inverse_keys_kernel(const int *__restrict__ idx, long long total, long long slots, int n,
                                    Key trash, Key *__restrict__ keys, int *__restrict__ vals) {
  for (long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long f = p / slots;
    const int a = idx[p];
    keys[p] = (a >= 0 && a < n) ? static_cast<Key>(f * n + a) : trash;
    vals[p] = static_cast<int>(p - f * slots);
  }
}

// starts[q] = first position of a key >= q in the sorted keys (a binary search), for q in [0, trash]: each entry is
// written once and independently of how the keys spread
template <typename Key>
__global__ void run_starts_kernel(const Key *__restrict__ keys, long long total, Key trash,
                                  long long *__restrict__ starts) {
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q <= static_cast<long long>(trash);
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long lo = 0, hi = total;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (static_cast<long long>(keys[mid]) < q) lo = mid + 1; else hi = mid;
    }
    starts[q] = lo;
  }
}

// grad_points[f, l, i] = sum over the run of point (f, i), in ascending slot order, of the slot's term in channel l.
// Terms: grad_out[f, l, s] (kGradGather), or fl(grad_out[f, l, s / 3] * weight[f, s]) (kGradInterp; the product is
// rounded before the add: __fmul_rn keeps it out of an FMA).  src_len is grad_out's row length.  T is the element
// type of grad_out and grad_points (one thread per point: the stores stay 2-byte for a 16-bit T).
template <int kMode, typename T>
__global__ void __launch_bounds__(kSumThreads)
ordered_sum_kernel(const T *__restrict__ grad_out, const float *__restrict__ weight,
                   const long long *__restrict__ starts, const int *__restrict__ sorted_slots, int c, int n,
                   long long src_len, long long slots, T *__restrict__ grad_points) {
  const int f = blockIdx.z;
  const int i = blockIdx.x * kSumThreads + threadIdx.x;
  if (i >= n) return;
  const long long q = static_cast<long long>(f) * n + i;
  const long long s0 = starts[q], s1 = starts[q + 1];
  const float *w = weight + static_cast<size_t>(f) * slots;
  for (int l0 = blockIdx.y * kSumChannels; l0 < c; l0 += gridDim.y * kSumChannels) {
    const int nl = min(kSumChannels, c - l0);
    const T *src = grad_out + (static_cast<size_t>(f) * c + l0) * src_len;
    float acc[kSumChannels];
#pragma unroll
    for (int k = 0; k < kSumChannels; ++k) acc[k] = 0.f;
    for (long long p = s0; p < s1; ++p) {
      const int s = sorted_slots[p];
#pragma unroll
      for (int k = 0; k < kSumChannels; ++k) {
        if (k < nl) {
          float t;
          if (kMode == kGradInterp)
            t = __fmul_rn(to_f32(__ldg(src + k * src_len + s / 3)), __ldg(w + s));
          else
            t = to_f32(__ldg(src + k * src_len + s));
          acc[k] = __fadd_rn(acc[k], t);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kSumChannels; ++k)
      if (k < nl) grad_points[(static_cast<size_t>(f) * c + l0 + k) * n + i] = from_f32<T>(acc[k]);
  }
}

// ---- the inverse index: a stable LSD radix sort of (key, slot) pairs, 8 bits per pass --------------------------------
// Each pass: per-tile digit counts (digit-major, so that one exclusive scan gives every (digit, tile) its first
// output position), the scan, then a stable scatter.  A tile is kSortTile consecutive pairs handled in kSortRounds
// rounds of one pair per thread in position order; within a round __match_any_sync ranks equal digits of a warp, and
// per-warp counts in shared memory order the warps, so the scatter keeps the input order of equal digits.  Every
// buffer size is arithmetic on (b, n, slots): the workspace query never touches the device.
constexpr int kSortThreads = 256;
constexpr int kSortRounds = 8;
constexpr int kSortTile = kSortThreads * kSortRounds;
constexpr int kRadix = 256;
constexpr int kScanThreads = 1024;

template <typename Key>
__global__ void __launch_bounds__(kSortThreads)
digit_count_kernel(const Key *__restrict__ keys, long long total, long long ntiles, int shift,
                   unsigned *__restrict__ counts) {
  __shared__ unsigned s_cnt[kRadix];
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const long long base = tile * kSortTile;
    for (int r = 0; r < kSortRounds; ++r) {
      const long long p = base + r * kSortThreads + threadIdx.x;
      if (p < total) atomicAdd(&s_cnt[static_cast<int>((keys[p] >> shift) & (kRadix - 1))], 1u);
    }
    __syncthreads();
    counts[threadIdx.x * ntiles + tile] = s_cnt[threadIdx.x];
    __syncthreads();
  }
}

// out[i] = in[0] + ... + in[i - 1], one CTA walking the array in chunks
__global__ void __launch_bounds__(kScanThreads)
exclusive_scan_kernel(const unsigned *__restrict__ in, long long len, long long *__restrict__ out) {
  __shared__ long long s_warp[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long carry = 0;
  for (long long base = 0; base < len; base += kScanThreads) {
    const long long i = base + threadIdx.x;
    const long long v = i < len ? in[i] : 0;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
      long long w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    if (i < len) out[i] = carry + x - v + (warp > 0 ? s_warp[warp - 1] : 0);
    carry += s_warp[kScanThreads / 32 - 1];
    __syncthreads();
  }
}

template <typename Key>
__global__ void __launch_bounds__(kSortThreads)
digit_scatter_kernel(const Key *__restrict__ keys_in, const int *__restrict__ vals_in, long long total,
                     long long ntiles, int shift, const long long *__restrict__ first, Key *__restrict__ keys_out,
                     int *__restrict__ vals_out) {
  __shared__ unsigned s_warp[kSortThreads / 32][kRadix];   // this round's count of each digit per warp
  __shared__ unsigned s_seen[kRadix];                      // earlier rounds' count of each digit in this tile
  const int t = threadIdx.x, warp = t >> 5;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    s_seen[t] = 0;
#pragma unroll
    for (int w = 0; w < kSortThreads / 32; ++w) s_warp[w][t] = 0;
    __syncthreads();
    const long long base = tile * kSortTile;
    for (int r = 0; r < kSortRounds; ++r) {
      const long long p = base + r * kSortThreads + t;
      const bool live = p < total;
      const Key k = live ? keys_in[p] : Key(0);
      const int d = live ? static_cast<int>((k >> shift) & (kRadix - 1)) : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      const unsigned rank = __popc(peers & lanemask_lt());
      if (live && rank == 0) s_warp[warp][d] = __popc(peers);
      __syncthreads();
      if (live) {
        unsigned before = s_seen[d] + rank;
        for (int w = 0; w < warp; ++w) before += s_warp[w][d];
        const long long dst = first[static_cast<long long>(d) * ntiles + tile] + before;
        keys_out[dst] = k;
        vals_out[dst] = vals_in[p];
      }
      __syncthreads();
      unsigned add = 0;
#pragma unroll
      for (int w = 0; w < kSortThreads / 32; ++w) {
        add += s_warp[w][t];
        s_warp[w][t] = 0;
      }
      s_seen[t] += add;
      __syncthreads();
    }
  }
}

struct InverseLayout {
  bool wide;            // 64-bit keys (b * n does not fit 32 bits)
  int passes;           // 8-bit digits of the largest key (the trash key b * n)
  long long total, ntiles;
  size_t keys[2], vals[2], starts, counts, first, total_bytes;
};

static InverseLayout inverse_layout(int b, int n, long long slots) {
  InverseLayout L{};
  const unsigned long long trash = static_cast<unsigned long long>(b) * static_cast<unsigned long long>(n);
  L.wide = trash > 0xffffffffull;
  int bits = 1;
  while (bits < 64 && (trash >> bits) != 0ull) ++bits;
  L.passes = (bits + 7) / 8;
  L.total = static_cast<long long>(b) * slots;
  L.ntiles = (L.total + kSortTile - 1) / kSortTile;
  const size_t ks = L.wide ? sizeof(unsigned long long) : sizeof(unsigned);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off += align_up(bytes, 256); return at; };
  for (int i = 0; i < 2; ++i) L.keys[i] = take(ks * L.total);
  for (int i = 0; i < 2; ++i) L.vals[i] = take(sizeof(int) * L.total);
  L.starts = take(sizeof(long long) * (trash + 1));
  L.counts = take(sizeof(unsigned) * kRadix * L.ntiles);
  L.first = take(sizeof(long long) * kRadix * L.ntiles);
  L.total_bytes = off;
  return L;
}

static int launch_blocks(long long work, int per_block) {
  const long long want = (work + per_block - 1) / per_block, cap = 16ll * sm_count();
  return static_cast<int>(want < 1 ? 1 : (want < cap ? want : cap));
}

// sorts the (key, slot) pairs; returns the buffer index (0 or 1) holding the result
template <typename Key>
static int build_inverse(const int *idx, int b, int n, long long slots, const InverseLayout &L, unsigned char *ws,
                         cudaStream_t st, int *sorted) {
  const long long total = L.total;
  const Key trash = static_cast<Key>(static_cast<unsigned long long>(b) * n);
  Key *keys[2] = {reinterpret_cast<Key *>(ws + L.keys[0]), reinterpret_cast<Key *>(ws + L.keys[1])};
  int *vals[2] = {reinterpret_cast<int *>(ws + L.vals[0]), reinterpret_cast<int *>(ws + L.vals[1])};
  unsigned *counts = reinterpret_cast<unsigned *>(ws + L.counts);
  long long *first = reinterpret_cast<long long *>(ws + L.first);
  inverse_keys_kernel<Key><<<launch_blocks(total, 256), 256, 0, st>>>(idx, total, slots, n, trash, keys[0], vals[0]);
  int rc = check_launch("inverse_keys_kernel");
  const int tiles_grid = launch_blocks(L.ntiles, 1);
  int cur = 0;
  for (int pass = 0; pass < L.passes && rc == PVN3D_OK; ++pass, cur ^= 1) {
    digit_count_kernel<Key><<<tiles_grid, kSortThreads, 0, st>>>(keys[cur], total, L.ntiles, 8 * pass, counts);
    rc = check_launch("digit_count_kernel");
    if (rc != PVN3D_OK) break;
    exclusive_scan_kernel<<<1, kScanThreads, 0, st>>>(counts, kRadix * L.ntiles, first);
    rc = check_launch("exclusive_scan_kernel");
    if (rc != PVN3D_OK) break;
    digit_scatter_kernel<Key><<<tiles_grid, kSortThreads, 0, st>>>(keys[cur], vals[cur], total, L.ntiles, 8 * pass,
                                                                    first, keys[cur ^ 1], vals[cur ^ 1]);
    rc = check_launch("digit_scatter_kernel");
  }
  if (rc != PVN3D_OK) return rc;
  *sorted = cur;
  run_starts_kernel<Key><<<launch_blocks(static_cast<long long>(trash) + 1, 256), 256, 0, st>>>(
      keys[cur], total, trash, reinterpret_cast<long long *>(ws + L.starts));
  return check_launch("run_starts_kernel");
}

// the inverse index of idx (b frames of `slots` entries into [0, n)), then the ordered sums into grad_points
template <int kMode, typename T>
static int ordered_grad(const T *grad_out, const int *idx, const float *weight, int b, int c, int n,
                        long long slots, long long src_len, T *grad_points, void *workspace,
                        size_t workspace_bytes, cudaStream_t st) {
  const InverseLayout L = inverse_layout(b, n, slots);
  if (!workspace || workspace_bytes < L.total_bytes) return PVN3D_ERR_WORKSPACE;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  int sorted = 0;
  int rc = L.wide ? build_inverse<unsigned long long>(idx, b, n, slots, L, ws, st, &sorted)
                  : build_inverse<unsigned>(idx, b, n, slots, L, ws, st, &sorted);
  if (rc != PVN3D_OK) return rc;
  const int gx = ceil_div(n, kSumThreads);
  int gy = ceil_div(4 * sm_count(), gx * b);
  gy = max(1, min(gy, min(ceil_div(c, kSumChannels), 65535)));
  ordered_sum_kernel<kMode, T><<<dim3(gx, gy, b), kSumThreads, 0, st>>>(
      grad_out, weight, reinterpret_cast<const long long *>(ws + L.starts),
      reinterpret_cast<const int *>(ws + L.vals[sorted]), c, n, src_len, slots, grad_points);
  return check_launch("ordered_sum_kernel");
}

// ---- PSPNet's pooling and upsampling ------------------------------------------------------------------------------
// torch's adaptive pooling bins: [floor(o in / out), ceil((o + 1) in / out))
// (sides below 2^16, so the products fit 32 bits)
__device__ __forceinline__ int bin_start(int o, int out, int in) {
  return static_cast<int>(static_cast<unsigned>(o) * static_cast<unsigned>(in) / static_cast<unsigned>(out));
}
__device__ __forceinline__ int bin_end(int o, int out, int in) {
  return static_cast<int>((static_cast<unsigned>(o + 1) * static_cast<unsigned>(in) + out - 1) /
                          static_cast<unsigned>(out));
}

// one thread per element of the nc planes: one 64-bit division finds the plane, the rest is 32-bit within it
#define PSP_FOR_EACH_ELEMENT(nc, ih, iw)                                                                          \
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, plane = e / ((ih) * (iw));   \
       plane < (nc); e += static_cast<long long>(gridDim.x) * blockDim.x, plane = e / ((ih) * (iw)))            \
    for (int pix = static_cast<int>(e - plane * ((ih) * (iw))), y = pix / (iw), x = pix - y * (iw), once = 1;    \
         once; once = 0)

// grad_in[p, y, x] = sum over the bins (oy, ox) holding (y, x), ascending, of (g[p, oy, ox] / kW) / kH
template <typename T>
__global__ void adaptive_avg_pool2d_backward_kernel(const T *__restrict__ grad_out, long long nc, int ih,
                                                    int iw, int oh, int ow, T *__restrict__ grad_in) {

  PSP_FOR_EACH_ELEMENT(nc, ih, iw) {
    const T *g = grad_out + plane * oh * ow;
    // the bins holding y: floor(y out / in) <= o < ceil((y + 1) out / in)
    const int oy0 = bin_start(y, ih, oh), oy1 = min(bin_end(y, ih, oh), oh);
    const int ox0 = bin_start(x, iw, ow), ox1 = min(bin_end(x, iw, ow), ow);
    float acc = 0.f;
    for (int oy = oy0; oy < oy1; ++oy) {
      const float kh = static_cast<float>(bin_end(oy, oh, ih) - bin_start(oy, oh, ih));
      for (int ox = ox0; ox < ox1; ++ox) {
        const float kw = static_cast<float>(bin_end(ox, ow, iw) - bin_start(ox, ow, iw));
        const float v = to_f32(g[oy * ow + ox]);
        acc = __fadd_rn(acc, __fdiv_rn(__fdiv_rn(v, kw), kh));   // width first, as torch's backward divides
      }
    }
    grad_in[plane * ih * iw + pix] = from_f32<T>(acc);
  }
}

// torch's bilinear taps of output row / column o: i1 = (int) src, i1p = 1 if i1 < in - 1, lambda1 = src - i1,
// lambda0 = 1 - lambda1, with src = scale * o (align_corners) or max(fma(scale, o + 0.5, -0.5), 0)
struct Taps {
  int i1, i1p;
  float l0, l1;
};
__device__ __forceinline__ Taps bilinear_taps(float scale, int o, int in, bool align) {
  float src;
  if (align) {
    src = __fmul_rn(scale, static_cast<float>(o));
  } else {
    src = __fmaf_rn(scale, __fadd_rn(static_cast<float>(o), 0.5f), -0.5f);
    src = src < 0.f ? 0.f : src;
  }
  Taps t;
  t.i1 = static_cast<int>(src);
  t.i1p = t.i1 < in - 1 ? 1 : 0;
  t.l1 = __fsub_rn(src, static_cast<float>(t.i1));
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}

// the outputs whose taps can reach input row v: a window around the inverse of the source map, checked exactly
__device__ __forceinline__ void tap_window(float scale, int v, int in, int out, bool align, int &lo, int &hi) {
  if (!(scale > 0.f)) {
    lo = 0;
    hi = out - 1;
    return;
  }
  const double s = scale;
  const double a = align ? (v - 1) / s : (v - 1 + 0.5) / s - 0.5;   // src >= v - 1
  const double b = align ? (v + 1) / s : (v + 1 + 0.5) / s - 0.5;   // src < v + 1
  lo = max(0, static_cast<int>(floor(a)) - 2);
  hi = min(out - 1, static_cast<int>(ceil(b)) + 2);
}

// grad_in[p, y, x] = sum over the outputs (oy, ox) in ascending order, and over their four taps in torch's order
// (i1, j1), (i1, j1 + j1p), (i1 + i1p, j1), (i1 + i1p, j1 + j1p), of fl(fl(lambda_h lambda_w) g[p, oy, ox]) for the
// taps that land on (y, x)
template <typename T>
__global__ void upsample_bilinear2d_backward_kernel(const T *__restrict__ grad_out, long long nc, int ih,
                                                    int iw, int oh, int ow, int align, float rh, float rw,
                                                    T *__restrict__ grad_in) {
  PSP_FOR_EACH_ELEMENT(nc, ih, iw) {
    const T *g = grad_out + plane * oh * ow;
    int oy0, oy1, ox0, ox1;
    tap_window(rh, y, ih, oh, align, oy0, oy1);
    tap_window(rw, x, iw, ow, align, ox0, ox1);
    float acc = 0.f;
    for (int oy = oy0; oy <= oy1; ++oy) {
      const Taps th = bilinear_taps(rh, oy, ih, align);
      const bool h0 = th.i1 == y, h1 = th.i1 + th.i1p == y;
      if (!h0 && !h1) continue;
      for (int ox = ox0; ox <= ox1; ++ox) {
        const Taps tw = bilinear_taps(rw, ox, iw, align);
        const bool w0 = tw.i1 == x, w1 = tw.i1 + tw.i1p == x;
        if (!w0 && !w1) continue;
        const float v = to_f32(g[oy * ow + ox]);
        if (h0 && w0) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(th.l0, tw.l0), v));
        if (h0 && w1) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(th.l0, tw.l1), v));
        if (h1 && w0) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(th.l1, tw.l0), v));
        if (h1 && w1) acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(th.l1, tw.l1), v));
      }
    }
    grad_in[plane * ih * iw + pix] = from_f32<T>(acc);
  }
}

// torch's area_pixel_compute_scale for bilinear: (in - 1) / (out - 1) with align_corners (0 for out = 1), else
// 1 / scale_factor when one is given (> 0), else in / out -- in float
float bilinear_scale(int in, int out, bool align, double scale_factor) {
  if (align) return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
  if (scale_factor > 0.) return static_cast<float>(1.0 / scale_factor);
  return static_cast<float>(in) / static_cast<float>(out);
}

// sides below 2^15 and planes up to 2^30 elements keep the per-plane index arithmetic in 32 bits
bool psp_sides_supported(int ih, int iw, int oh, int ow) {
  return ih < 32768 && iw < 32768 && oh < 32768 && ow < 32768 && static_cast<long long>(ih) * iw <= (1ll << 30) &&
         static_cast<long long>(oh) * ow <= (1ll << 30);
}

int psp_grid(long long nc, int hw) { return launch_blocks(nc * hw, 256); }

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_ordered_grad_workspace_bytes(int b, int n, long long slots) {
  if (b <= 0 || n <= 0 || slots <= 0 || b > 65535 || slots > 0x7fffffffll) return 0;
  return inverse_layout(b, n, slots).total_bytes;
}

extern "C" int pvn3d_gather_points_grad_ordered(const float *grad_out, const int *idx, int b, int c, int n, int m,
                                                float *grad_points, void *workspace, size_t workspace_bytes,
                                                pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || n <= 0 || m < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  if (!grad_points || (m > 0 && (!grad_out || !idx))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  if (m == 0) {
    PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)n, as_stream(stream)), "memset");
    return PVN3D_OK;
  }
  return ordered_grad<kGradGather>(grad_out, idx, nullptr, b, c, n, m, m, grad_points, workspace, workspace_bytes,
                                   as_stream(stream));
}

extern "C" int pvn3d_group_points_grad_ordered(const float *grad_out, const int *idx, int b, int c, int n,
                                               int npoints, int nsample, float *grad_points, void *workspace,
                                               size_t workspace_bytes, pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  const long long slots = static_cast<long long>(npoints) * nsample;
  if (!grad_points || (slots > 0 && (!grad_out || !idx))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535 || slots > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
  if (slots == 0) {
    PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)n, as_stream(stream)), "memset");
    return PVN3D_OK;
  }
  return ordered_grad<kGradGather>(grad_out, idx, nullptr, b, c, n, slots, slots, grad_points, workspace,
                                   workspace_bytes, as_stream(stream));
}

extern "C" int pvn3d_three_interpolate_grad_ordered(const float *grad_out, const int *idx, const float *weight, int b,
                                                    int c, int n, int m, float *grad_points, void *workspace,
                                                    size_t workspace_bytes, pvn3d_stream_t stream) {
  if (b < 0 || c < 0 || m <= 0 || n < 0) return PVN3D_ERR_INVALID_ARG;
  if (b == 0 || c == 0) return PVN3D_OK;
  if (!grad_points || (n > 0 && (!grad_out || !idx || !weight))) return PVN3D_ERR_INVALID_ARG;
  if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
  if (n == 0) {
    PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(float) * b * c * (size_t)m, as_stream(stream)), "memset");
    return PVN3D_OK;
  }
  return ordered_grad<kGradInterp>(grad_out, idx, weight, b, c, m, 3ll * n, n, grad_points, workspace,
                                   workspace_bytes, as_stream(stream));
}

extern "C" int pvn3d_adaptive_avg_pool2d_backward(const float *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                                  float *grad_in, pvn3d_stream_t stream) {
  if (nc < 0 || ih < 0 || iw < 0 || oh <= 0 || ow <= 0) return PVN3D_ERR_INVALID_ARG;
  const long long total = nc * ih * iw;
  if (total == 0) return PVN3D_OK;
  if (!grad_out || !grad_in) return PVN3D_ERR_INVALID_ARG;
  if (!psp_sides_supported(ih, iw, oh, ow)) return PVN3D_ERR_UNSUPPORTED;
  adaptive_avg_pool2d_backward_kernel<float><<<psp_grid(nc, ih * iw), 256, 0, as_stream(stream)>>>(grad_out, nc, ih, iw, oh,
                                                                                            ow, grad_in);
  return check_launch("adaptive_avg_pool2d_backward_kernel");
}

extern "C" int pvn3d_upsample_bilinear2d_backward(const float *grad_out, long long nc, int ih, int iw, int oh, int ow,
                                                  int align_corners, double scale_h, double scale_w, float *grad_in,
                                                  pvn3d_stream_t stream) {
  if (nc < 0 || ih < 0 || iw < 0 || oh <= 0 || ow <= 0) return PVN3D_ERR_INVALID_ARG;
  const long long total = nc * ih * iw;
  if (total == 0) return PVN3D_OK;
  if (!grad_out || !grad_in) return PVN3D_ERR_INVALID_ARG;
  const bool align = align_corners != 0;
  if (!psp_sides_supported(ih, iw, oh, ow)) return PVN3D_ERR_UNSUPPORTED;
  upsample_bilinear2d_backward_kernel<float><<<psp_grid(nc, ih * iw), 256, 0, as_stream(stream)>>>(
      grad_out, nc, ih, iw, oh, ow, align ? 1 : 0, bilinear_scale(ih, oh, align, scale_h),
      bilinear_scale(iw, ow, align, scale_w), grad_in);
  return check_launch("upsample_bilinear2d_backward_kernel");
}

// ---- 16-bit forms (torch.autocast): the same inverse index and launches on __half / __nv_bfloat16 gradients --------
extern "C" int pvn3d_group_points_grad_ordered_16(int dtype, const void *grad_out, const int *idx, int b, int c, int n,
                                                  int npoints, int nsample, void *grad_points, void *workspace,
                                                  size_t workspace_bytes, pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (b < 0 || c < 0 || n <= 0 || npoints < 0 || nsample < 0) return PVN3D_ERR_INVALID_ARG;
    if (b == 0 || c == 0) return PVN3D_OK;
    const long long slots = static_cast<long long>(npoints) * nsample;
    if (!grad_points || (slots > 0 && (!grad_out || !idx))) return PVN3D_ERR_INVALID_ARG;
    if (b > 65535 || slots > 0x7fffffffll) return PVN3D_ERR_UNSUPPORTED;
    if (slots == 0) {
      PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(T) * b * c * (size_t)n, as_stream(stream)), "memset");
      return PVN3D_OK;
    }
    return ordered_grad<kGradGather>(static_cast<const T *>(grad_out), idx, nullptr, b, c, n, slots, slots,
                                     static_cast<T *>(grad_points), workspace, workspace_bytes, as_stream(stream));
  });
}

extern "C" int pvn3d_three_interpolate_grad_ordered_16(int dtype, const void *grad_out, const int *idx,
                                                       const float *weight, int b, int c, int n, int m,
                                                       void *grad_points, void *workspace, size_t workspace_bytes,
                                                       pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (b < 0 || c < 0 || m <= 0 || n < 0) return PVN3D_ERR_INVALID_ARG;
    if (b == 0 || c == 0) return PVN3D_OK;
    if (!grad_points || (n > 0 && (!grad_out || !idx || !weight))) return PVN3D_ERR_INVALID_ARG;
    if (b > 65535) return PVN3D_ERR_UNSUPPORTED;
    if (n == 0) {
      PVN3D_CUDA_TRY(cudaMemsetAsync(grad_points, 0, sizeof(T) * b * c * (size_t)m, as_stream(stream)), "memset");
      return PVN3D_OK;
    }
    return ordered_grad<kGradInterp>(static_cast<const T *>(grad_out), idx, weight, b, c, m, 3ll * n, n,
                                     static_cast<T *>(grad_points), workspace, workspace_bytes, as_stream(stream));
  });
}

extern "C" int pvn3d_adaptive_avg_pool2d_backward_16(int dtype, const void *grad_out, long long nc, int ih, int iw,
                                                     int oh, int ow, void *grad_in, pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (nc < 0 || ih < 0 || iw < 0 || oh <= 0 || ow <= 0) return PVN3D_ERR_INVALID_ARG;
    const long long total = nc * ih * iw;
    if (total == 0) return PVN3D_OK;
    if (!grad_out || !grad_in) return PVN3D_ERR_INVALID_ARG;
    if (!psp_sides_supported(ih, iw, oh, ow)) return PVN3D_ERR_UNSUPPORTED;
    adaptive_avg_pool2d_backward_kernel<T><<<psp_grid(nc, ih * iw), 256, 0, as_stream(stream)>>>(
        static_cast<const T *>(grad_out), nc, ih, iw, oh, ow, static_cast<T *>(grad_in));
    return check_launch("adaptive_avg_pool2d_backward_kernel");
  });
}

extern "C" int pvn3d_upsample_bilinear2d_backward_16(int dtype, const void *grad_out, long long nc, int ih, int iw,
                                                     int oh, int ow, int align_corners, double scale_h, double scale_w,
                                                     void *grad_in, pvn3d_stream_t stream) {
  return with_dtype16(dtype, [&](auto tag) -> int {
    using T = decltype(tag);
    if (nc < 0 || ih < 0 || iw < 0 || oh <= 0 || ow <= 0) return PVN3D_ERR_INVALID_ARG;
    const long long total = nc * ih * iw;
    if (total == 0) return PVN3D_OK;
    if (!grad_out || !grad_in) return PVN3D_ERR_INVALID_ARG;
    const bool align = align_corners != 0;
    if (!psp_sides_supported(ih, iw, oh, ow)) return PVN3D_ERR_UNSUPPORTED;
    upsample_bilinear2d_backward_kernel<T><<<psp_grid(nc, ih * iw), 256, 0, as_stream(stream)>>>(
        static_cast<const T *>(grad_out), nc, ih, iw, oh, ow, align ? 1 : 0, bilinear_scale(ih, oh, align, scale_h),
        bilinear_scale(iw, ow, align, scale_w), static_cast<T *>(grad_in));
    return check_launch("upsample_bilinear2d_backward_kernel");
  });
}
