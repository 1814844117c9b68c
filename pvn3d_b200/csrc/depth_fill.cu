// depth_fill.cu -- ip_basic's multiscale depth completion as Basic_Utils.fill_missing runs it for YCB
// (fill_in_multiscale with max_depth 3, extrapolate False, blur 'bilateral'), batched on the stream.
//
// One thread per pixel, frames along grid.z.  The stages ping-pong between two whole-batch images in
// the workspace (a 16-frame YCB batch is 20 MB, resident in L2); a kernel boundary sits wherever the
// next stage needs neighbours of the previous one, a column scan or the frame's min/max:
//   init           top rows := H, min/max keys := empty
//   s2             s1 and the three binned cross dilations, from the depth itself     -> A
//   close          5x5 dilate (A -> B), 5x5 erode (B -> A)                             s3 in A
//   s4             masked median; top1 by atomicMin                                     -> B
//   s5             9x9 hole fill under top1; top2 by atomicMin                          -> A
//   fill x6        masked 5x5 dilation under top2                                       A <-> B, ends in A
//   median         V = (s > 0.01) & under top2, masked median; min/max by atomics       -> B
//   lut            per frame: cv2's 4096(+2)-bin range table and scale
//   bilateral      masked bilateral of B (V from A), inversion, rescale                 -> out
// Every comparison is against 0.01f, 1.0f, 2.0f as float32; the arithmetic steps are single
// round-to-nearest float32 operations written as intrinsics, so nothing is contracted into an FMA.
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr float kT = 0.01f;      // the validity threshold of every step
constexpr float kMax = 3.0f;     // fill_missing's max_depth
constexpr int kBins = 1 << 12;   // cv2's kExpNumBinsPerChannel
constexpr int kLut = kBins + 2;
constexpr int kTaps = 13;        // offsets with sqrt(dy^2 + dx^2) <= 2: cv2's taps for d = 5
constexpr int kBx = 32, kBy = 8;

bool fits_int32(long long v) { return v < 0x80000000ll; }

struct Taps {
  float w[kTaps];
};

struct FrameLut {
  float scale_index;
  int copy;  // |max - min| < FLT_EPSILON: cv2 returns the source unfiltered
};

struct FillWs {
  size_t a, b, top, minmax, params, lut, total;
};

FillWs fill_ws_layout(int b, int h, int w) {
  FillWs L;
  const size_t img = align_up(static_cast<size_t>(b) * h * w * 4, 256);
  L.a = 0;
  L.b = L.a + img;
  L.top = L.b + img;
  L.minmax = L.top + align_up(static_cast<size_t>(b) * 2 * w * 4, 256);
  L.params = L.minmax + align_up(static_cast<size_t>(b) * 2 * 4, 256);
  L.lut = L.params + align_up(static_cast<size_t>(b) * sizeof(FrameLut), 256);
  L.total = L.lut + align_up(static_cast<size_t>(b) * kLut * 4, 256);
  return L;
}

// float -> int with the same order (for atomicMin / atomicMax), and back
__device__ __forceinline__ int ord_key(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord_val(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

struct Px {
  int x, y, b, frame, idx;  // frame = b * h * w, idx = frame + y * w + x
};
// element (stage k, pixel p) of stages [B,4,H,W]
__device__ __forceinline__ long long stage_at(const Px &p, int k, int h, int w) {
  return 4ll * p.frame + static_cast<long long>(k) * h * w + p.y * w + p.x;
}
__device__ __forceinline__ bool pixel(int h, int w, Px &p) {
  p.x = blockIdx.x * kBx + threadIdx.x;
  p.y = blockIdx.y * kBy + threadIdx.y;
  p.b = blockIdx.z;
  p.frame = p.b * h * w;
  p.idx = p.frame + p.y * w + p.x;
  return p.x < w && p.y < h;
}

// the first row with a value > 0.01, np.argmax's 0 when the column has none
__device__ __forceinline__ int top_row(const int *top, int h) {
  const int t = *top;
  return t >= h ? 0 : t;
}

__device__ __forceinline__ float input_depth(const float *depth, int i, float cs, float s2s) {
  return __fmul_rn(__fdiv_rn(__ldg(depth + i), cs), s2s);
}
__device__ __forceinline__ float invert(float d) { return d > kT ? __fsub_rn(kMax, d) : d; }

// window maximum / minimum of radius R over the pixels inside the image (cv2's -inf / +inf border)
template <int R, bool kIsMax>
__device__ __forceinline__ float morph(const float *img, int h, int w, const Px &p) {
  float m = img[p.idx];
  for (int dy = -R; dy <= R; ++dy) {
    const int yy = p.y + dy;
    if (yy < 0 || yy >= h) continue;
    const float *row = img + p.frame + yy * w;
#pragma unroll
    for (int dx = -R; dx <= R; ++dx) {
      const int xx = p.x + dx;
      if (xx < 0 || xx >= w) continue;
      const float v = row[xx];
      m = kIsMax ? fmaxf(m, v) : fminf(m, v);
    }
  }
  return m;
}

// cv2.medianBlur(img, 5) at the pixel: replicated edge, the 13th of the 25 values
__device__ __forceinline__ float median5(const float *img, int h, int w, const Px &p) {
  float v[25];
#pragma unroll
  for (int dy = 0; dy < 5; ++dy) {
    const int yy = min(max(p.y + dy - 2, 0), h - 1);
#pragma unroll
    for (int dx = 0; dx < 5; ++dx) v[dy * 5 + dx] = img[p.frame + yy * w + min(max(p.x + dx - 2, 0), w - 1)];
  }
  // 13 bubble passes put the 13 largest, sorted, in v[12..24]
#pragma unroll
  for (int pass = 0; pass < 13; ++pass) {
#pragma unroll
    for (int i = 0; i < 24 - pass; ++i) {
      const float a = v[i], c = v[i + 1];
      v[i] = fminf(a, c);
      v[i + 1] = fmaxf(a, c);
    }
  }
  return v[12];
}

__global__ void fill_init_kernel(int b, int h, int w, int *__restrict__ top, int *__restrict__ minmax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < b * 2 * w) top[i] = h;
  if (i < b) {
    minmax[2 * i] = 0x7fffffff;
    minmax[2 * i + 1] = static_cast<int>(0x80000000u);
  }
}

// s1 = 3 - d where d > 0.01; s2 = s1 overwritten by the far (cross 3), med (cross 5) and near (cross 7)
// dilations of s1 * bin where they are > 0.01.  A dilation's value matters only where it is > 0.01, so
// the out-of-bin pixels' zeros enter as the starting value 0.
__global__ void __launch_bounds__(kBx *kBy)
fill_s2_kernel(const float *__restrict__ depth, const float *__restrict__ cam_scale, float s2s, int h, int w,
               float *__restrict__ s2) {
  Px p;
  if (!pixel(h, w, p)) return;
  const float cs = __ldg(cam_scale + p.b);
  float dn = 0.f, dm = 0.f, df = 0.f;
#pragma unroll
  for (int k = -3; k <= 3; ++k) {
#pragma unroll
    for (int axis = 0; axis < 2; ++axis) {
      if (axis == 1 && k == 0) continue;
      const int yy = p.y + (axis == 0 ? k : 0), xx = p.x + (axis == 0 ? 0 : k);
      if (yy < 0 || yy >= h || xx < 0 || xx >= w) continue;
      const float d = input_depth(depth, p.frame + yy * w + xx, cs, s2s);
      const float s1 = invert(d);
      const int r = k < 0 ? -k : k;
      if (d > kT && d <= 1.0f) dn = fmaxf(dn, s1);
      if (r <= 2 && d > 1.0f && d <= 2.0f) dm = fmaxf(dm, s1);
      if (r <= 1 && d > 2.0f) df = fmaxf(df, s1);
    }
  }
  float s = invert(input_depth(depth, p.idx, cs, s2s));
  if (df > kT) s = df;
  if (dm > kT) s = dm;
  if (dn > kT) s = dn;
  s2[p.idx] = s;
}

template <bool kIsMax>
__global__ void __launch_bounds__(kBx *kBy)
fill_morph5_kernel(const float *__restrict__ in, int h, int w, float *__restrict__ out) {
  Px p;
  if (!pixel(h, w, p)) return;
  out[p.idx] = morph<2, kIsMax>(in, h, w, p);
}

// s4 = median where s3 > 0.01; top1 = the first row of each column with s4 > 0.01
__global__ void __launch_bounds__(kBx *kBy)
fill_s4_kernel(const float *__restrict__ s3, int h, int w, float *__restrict__ s4, int *__restrict__ top,
               float *__restrict__ stages) {
  Px p;
  if (!pixel(h, w, p)) return;
  float v = s3[p.idx];
  if (v > kT) v = median5(s3, h, w, p);
  s4[p.idx] = v;
  if (v > kT) atomicMin(top + p.b * 2 * w + p.x, p.y);
  if (stages) stages[stage_at(p, 0, h, w)] = v;
}

// s5 = 9x9 dilation where s4 is not > 0.01 and the pixel is under top1; top2 from s5
__global__ void __launch_bounds__(kBx *kBy)
fill_s5_kernel(const float *__restrict__ s4, int h, int w, float *__restrict__ s5, int *__restrict__ top,
               float *__restrict__ stages) {
  Px p;
  if (!pixel(h, w, p)) return;
  float v = s4[p.idx];
  if (!(v > kT) && p.y >= top_row(top + p.b * 2 * w + p.x, h)) v = morph<4, true>(s4, h, w, p);
  s5[p.idx] = v;
  if (v > kT) atomicMin(top + p.b * 2 * w + w + p.x, p.y);
  if (stages) stages[stage_at(p, 1, h, w)] = v;
}

// one of the six fill iterations: the 5x5 dilation where s < 0.01 under top2
__global__ void __launch_bounds__(kBx *kBy)
fill_iter_kernel(const float *__restrict__ in, int h, int w, const int *__restrict__ top, float *__restrict__ out) {
  Px p;
  if (!pixel(h, w, p)) return;
  float v = in[p.idx];
  if (v < kT && p.y >= top_row(top + p.b * 2 * w + w + p.x, h)) v = morph<2, true>(in, h, w, p);
  out[p.idx] = v;
}

// V = (s > 0.01) & under top2 before the median; s = median at V; the frame's min / max of the result
__global__ void __launch_bounds__(kBx *kBy)
fill_median_kernel(const float *__restrict__ in, int h, int w, const int *__restrict__ top, float *__restrict__ out,
                   int *__restrict__ minmax, float *__restrict__ stages) {
  Px p;
  const bool inside = pixel(h, w, p);
  int kmin = 0x7fffffff, kmax = static_cast<int>(0x80000000u);
  if (inside) {
    float v = in[p.idx];
    if (v > kT && p.y >= top_row(top + p.b * 2 * w + w + p.x, h)) v = median5(in, h, w, p);
    out[p.idx] = v;
    if (stages) stages[stage_at(p, 2, h, w)] = v;
    kmin = kmax = ord_key(v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
    kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(minmax + 2 * p.b, kmin);
    atomicMax(minmax + 2 * p.b + 1, kmax);
  }
}

// cv2's float32 bilateral set-up for frame blockIdx.x: len = (float)(max - min), scale_index =
// 4096 / len, lut[i] = (float)exp(-2 * (i / scale_index)^2) (sigma_color 0.5); also the top rows out
__global__ void fill_lut_kernel(const int *__restrict__ minmax, int h, int w, const int *__restrict__ top,
                                FrameLut *__restrict__ params, float *__restrict__ lut, int *__restrict__ top_rows) {
  const int b = blockIdx.x;
  const double mn = ord_val(minmax[2 * b]), mx = ord_val(minmax[2 * b + 1]);
  const double diff = mx - mn;
  const float len = static_cast<float>(diff);
  const float scale = __fdiv_rn(static_cast<float>(kBins), len);
  if (threadIdx.x == 0) params[b] = FrameLut{scale, fabs(diff) < FLT_EPSILON ? 1 : 0};
  if (!(fabs(diff) < FLT_EPSILON))
    for (int i = threadIdx.x; i < kLut; i += blockDim.x) {
      const double v = __fdiv_rn(static_cast<float>(i), scale);
      lut[b * kLut + i] = static_cast<float>(exp(__dmul_rn(__dmul_rn(v, v), -2.0)));
    }
  if (top_rows)
    for (int i = threadIdx.x; i < 2 * w; i += blockDim.x) top_rows[b * 2 * w + i] = top_row(top + b * 2 * w + i, h);
}

__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  do {
    p = p < 0 ? -p : 2 * (n - 1) - p;
  } while (static_cast<unsigned>(p) >= static_cast<unsigned>(n));
  return p;
}

// s7 = cv2.bilateralFilter(s, 5, 0.5, 2.0) at V, else s; s8 = 3 - s7 where s7 > 0.01; out = s8 / s2s * cs.
// Per tap, in cv2's order and float32 as cv2 computes it: alpha = |val - s| * scale_index,
// i = floor(alpha), w = space_w * (lut[i] + (alpha - i) * (lut[i + 1] - lut[i])); sum += val * w, wsum += w.
__global__ void __launch_bounds__(kBx *kBy)
fill_bilateral_kernel(const float *__restrict__ pre, const float *__restrict__ vsrc, const int *__restrict__ top,
                      const FrameLut *__restrict__ params, const float *__restrict__ lut,
                      const float *__restrict__ cam_scale, float s2s, int h, int w, Taps taps,
                      float *__restrict__ out, float *__restrict__ stages) {
  Px p;
  if (!pixel(h, w, p)) return;
  float s = pre[p.idx];
  const bool V = vsrc[p.idx] > kT && p.y >= top_row(top + p.b * 2 * w + w + p.x, h);
  const FrameLut prm = params[p.b];
  if (V && !prm.copy) {
    const float *tab = lut + p.b * kLut;
    float sum = 0.f, wsum = 0.f;
    int k = 0;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
      const int yy = reflect101(p.y + dy, h);
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) {
        if (dy * dy + dx * dx > 4) continue;
        const float val = pre[p.frame + yy * w + reflect101(p.x + dx, w)];
        float alpha = __fmul_rn(fabsf(__fsub_rn(val, s)), prm.scale_index);
        const int i = static_cast<int>(floorf(alpha));
        alpha = __fsub_rn(alpha, static_cast<float>(i));
        const float lo = __ldg(tab + i), hi = __ldg(tab + i + 1);
        const float wt = __fmul_rn(taps.w[k], __fadd_rn(lo, __fmul_rn(alpha, __fsub_rn(hi, lo))));
        sum = __fadd_rn(sum, __fmul_rn(val, wt));
        wsum = __fadd_rn(wsum, wt);
        ++k;
      }
    }
    s = __fdiv_rn(sum, wsum);
  }
  if (stages) stages[stage_at(p, 3, h, w)] = s;
  if (s > kT) s = __fsub_rn(kMax, s);
  out[p.idx] = __fmul_rn(__fdiv_rn(s, s2s), __ldg(cam_scale + p.b));
}

Taps space_taps() {
  // cv2: r = sqrt(i*i + j*j) in double, weight (float)exp(r * r * (-0.5 / (sigma_space^2))), sigma_space 2
  Taps t{};
  int k = 0;
  for (int i = -2; i <= 2; ++i)
    for (int j = -2; j <= 2; ++j) {
      const double r = std::sqrt(static_cast<double>(i * i + j * j));
      if (r > 2) continue;
      t.w[k++] = static_cast<float>(std::exp(r * r * (-0.5 / (2.0 * 2.0))));
    }
  return t;
}

bool fill_size_ok(int b, int h, int w) {
  return b >= 1 && h >= 1 && w >= 1 && fits_int32(static_cast<long long>(b) * h * w) && b <= 65535 &&
         ceil_div(h, kBy) <= 65535;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_depth_fill_workspace_bytes(int b, int h, int w) {
  if (!fill_size_ok(b, h, w)) return 0;
  return fill_ws_layout(b, h, w).total;
}

extern "C" int pvn3d_depth_fill(const float *depth, const float *cam_scale, float scale_2_80m, int b, int h, int w,
                                float *out, float *stages, int *top_rows, void *workspace, size_t workspace_bytes,
                                pvn3d_stream_t stream) {
  if (!depth || !cam_scale || !out || !workspace || b < 1 || h < 1 || w < 1 || !std::isfinite(scale_2_80m) ||
      !(scale_2_80m > 0.f))
    return PVN3D_ERR_INVALID_ARG;
  if (!fill_size_ok(b, h, w)) return PVN3D_ERR_UNSUPPORTED;
  const FillWs L = fill_ws_layout(b, h, w);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  float *A = reinterpret_cast<float *>(ws + L.a), *B = reinterpret_cast<float *>(ws + L.b);
  int *top = reinterpret_cast<int *>(ws + L.top), *minmax = reinterpret_cast<int *>(ws + L.minmax);
  auto *params = reinterpret_cast<FrameLut *>(ws + L.params);
  float *lut = reinterpret_cast<float *>(ws + L.lut);
  cudaStream_t st = as_stream(stream);
  const dim3 grid(ceil_div(w, kBx), ceil_div(h, kBy), b), block(kBx, kBy);
  const int n_init = max(b * 2 * w, b);
  fill_init_kernel<<<ceil_div(n_init, 256), 256, 0, st>>>(b, h, w, top, minmax);
  int rc = check_launch("fill_init_kernel");
  if (rc != PVN3D_OK) return rc;
  fill_s2_kernel<<<grid, block, 0, st>>>(depth, cam_scale, scale_2_80m, h, w, A);
  if ((rc = check_launch("fill_s2_kernel")) != PVN3D_OK) return rc;
  fill_morph5_kernel<true><<<grid, block, 0, st>>>(A, h, w, B);
  if ((rc = check_launch("fill_morph5_kernel<dilate>")) != PVN3D_OK) return rc;
  fill_morph5_kernel<false><<<grid, block, 0, st>>>(B, h, w, A);
  if ((rc = check_launch("fill_morph5_kernel<erode>")) != PVN3D_OK) return rc;
  fill_s4_kernel<<<grid, block, 0, st>>>(A, h, w, B, top, stages);
  if ((rc = check_launch("fill_s4_kernel")) != PVN3D_OK) return rc;
  fill_s5_kernel<<<grid, block, 0, st>>>(B, h, w, A, top, stages);
  if ((rc = check_launch("fill_s5_kernel")) != PVN3D_OK) return rc;
  for (int it = 0; it < 6; ++it) {
    const bool even = (it & 1) == 0;
    fill_iter_kernel<<<grid, block, 0, st>>>(even ? A : B, h, w, top, even ? B : A);
    if ((rc = check_launch("fill_iter_kernel")) != PVN3D_OK) return rc;
  }
  fill_median_kernel<<<grid, block, 0, st>>>(A, h, w, top, B, minmax, stages);
  if ((rc = check_launch("fill_median_kernel")) != PVN3D_OK) return rc;
  fill_lut_kernel<<<b, 256, 0, st>>>(minmax, h, w, top, params, lut, top_rows);
  if ((rc = check_launch("fill_lut_kernel")) != PVN3D_OK) return rc;
  fill_bilateral_kernel<<<grid, block, 0, st>>>(B, A, top, params, lut, cam_scale, scale_2_80m, h, w, space_taps(),
                                                out, stages);
  return check_launch("fill_bilateral_kernel");
}
