// augment.cu -- get_item's training augmentation (ColorJitter, rgb_add_noise, add_real_back) of a batch, from
// per-frame parameter records drawn on the device.
//
// One thread per pixel (all three channels), frames along grid.z.  Every flag of a record is a per-frame branch
// read on the device, so a batch is a fixed sequence of launches with no host sync:
//   4 x (luma sum, jitter step)   step s applies order[s] in place (step 0 reads the input); the luma sum feeds
//                                 contrast's rounded mean; step 3 also flips LineMOD to BGR            -> A
//   2 x noise pass                hsv (in place), sharpen A -> B, motion B -> A, gauss A -> B, then noise with
//                                 the composite and the depth (pass 1, B -> A) or the CHW store (pass 2)
// A step that does not run for a frame copies its input, so each frame's image is always in the same buffer.
// The exact paths are written with _rn intrinsics so that nothing is contracted into an FMA except where
// the library being matched fuses (cv2's HSV2BGR).
#include <curand_kernel.h>

#include <cmath>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kBx = 32, kBy = 8;
constexpr int kStages = 12;
constexpr int kMaxA = 30;       // motion kernel side: int(max(|cos|,|sin|) * 15 * 2)
constexpr int kMaxTaps = 64;

__constant__ double c_cos[360], c_sin[360];  // the host's libm cos / sin of angle * (pi / 180)

struct AugWs {
  size_t a, b, sums, total;
};

AugWs aug_ws_layout(int b, int h, int w) {
  AugWs L;
  const size_t img = align_up(static_cast<size_t>(b) * h * w * 3, 256);
  L.a = 0;
  L.b = img;
  L.sums = 2 * img;
  L.total = L.sums + align_up(static_cast<size_t>(b) * 4 * 8, 256);
  return L;
}

__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  const int period = 2 * (n - 1);
  i = abs(i) % period;
  return i >= n ? period - i : i;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ---- PIL 12.2 ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ int pil_l(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

// Image.blend: (int)in1 + alpha * ((int)in2 - (int)in1) in float32, truncating store, clamped
__device__ __forceinline__ int pil_blend(int i1, int i2, float a) {
  const float t = __fadd_rn(static_cast<float>(i1), __fmul_rn(a, static_cast<float>(i2 - i1)));
  if (t <= 0.f) return 0;
  if (t >= 255.f) return 255;
  return static_cast<int>(t);
}

__device__ __forceinline__ int clip8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// Convert.c rgb2hsv_row: float32 variables, double literals
__device__ void pil_rgb2hsv(int r, int g, int b, int &oh, int &os, int &ov) {
  const int mx = max(r, max(g, b)), mn = min(r, min(g, b));
  ov = mx;
  if (mx == mn) {
    oh = os = 0;
    return;
  }
  const float cr = static_cast<float>(mx - mn);
  const float s = __fdiv_rn(cr, static_cast<float>(mx));
  const float rc = __fdiv_rn(static_cast<float>(mx - r), cr);
  const float gc = __fdiv_rn(static_cast<float>(mx - g), cr);
  const float bc = __fdiv_rn(static_cast<float>(mx - b), cr);
  float h;
  if (r == mx)
    h = __fsub_rn(bc, gc);
  else if (g == mx)
    h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, static_cast<double>(rc)), static_cast<double>(bc)));
  else
    h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, static_cast<double>(gc)), static_cast<double>(rc)));
  h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn(static_cast<double>(h), 6.0), 1.0), 1.0));
  oh = clip8(static_cast<int>(__dmul_rn(static_cast<double>(h), 255.0)));
  os = clip8(static_cast<int>(__dmul_rn(static_cast<double>(s), 255.0)));
}

__device__ __forceinline__ int c_round(double x) { return static_cast<int>(x >= 0 ? floor(x + 0.5) : ceil(x - 0.5)); }

// Convert.c hsv2rgb
__device__ void pil_hsv2rgb(int h, int s, int v, int &r, int &g, int &b) {
  if (s == 0) {
    r = g = b = v;
    return;
  }
  const double h6 = __ddiv_rn(__dmul_rn(static_cast<double>(h), 6.0), 255.0);
  const int i = static_cast<int>(floor(h6));
  const float f = __double2float_rn(__dsub_rn(h6, static_cast<double>(static_cast<float>(i))));
  const float fs = __double2float_rn(__ddiv_rn(static_cast<double>(s), 255.0));
  const double vf = static_cast<double>(v);
  const int p = clip8(c_round(__dmul_rn(vf, __dsub_rn(1.0, static_cast<double>(fs)))));
  const int q = clip8(c_round(__dmul_rn(vf, __dsub_rn(1.0, static_cast<double>(__fmul_rn(fs, f))))));
  const int t = clip8(c_round(__dmul_rn(vf, __dsub_rn(1.0, __dmul_rn(static_cast<double>(fs),
                                                                        __dsub_rn(1.0, static_cast<double>(f)))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// ---- cv2 4.13 ----------------------------------------------------------------------------------------------------
// BGR2HSV 8U: 12-bit fixed point with sdiv[v] = round(255 * 4096 / v), hdiv[d] = round(180 * 4096 / (6 d))
__device__ void cv_bgr2hsv(int b, int g, int r, int &oh, int &os, int &ov) {
  const int v = max(b, max(g, r));
  const int diff = v - min(b, min(g, r));
  const int sdiv = v == 0 ? 0 : __double2int_rn(__ddiv_rn(1044480.0, static_cast<double>(v)));
  const int hdiv = diff == 0 ? 0 : __double2int_rn(__ddiv_rn(737280.0, __dmul_rn(6.0, static_cast<double>(diff))));
  const int s = (diff * sdiv + 2048) >> 12;
  int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv + 2048) >> 12;
  if (h < 0) h += 180;
  oh = h;
  os = s;
  ov = v;
}

// HSV2BGR 8U: float32, s and v scaled by 1/255, 1 - s h and 1 - s (1 - h) fused, times 255 -- truncated in cv2's
// 32-pixel vector loop, rounded to nearest even in the per-pixel tail of a row (`tail`)
constexpr int kCvVector = 32;

__device__ void cv_hsv2bgr(int hi, int si, int vi, int &ob, int &og, int &orr, bool tail) {
  float h = __fmul_rn(static_cast<float>(hi), 6.0f / 180.0f);
  const float s = __fmul_rn(static_cast<float>(si), 1.0f / 255.0f);
  const float v = __fmul_rn(static_cast<float>(vi), 1.0f / 255.0f);
  float bb, gg, rr;
  if (s == 0.f) {
    bb = gg = rr = v;
  } else {
    const float fl = floorf(h);
    int sec = static_cast<int>(fl) % 6;
    h = __fsub_rn(h, fl);
    float tab[4];
    tab[0] = v;
    tab[1] = __fmul_rn(v, __fsub_rn(1.f, s));
    tab[2] = __fmul_rn(v, __fmaf_rn(-s, h, 1.f));
    tab[3] = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, h), 1.f));
    const int idx[6][3] = {{1, 3, 0}, {1, 0, 2}, {3, 0, 1}, {0, 2, 1}, {0, 1, 3}, {2, 1, 0}};
    bb = tab[idx[sec][0]];
    gg = tab[idx[sec][1]];
    rr = tab[idx[sec][2]];
  }
  bb = __fmul_rn(bb, 255.f);
  gg = __fmul_rn(gg, 255.f);
  rr = __fmul_rn(rr, 255.f);
  ob = clip8(tail ? __float2int_rn(bb) : static_cast<int>(bb));
  og = clip8(tail ? __float2int_rn(gg) : static_cast<int>(gg));
  orr = clip8(tail ? __float2int_rn(rr) : static_cast<int>(rr));
}

// getGaussianKernelBitExact + getGaussianKernelFixedPoint_ED with 8 fractional bits
__device__ void gauss_taps(int ksize, double sigma, int *k) {
  const int half = ksize / 2;
  double vals[2];
  if (!(sigma > 0.0)) {
    if (ksize == 3) {
      vals[0] = 0.25;
    } else {
      vals[0] = 0.0625;
      vals[1] = 0.25;
    }
  } else {
    const double scale2 = __ddiv_rn(-0.125, __dmul_rn(sigma, sigma));
    double tot = 0.0;
    int x = 1 - ksize;
    for (int i = 0; i < half; ++i, x += 2) {
      vals[i] = exp(__dmul_rn(static_cast<double>(x * x), scale2));
      tot = __dadd_rn(tot, vals[i]);
    }
    tot = __dadd_rn(__dmul_rn(tot, 2.0), 1.0);
    const double inv = __ddiv_rn(1.0, tot);
    for (int i = 0; i < half; ++i) vals[i] = __dmul_rn(vals[i], inv);
  }
  double err = 0.0;
  int sum = 0;
  for (int i = 0; i < half; ++i) {
    const double adj = __dadd_rn(__dmul_rn(vals[i], 256.0), err);
    const int v = __double2int_rn(adj);
    err = __dsub_rn(adj, static_cast<double>(v));
    k[i] = k[ksize - 1 - i] = v;
    sum += v;
  }
  k[half] = 256 - 2 * sum;
}

// linear_motion_blur's cv2.line into an a x a grid, clipped as cv::clipLine and walked as the 8-connected
// cv::LineIterator; the taps come out in row-major order.  Returns a (0: the image is left unchanged).
__device__ int motion_taps(int angle, int length, int *taps, int *count) {
  angle = clampi(angle, 0, 359);
  length = clampi(length, 1, 15);
  const double dx = c_cos[angle], dy = c_sin[angle];
  const int a = static_cast<int>(__dmul_rn(__dmul_rn(fmax(fabs(dx), fabs(dy)), static_cast<double>(length)), 2.0));
  *count = 0;
  if (a <= 0) return 0;
  const int c = a / 2;
  int x1 = c, y1 = c;
  int x2 = static_cast<int>(__dadd_rn(__dmul_rn(dx, static_cast<double>(length)), static_cast<double>(c)));
  int y2 = static_cast<int>(__dadd_rn(__dmul_rn(dy, static_cast<double>(length)), static_cast<double>(c)));
  const int right = a - 1, bottom = a - 1;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if (c2) {
    if (c2 & 12) {
      const int t = c2 < 8 ? 0 : bottom;
      x2 += static_cast<int>(__ddiv_rn(__dmul_rn(static_cast<double>(t - y2), static_cast<double>(x2 - x1)),
                                       static_cast<double>(y2 - y1)));
      y2 = t;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if (c2) {
      const int t = c2 == 1 ? 0 : right;
      y2 += static_cast<int>(__ddiv_rn(__dmul_rn(static_cast<double>(t - x2), static_cast<double>(y2 - y1)),
                                       static_cast<double>(x2 - x1)));
      x2 = t;
    }
  }
  if (x2 < x1) {
    int t = x1; x1 = x2; x2 = t;
    t = y1; y1 = y2; y2 = t;
  }
  int ddx = x2 - x1, ddy = y2 - y1, sy = 1;
  if (ddy < 0) {
    ddy = -ddy;
    sy = -1;
  }
  const bool vert = ddy > ddx;
  if (vert) {
    const int t = ddx; ddx = ddy; ddy = t;
  }
  int err = ddx - (ddy + ddy);
  const int plus = ddx + ddx, minus = -(ddy + ddy);
  // mark the pixels in a bit grid (a <= 30 columns per 32-bit row), then list them in row-major order
  uint32_t rows[kMaxA];
  for (int i = 0; i < a; ++i) rows[i] = 0u;
  int x = x1, y = y1;
  for (int i = 0; i <= ddx; ++i) {
    if (x >= 0 && x < a && y >= 0 && y < a) rows[y] |= 1u << x;
    const bool m = err < 0;
    err += minus + (m ? plus : 0);
    if (vert) {
      y += sy;
      x += m ? 1 : 0;
    } else {
      x += 1;
      y += m ? sy : 0;
    }
  }
  int n = 0;
  for (int r = 0; r < a; ++r)
    for (int q = 0; q < a; ++q)
      if ((rows[r] >> q) & 1u && n < kMaxTaps) taps[n++] = r * 256 + q;
  if (n == 0) taps[n++] = c * 256 + c;
  *count = n;
  return a;
}

struct Px {
  int c[3];
};

__device__ __forceinline__ Px load_px(const uint8_t *img, size_t i) {
  Px p;
  p.c[0] = img[3 * i];
  p.c[1] = img[3 * i + 1];
  p.c[2] = img[3 * i + 2];
  return p;
}

__device__ __forceinline__ void store_px(uint8_t *img, size_t i, const Px &p) {
  img[3 * i] = static_cast<uint8_t>(p.c[0]);
  img[3 * i + 1] = static_cast<uint8_t>(p.c[1]);
  img[3 * i + 2] = static_cast<uint8_t>(p.c[2]);
}

__device__ __forceinline__ void stage_px(uint8_t *stages, int f, int stage, size_t hw, size_t p, const Px &px) {
  if (stages) store_px(stages + (static_cast<size_t>(f) * kStages + stage) * hw * 3, p, px);
}

// ---- the draw ----------------------------------------------------------------------------------------------------
struct Draw {
  curandStatePhilox4_32_10_t st;
  __device__ uint32_t u32() { return curand(&st); }
  __device__ double u01() {  // numpy's 53-bit double from two words
    const uint32_t a = u32() >> 5, b = u32() >> 6;
    return (a * 67108864.0 + b) / 9007199254740992.0;
  }
  __device__ double range(double lo, double hi) { return u01() * (hi - lo) + lo; }
  __device__ int randint(int n) { return min(static_cast<int>(u01() * n), n - 1); }
  __device__ uint64_t key() {
    const uint64_t hi = u32();
    return (hi << 32) | u32();
  }
};

__global__ void __launch_bounds__(128) augment_draw_kernel(unsigned long long seed, const int32_t *kinds, int nb,
                                                           int dataset, pvn3d_augment_params_t *params) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= nb) return;
  Draw d;
  curand_init(seed, static_cast<unsigned long long>(f), 0ull, &d.st);
  pvn3d_augment_params_t p = {};
  const bool ycb = dataset == PVN3D_AUG_YCB;
  p.kind = kinds[f];
  p.jitter = ycb || p.kind == 0;
  for (int i = 0; i < 4; ++i) p.order[i] = i;
  p.brightness = p.contrast = p.saturation = 1.f;
  if (p.jitter) {
    for (int i = 3; i > 0; --i) {  // Fisher-Yates: a uniform permutation, as torch.randperm(4)
      const int j = d.randint(i + 1);
      const int t = p.order[i];
      p.order[i] = p.order[j];
      p.order[j] = t;
    }
    p.brightness = static_cast<float>(d.range(0.8, 1.2));
    p.contrast = static_cast<float>(d.range(0.8, 1.2));
    p.saturation = static_cast<float>(d.range(0.8, 1.2));
    p.hue = static_cast<float>(d.range(-0.05, 0.05));
  }
  const bool noisy = p.kind == 1;  // YCB syn, LineMOD render
  if (noisy) {
    p.back = 1;
    p.n_pass = 1 + (d.u01() > 0.8);
  }
  for (int q = 0; q < 2; ++q) {
    pvn3d_augment_pass_t &ps = p.passes[q];
    ps.s_factor = ps.v_factor = 1.0;
    ps.ksize = 3;
    if (q >= p.n_pass) continue;
    ps.s_factor = ycb ? d.range(1.25, 1.45) : d.range(0.75, 1.25);
    ps.v_factor = ycb ? d.range(1.15, 1.35) : d.range(0.85, 1.15);
    if (ycb) {
      ps.sharpen = d.u01() > 0.8;
      ps.sharpen_w = d.u01() * 3 + 9;
    }
    ps.motion = d.u01() > 0.8;
    ps.angle = static_cast<int>(d.u01() * 360);
    ps.length = static_cast<int>(d.u01() * 15) + 1;
    ps.gauss = d.u01() > 0.8;
    ps.ksize = d.u01() > 0.2 ? 3 : 5;
    ps.sigma = d.u01();
    if (ycb) {
      ps.noise_sigma = d.u01() > 0.2 ? d.randint(15) : d.randint(25);
      ps.extra = d.u01() > 0.8;
    }
    ps.noise_key = d.key();
    ps.extra_key = d.key();
  }
  params[f] = p;
}

// ---- the jitter --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBx *kBy) luma_sum_kernel(const uint8_t *img, const pvn3d_augment_params_t *params,
                                                             int step, int h, int w, unsigned long long *sums) {
  const int f = blockIdx.z;
  const pvn3d_augment_params_t &p = params[f];
  if (!p.jitter || p.order[step & 3] != 1) return;
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  unsigned v = 0;
  if (x < w && y < h) {
    const Px px = load_px(img, (static_cast<size_t>(f) * h + y) * w + x);
    v = pil_l(px.c[0], px.c[1], px.c[2]);
  }
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(&sums[f * 4 + step], static_cast<unsigned long long>(v));
}

__device__ Px jitter_op(Px px, int op, const pvn3d_augment_params_t &p, int mean) {
  switch (op) {
    case 0:
      for (int c = 0; c < 3; ++c) px.c[c] = pil_blend(0, px.c[c], p.brightness);
      break;
    case 1:
      for (int c = 0; c < 3; ++c) px.c[c] = pil_blend(mean, px.c[c], p.contrast);
      break;
    case 2: {
      const int l = pil_l(px.c[0], px.c[1], px.c[2]);
      for (int c = 0; c < 3; ++c) px.c[c] = pil_blend(l, px.c[c], p.saturation);
      break;
    }
    default: {
      int hh, ss, vv;
      pil_rgb2hsv(px.c[0], px.c[1], px.c[2], hh, ss, vv);
      // torchvision: np.int32(hue_factor * 255).astype(np.uint8), added modulo 256
      const int shift = static_cast<int>(__dmul_rn(static_cast<double>(p.hue), 255.0)) & 0xff;
      pil_hsv2rgb((hh + shift) & 0xff, ss, vv, px.c[0], px.c[1], px.c[2]);
    }
  }
  return px;
}

__global__ void __launch_bounds__(kBx *kBy) jitter_step_kernel(const uint8_t *src, uint8_t *dst,
                                                                const pvn3d_augment_params_t *params, int step,
                                                                int h, int w, int dataset,
                                                                const unsigned long long *sums, uint8_t *stages) {
  const int f = blockIdx.z;
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const pvn3d_augment_params_t &p = params[f];
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  Px px = load_px(src, i);
  if (p.jitter) {
    const int op = clampi(p.order[step], 0, 3);
    int mean = 0;
    if (op == 1)  // ImageStat's mean of convert("L") in float64, + 0.5, int()
      mean = static_cast<int>(__dadd_rn(__ddiv_rn(static_cast<double>(sums[f * 4 + step]), static_cast<double>(hw)),
                                        0.5));
    px = jitter_op(px, op, p, mean);
  }
  if (step == 3) {
    if (dataset == PVN3D_AUG_LINEMOD) {
      const int t = px.c[0];
      px.c[0] = px.c[2];
      px.c[2] = t;
    }
    stage_px(stages, f, 0, hw, pix, px);
  }
  if (p.jitter || step == 0 || step == 3) store_px(dst, i, px);
}

// ---- the noise passes --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBx *kBy) hsv_kernel(uint8_t *img, const pvn3d_augment_params_t *params, int q,
                                                        int h, int w, uint8_t *stages) {
  const int f = blockIdx.z;
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const pvn3d_augment_params_t &p = params[f];
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  Px px = load_px(img, i);
  if (q < p.n_pass) {
    const pvn3d_augment_pass_t &ps = p.passes[q];
    int hh, ss, vv;
    cv_bgr2hsv(px.c[0], px.c[1], px.c[2], hh, ss, vv);
    // uint16 * float64 truncated on assignment, then clipped to 255
    ss = min(static_cast<int>(static_cast<uint16_t>(__dmul_rn(static_cast<double>(ss), ps.s_factor))), 255);
    vv = min(static_cast<int>(static_cast<uint16_t>(__dmul_rn(static_cast<double>(vv), ps.v_factor))), 255);
    cv_hsv2bgr(hh, ss, vv, px.c[0], px.c[1], px.c[2], x >= w / kCvVector * kCvVector);
    store_px(img, i, px);
  }
  stage_px(stages, f, 1 + 6 * q, hw, pix, px);
}

// filter2D with a float kernel given as taps (offsets from the anchor, float32 weights) in row-major order
__device__ Px filter_taps(const uint8_t *src, int f, int h, int w, int x, int y, int n, const int *tdy,
                          const int *tdx, const float *tw) {
  float acc[3] = {0.f, 0.f, 0.f};
  const size_t base = static_cast<size_t>(f) * h * w;
  for (int t = 0; t < n; ++t) {
    const int yy = reflect101(y + tdy[t], h), xx = reflect101(x + tdx[t], w);
    const uint8_t *s = src + 3 * (base + static_cast<size_t>(yy) * w + xx);
    for (int c = 0; c < 3; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(tw[t], static_cast<float>(s[c])));
  }
  Px o;
  for (int c = 0; c < 3; ++c) o.c[c] = clip8(__float2int_rn(acc[c]));
  return o;
}

__global__ void __launch_bounds__(kBx *kBy) sharpen_kernel(const uint8_t *src, uint8_t *dst,
                                                            const pvn3d_augment_params_t *params, int q, int h, int w,
                                                            uint8_t *stages) {
  __shared__ int s_dy[9], s_dx[9];
  __shared__ float s_w[9];
  const int f = blockIdx.z;
  const pvn3d_augment_params_t &p = params[f];
  const bool on = q < p.n_pass && p.passes[q].sharpen;
  const int tid = threadIdx.y * kBx + threadIdx.x;
  if (on && tid < 9) {
    // -1 everywhere, w at the centre, divided by the sum w - 8 (exact in float64), then float32
    const double cw = p.passes[q].sharpen_w, sum = __dsub_rn(cw, 8.0);
    s_dy[tid] = tid / 3 - 1;
    s_dx[tid] = tid % 3 - 1;
    s_w[tid] = __double2float_rn(__ddiv_rn(tid == 4 ? cw : -1.0, sum));
  }
  __syncthreads();
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  const Px px = on ? filter_taps(src, f, h, w, x, y, 9, s_dy, s_dx, s_w) : load_px(src, i);
  store_px(dst, i, px);
  stage_px(stages, f, 2 + 6 * q, hw, pix, px);
}

__global__ void __launch_bounds__(kBx *kBy) motion_kernel(const uint8_t *src, uint8_t *dst,
                                                           const pvn3d_augment_params_t *params, int q, int h, int w,
                                                           uint8_t *stages) {
  __shared__ int s_dy[kMaxTaps], s_dx[kMaxTaps], s_n;
  __shared__ float s_w[kMaxTaps];
  const int f = blockIdx.z;
  const pvn3d_augment_params_t &p = params[f];
  bool on = q < p.n_pass && p.passes[q].motion;
  if (on && threadIdx.x == 0 && threadIdx.y == 0) {
    int taps[kMaxTaps], n;
    const int a = motion_taps(p.passes[q].angle, p.passes[q].length, taps, &n);
    const float wt = __double2float_rn(__ddiv_rn(1.0, static_cast<double>(n)));
    for (int t = 0; t < n; ++t) {
      s_dy[t] = (taps[t] >> 8) - a / 2;
      s_dx[t] = (taps[t] & 255) - a / 2;
      s_w[t] = wt;
    }
    s_n = a > 0 ? n : 0;
  }
  __syncthreads();
  if (on) on = s_n > 0;
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  const Px px = on ? filter_taps(src, f, h, w, x, y, s_n, s_dy, s_dx, s_w) : load_px(src, i);
  store_px(dst, i, px);
  stage_px(stages, f, 3 + 6 * q, hw, pix, px);
}

__global__ void __launch_bounds__(kBx *kBy) gauss_kernel(const uint8_t *src, uint8_t *dst,
                                                          const pvn3d_augment_params_t *params, int q, int h, int w,
                                                          uint8_t *stages) {
  __shared__ int s_k[5];
  const int f = blockIdx.z;
  const pvn3d_augment_params_t &p = params[f];
  const bool on = q < p.n_pass && p.passes[q].gauss;
  const int ks = on && p.passes[q].ksize == 5 ? 5 : 3;
  if (on && threadIdx.x == 0 && threadIdx.y == 0) gauss_taps(ks, p.passes[q].sigma, s_k);
  __syncthreads();
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  Px px;
  if (on) {
    // rows then columns in fixed point: sum_v k_v * (sum_u k_u * x), + 2^15, >> 16 (exact in int32)
    const int r = ks / 2;
    int col[3] = {0, 0, 0};
    for (int v = 0; v < ks; ++v) {
      const int yy = reflect101(y + v - r, h);
      const uint8_t *row = src + 3 * (f * hw + static_cast<size_t>(yy) * w);
      int acc[3] = {0, 0, 0};
      for (int u = 0; u < ks; ++u) {
        const int xx = reflect101(x + u - r, w);
        for (int c = 0; c < 3; ++c) acc[c] += s_k[u] * row[3 * xx + c];
      }
      for (int c = 0; c < 3; ++c) col[c] += s_k[v] * acc[c];
    }
    for (int c = 0; c < 3; ++c) px.c[c] = min((col[c] + (1 << 15)) >> 16, 255);
  } else {
    px = load_px(src, i);
  }
  store_px(dst, i, px);
  stage_px(stages, f, 4 + 6 * q, hw, pix, px);
}

// YCB's gaussian_noise (and the extra noise), then for pass 1 add_real_back and the depth, for pass 2 the CHW store
__global__ void __launch_bounds__(kBx *kBy) noise_kernel(const uint8_t *src, uint8_t *dst, uint8_t *rgb_out,
                                                          const pvn3d_augment_params_t *params, int q, int h, int w,
                                                          int dataset, const uint8_t *labels, const uint8_t *back_rgb,
                                                          const uint8_t *back_labels, int back_ch,
                                                          const float *depth, const float *back_depth,
                                                          float *depth_out, uint8_t *stages, float *noise) {
  const int f = blockIdx.z;
  const int x = blockIdx.x * kBx + threadIdx.x, y = blockIdx.y * kBy + threadIdx.y;
  if (x >= w || y >= h) return;
  const pvn3d_augment_params_t &p = params[f];
  const size_t hw = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x, i = f * hw + pix;
  Px px = load_px(src, i);
  if (q < p.n_pass && dataset == PVN3D_AUG_YCB) {
    const pvn3d_augment_pass_t &ps = p.passes[q];
    float *nf = noise ? noise + (static_cast<size_t>(f) * 4 + 2 * q) * hw * 3 : nullptr;
    for (int k = 0; k < 1 + (ps.extra != 0); ++k) {
      curandStatePhilox4_32_10_t st;
      curand_init(k ? ps.extra_key : ps.noise_key, static_cast<unsigned long long>(pix), 0ull, &st);
      const float4 n4 = curand_normal4(&st);
      const float n[3] = {n4.x, n4.y, n4.z};
      const float sg = k ? 7.f : static_cast<float>(ps.noise_sigma);
      for (int c = 0; c < 3; ++c) {
        const float t = __fadd_rn(static_cast<float>(px.c[c]), __fmul_rn(n[c], sg));
        px.c[c] = static_cast<int>(fminf(fmaxf(t, 0.f), 255.f));
        if (nf) nf[k * hw * 3 + 3 * pix + c] = n[c];
      }
    }
  }
  stage_px(stages, f, 5 + 6 * q, hw, pix, px);
  if (q == 0) {
    float d = depth[i];
    if (p.back) {
      const uint8_t *bl = back_labels + static_cast<size_t>(back_ch) * i;
      const uint8_t *br = back_rgb + 3 * i;
      if (labels[i] == 0) {
        for (int c = 0; c < 3; ++c) {
          const int sc = dataset == PVN3D_AUG_LINEMOD ? 2 - c : c;  // the background flipped to BGR
          px.c[c] = bl[back_ch == 3 ? sc : 0] == 0 ? br[sc] : 0;
        }
      }
      if (!(static_cast<double>(d) > 1e-6)) d = bl[0] == 0 ? back_depth[i] : 0.f;
    }
    depth_out[i] = d;
    stage_px(stages, f, 6, hw, pix, px);
    store_px(dst, i, px);
  } else {
    for (int c = 0; c < 3; ++c) rgb_out[(static_cast<size_t>(f) * 3 + c) * hw + pix] = static_cast<uint8_t>(px.c[c]);
  }
}

// ---- the probe ---------------------------------------------------------------------------------------------------
__global__ void augment_probe_kernel(int op, const void *in, long long n, void *out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (op <= 4 || op == 7) {
    const uint8_t *s = static_cast<const uint8_t *>(in) + 3 * i;
    uint8_t *d = static_cast<uint8_t *>(out);
    int a, b, c;
    switch (op) {
      case 0: cv_bgr2hsv(s[0], s[1], s[2], a, b, c); break;
      case 1: cv_hsv2bgr(s[0], s[1], s[2], a, b, c, false); break;
      case 7: cv_hsv2bgr(s[0], s[1], s[2], a, b, c, true); break;
      case 2: pil_rgb2hsv(s[0], s[1], s[2], a, b, c); break;
      case 3: pil_hsv2rgb(s[0], s[1], s[2], a, b, c); break;
      default: d[i] = static_cast<uint8_t>(pil_l(s[0], s[1], s[2])); return;
    }
    d[3 * i] = static_cast<uint8_t>(a);
    d[3 * i + 1] = static_cast<uint8_t>(b);
    d[3 * i + 2] = static_cast<uint8_t>(c);
  } else if (op == 5) {
    const double *s = static_cast<const double *>(in) + 2 * i;
    int *d = static_cast<int *>(out) + 5 * i;
    int k[5] = {0, 0, 0, 0, 0};
    gauss_taps(s[0] == 5.0 ? 5 : 3, s[1], k);
    for (int j = 0; j < 5; ++j) d[j] = k[j];
  } else {
    const int *s = static_cast<const int *>(in) + 2 * i;
    int *d = static_cast<int *>(out) + 64 * i;
    int taps[kMaxTaps], cnt;
    d[0] = motion_taps(s[0], s[1], taps, &cnt);
    d[1] = cnt;
    for (int j = 0; j < 62; ++j) d[2 + j] = j < cnt ? taps[j] : -1;
  }
}

PerDeviceOnce g_trig_once;

int upload_trig() {
  double c[360], s[360];
  for (int a = 0; a < 360; ++a) {
    const double rad = a * (3.141592653589793 / 180.0);  // numpy's deg2rad
    c[a] = std::cos(rad);
    s[a] = std::sin(rad);
  }
  PVN3D_ONCE_PER_DEVICE(g_trig_once, (cudaMemcpyToSymbol(c_cos, c, sizeof(c)) == cudaSuccess
                                          ? cudaMemcpyToSymbol(c_sin, s, sizeof(s))
                                          : cudaGetLastError()),
                        "augment: cos/sin table");
  return PVN3D_OK;
}

bool aug_size_ok(int b, int h, int w) {
  return b >= 1 && h >= 1 && w >= 1 && b <= 65535 && (h + kBy - 1) / kBy <= 65535 &&
         static_cast<long long>(b) * h * w * 3 < 0x80000000ll;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" int pvn3d_augment_draw(unsigned long long seed, const int32_t *kinds, int b, int dataset,
                                  pvn3d_augment_params_t *params, pvn3d_stream_t stream) {
  if (!kinds || !params || b < 1 || (dataset != PVN3D_AUG_YCB && dataset != PVN3D_AUG_LINEMOD))
    return PVN3D_ERR_INVALID_ARG;
  augment_draw_kernel<<<ceil_div(b, 128), 128, 0, as_stream(stream)>>>(seed, kinds, b, dataset, params);
  return check_launch("augment_draw_kernel");
}

extern "C" size_t pvn3d_augment_workspace_bytes(int b, int h, int w) {
  return aug_size_ok(b, h, w) ? aug_ws_layout(b, h, w).total : 0;
}

extern "C" int pvn3d_augment_apply(const uint8_t *rgb, const float *depth, const uint8_t *labels,
                                   const uint8_t *back_rgb, const uint8_t *back_labels, int back_label_channels,
                                   const float *back_depth, const pvn3d_augment_params_t *params, int b, int h, int w,
                                   int dataset, uint8_t *rgb_out, float *depth_out, uint8_t *stages, float *noise,
                                   void *workspace, size_t workspace_bytes, pvn3d_stream_t stream) {
  if (!rgb || !depth || !labels || !back_rgb || !back_labels || !back_depth || !params || !rgb_out || !depth_out ||
      !workspace || b < 1 || h < 1 || w < 1 || (back_label_channels != 1 && back_label_channels != 3) ||
      (dataset != PVN3D_AUG_YCB && dataset != PVN3D_AUG_LINEMOD))
    return PVN3D_ERR_INVALID_ARG;
  if (!aug_size_ok(b, h, w)) return PVN3D_ERR_UNSUPPORTED;
  const AugWs L = aug_ws_layout(b, h, w);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  int rc = upload_trig();
  if (rc != PVN3D_OK) return rc;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  uint8_t *A = ws + L.a, *B = ws + L.b;
  auto *sums = reinterpret_cast<unsigned long long *>(ws + L.sums);
  cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(sums, 0, static_cast<size_t>(b) * 4 * 8, st), "augment: luma sums");
  const dim3 grid(ceil_div(w, kBx), ceil_div(h, kBy), b), block(kBx, kBy);
  for (int s = 0; s < 4; ++s) {
    const uint8_t *src = s == 0 ? rgb : A;
    luma_sum_kernel<<<grid, block, 0, st>>>(src, params, s, h, w, sums);
    if ((rc = check_launch("luma_sum_kernel")) != PVN3D_OK) return rc;
    jitter_step_kernel<<<grid, block, 0, st>>>(src, A, params, s, h, w, dataset, sums, stages);
    if ((rc = check_launch("jitter_step_kernel")) != PVN3D_OK) return rc;
  }
  for (int q = 0; q < 2; ++q) {
    hsv_kernel<<<grid, block, 0, st>>>(A, params, q, h, w, stages);
    if ((rc = check_launch("hsv_kernel")) != PVN3D_OK) return rc;
    sharpen_kernel<<<grid, block, 0, st>>>(A, B, params, q, h, w, stages);
    if ((rc = check_launch("sharpen_kernel")) != PVN3D_OK) return rc;
    motion_kernel<<<grid, block, 0, st>>>(B, A, params, q, h, w, stages);
    if ((rc = check_launch("motion_kernel")) != PVN3D_OK) return rc;
    gauss_kernel<<<grid, block, 0, st>>>(A, B, params, q, h, w, stages);
    if ((rc = check_launch("gauss_kernel")) != PVN3D_OK) return rc;
    noise_kernel<<<grid, block, 0, st>>>(B, A, rgb_out, params, q, h, w, dataset, labels, back_rgb, back_labels,
                                         back_label_channels, depth, back_depth, depth_out, stages, noise);
    if ((rc = check_launch("noise_kernel")) != PVN3D_OK) return rc;
  }
  return PVN3D_OK;
}

extern "C" int pvn3d_augment_probe(int op, const void *in, long long n, void *out, pvn3d_stream_t stream) {
  if (!in || !out || n < 1 || op < 0 || op > 7 || n > (1ll << 31)) return PVN3D_ERR_INVALID_ARG;
  if (op == 6) {
    const int rc = upload_trig();
    if (rc != PVN3D_OK) return rc;
  }
  augment_probe_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, as_stream(stream)>>>(op, in, n, out);
  return check_launch("augment_probe_kernel");
}
