// vis.cu -- demo.py's pose overlay (demo.py:122-145) on device:
//
//   every mesh point of every drawn slot moved by the slot's predicted pose, projected with the frame's K
//   (Basic_Utils.project_p3d, basic_utils.py:306-313), clipped to [0, w] x [0, h] and painted as a filled disc of
//   radius r in the slot's colour (Basic_Utils.draw_p2ds, basic_utils.py:315-323: one cv2.circle(img, c, r, color, -1)
//   per point).  Two launches after a memset of the stamp plane:
//
//   vis_mark_kernel   one thread per (frame, slot, point): the float64 transform and projection with numpy's
//                     semantics, then an integer atomicMax of slot + 1 into stamp[frame, y, x] for every pixel of
//                     the point's disc.  The largest slot index wins a pixel, which is the reference's rule: objects
//                     are drawn in slot order and a later disc overwrites an earlier one.  The points of one slot
//                     share one colour, so their order does not matter.
//   vis_paint_kernel  one thread per pixel: a stamped pixel takes its winning slot's colour.
//
// The drop-in (pvn3d_vis_draw_p2ds) runs the same two kernels on integer points that are already projected, and writes
// the clipped points back, as draw_p2ds does in place.  No float atomics: two calls give the same bits.
#include <math.h>

#include "common.cuh"

namespace pvn3d {
namespace {

constexpr int kMarkThreads = 128;
constexpr int kPaintThreads = 256;
constexpr int kMaxRadius = 32767;   // r * r fits in an int

// float64 -> int32 as numpy's astype(np.int32) does on x86-64 (cvttsd2si): NaN and anything outside the int32 range
// become INT_MIN.  The value is already integral here (np.around ran first).
__device__ __forceinline__ int np_to_int32(double v) {
  return (v >= -2147483648.0 && v <= 2147483647.0) ? static_cast<int>(v) : static_cast<int>(0x80000000u);
}

// a . b over three terms, left to right, every product and sum rounded on its own (no FMA contraction)
__device__ __forceinline__ double dot3(double x, double y, double z, double a, double b, double c) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, a), __dmul_rn(y, b)), __dmul_rn(z, c));
}

// Mark every pixel of the disc {(dx, dy) : dx^2 + dy^2 <= r^2} around (x, y), cut to the image, with `v` (integer max).
// The half-width of each row is the exact integer square root.  The loops run over absolute pixel coordinates, each
// bound clamped to the image on its own.  (Written as offsets from the centre, dx from max(-hw, -x) to
// min(hw, w - 1 - x), the CUDA 12.9 build ran the inner loop up to dx = hw for a centre clipped to x = w, so the disc
// wrapped into the next row; the SASS computed the trip count from max(min(hw, w - 1 - x), hw, -x).)
__device__ void mark_disc(int *stamp, int h, int w, int x, int y, int r, int v) {
  const int r2 = r * r;
  const int ya = max(y - r, 0), yb = min(y + r, h - 1);
  for (int yy = ya; yy <= yb; ++yy) {
    const int dy = yy - y;
    const int rem = r2 - dy * dy;
    int hw = static_cast<int>(sqrt(static_cast<double>(rem)));
    while (hw * hw > rem) --hw;
    while ((hw + 1) * (hw + 1) <= rem) ++hw;
    const int xa = max(x - hw, 0), xb = min(x + hw, w - 1);
    int *row = stamp + static_cast<size_t>(yy) * w;
    for (int xx = xa; xx <= xb; ++xx) {
      // values only grow during the launch: a stale read can only be smaller, so skipping on >= is safe
      if (*reinterpret_cast<volatile int *>(row + xx) < v) atomicMax(row + xx, v);
    }
  }
}

struct PoseArgs {
  const float *mesh_pts;   // [P_total, 3]
  const int *mesh_off;     // [n_cls + 1]
  int n_cls;
  const void *poses;       // [b, n_cls, 3, 4] f32 or f64
  int poses_f64;
  const uint8_t *present;  // [b, n_cls]
  const int *order;        // [b, s]
  int s;
  const double *k;         // [b, 3, 3]
  double cam_scale;
};

// grid (ceil(max_pts / kMarkThreads), s, b)
__global__ void __launch_bounds__(kMarkThreads)
    vis_mark_poses_kernel(const __grid_constant__ PoseArgs a, int h, int w, int r, int *__restrict__ stamp) {
  const int b = blockIdx.z, slot = blockIdx.y;
  const int c = a.order[static_cast<size_t>(b) * a.s + slot];
  if (c < 1 || c >= a.n_cls || !a.present[static_cast<size_t>(b) * a.n_cls + c]) return;   // not drawn
  const int base = a.mesh_off[c];
  const int i = blockIdx.x * kMarkThreads + threadIdx.x;
  if (i >= a.mesh_off[c + 1] - base) return;
  const float *p = a.mesh_pts + static_cast<size_t>(base + i) * 3;
  const double x = p[0], y = p[1], z = p[2];   // the float32 mesh promoted, as numpy does
  double rt[12];
  const size_t pe = (static_cast<size_t>(b) * a.n_cls + c) * 12;
  if (a.poses_f64) {
    for (int e = 0; e < 12; ++e) rt[e] = static_cast<const double *>(a.poses)[pe + e];
  } else {
    for (int e = 0; e < 12; ++e) rt[e] = static_cast<const float *>(a.poses)[pe + e];
  }
  // demo.py: np.dot(mesh_pts, pose[:, :3].T) + pose[:, 3]; project_p3d: p3d * cam_scale, then np.dot(p3d, K.T)
  double q[3];
  for (int j = 0; j < 3; ++j)
    q[j] = __dmul_rn(__dadd_rn(dot3(x, y, z, rt[j * 4], rt[j * 4 + 1], rt[j * 4 + 2]), rt[j * 4 + 3]), a.cam_scale);
  const double *k = a.k + static_cast<size_t>(b) * 9;
  const double u = dot3(q[0], q[1], q[2], k[0], k[1], k[2]);
  const double v = dot3(q[0], q[1], q[2], k[3], k[4], k[5]);
  double d = dot3(q[0], q[1], q[2], k[6], k[7], k[8]);
  if (d < 1e-8) d = 1.0;   // a NaN depth stays NaN
  // np.around (half to even), astype(np.int32), then draw_p2ds's clip to [0, w] / [0, h]
  const int px = min(max(np_to_int32(rint(__ddiv_rn(u, d))), 0), w);
  const int py = min(max(np_to_int32(rint(__ddiv_rn(v, d))), 0), h);
  mark_disc(stamp + static_cast<size_t>(b) * h * w, h, w, px, py, r, slot + 1);
}

// grid ceil(n / kMarkThreads): points [n, 2] i32, clipped in place
__global__ void __launch_bounds__(kMarkThreads)
    vis_mark_p2ds_kernel(int *__restrict__ p2ds, int n, int h, int w, int r, int *__restrict__ stamp) {
  const int i = blockIdx.x * kMarkThreads + threadIdx.x;
  if (i >= n) return;
  const int px = min(max(p2ds[2 * i], 0), w);
  const int py = min(max(p2ds[2 * i + 1], 0), h);
  p2ds[2 * i] = px;
  p2ds[2 * i + 1] = py;
  mark_disc(stamp, h, w, px, py, r, 1);
}

// grid-stride over the b*h*w pixels.  With order == NULL every stamped pixel takes `color` (c0 | c1 << 8 | c2 << 16);
// otherwise the colour of class order[frame, stamp - 1].
__global__ void __launch_bounds__(kPaintThreads)
    vis_paint_kernel(uint8_t *__restrict__ img, const int *__restrict__ stamp, long long hw, long long total,
                     const int *__restrict__ order, int s, const uint8_t *__restrict__ colors, unsigned color) {
  for (long long p = blockIdx.x * static_cast<long long>(kPaintThreads) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * kPaintThreads) {
    const int v = __ldcs(stamp + p);
    if (v == 0) continue;
    uint8_t c0, c1, c2;
    if (order) {
      const uint8_t *col = colors + static_cast<size_t>(order[(p / hw) * s + (v - 1)]) * 3;
      c0 = col[0];
      c1 = col[1];
      c2 = col[2];
    } else {
      c0 = color & 0xffu;
      c1 = (color >> 8) & 0xffu;
      c2 = (color >> 16) & 0xffu;
    }
    uint8_t *o = img + p * 3;
    o[0] = c0;
    o[1] = c1;
    o[2] = c2;
  }
}

int check_image(const uint8_t *img, int b, int h, int w, int r) {
  if (!img || b < 1 || h < 1 || w < 1 || r < 0) return PVN3D_ERR_INVALID_ARG;
  if (r > kMaxRadius || b > 65535 || h >= kMaxRadius * 2 || w >= kMaxRadius * 2) return PVN3D_ERR_UNSUPPORTED;
  return PVN3D_OK;
}

int check_workspace(const void *ws, size_t ws_bytes, int b, int h, int w) {
  if (!ws || (reinterpret_cast<uintptr_t>(ws) & 255u)) return PVN3D_ERR_INVALID_ARG;
  if (ws_bytes < pvn3d_vis_workspace_bytes(b, h, w)) return PVN3D_ERR_WORKSPACE;
  return PVN3D_OK;
}

int paint(uint8_t *img, const int *stamp, int b, int h, int w, const int *order, int s, const uint8_t *colors,
          unsigned color, cudaStream_t st) {
  const long long hw = static_cast<long long>(h) * w, total = hw * b;
  const long long blocks = min((total + kPaintThreads - 1) / kPaintThreads, static_cast<long long>(sm_count()) * 16);
  vis_paint_kernel<<<static_cast<unsigned>(blocks), kPaintThreads, 0, st>>>(img, stamp, hw, total, order, s, colors,
                                                                            color);
  return check_launch("vis_paint_kernel");
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_vis_workspace_bytes(int b, int h, int w) {
  if (b < 1 || h < 1 || w < 1) return 0;
  return align_up(static_cast<size_t>(b) * h * w * sizeof(int), 256);
}

extern "C" int pvn3d_vis_draw_poses(uint8_t *img, int b, int h, int w, const float *mesh_pts, const int *mesh_off,
                                    int n_cls, int max_pts, const void *poses, int poses_f64, const uint8_t *present,
                                    const int *order, int s, const double *k, double cam_scale, const uint8_t *colors,
                                    int r, void *workspace, size_t workspace_bytes, pvn3d_stream_t stream) {
  int rc = check_image(img, b, h, w, r);
  if (rc != PVN3D_OK) return rc;
  if (!mesh_pts || !mesh_off || !poses || !present || !order || !k || !colors || n_cls < 2 || max_pts < 1 || s < 1 ||
      (poses_f64 != 0 && poses_f64 != 1))
    return PVN3D_ERR_INVALID_ARG;
  if (s > 65535) return PVN3D_ERR_UNSUPPORTED;
  if ((rc = check_workspace(workspace, workspace_bytes, b, h, w)) != PVN3D_OK) return rc;
  int *stamp = static_cast<int *>(workspace);
  const cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(stamp, 0, static_cast<size_t>(b) * h * w * sizeof(int), st), "vis stamp memset");
  const PoseArgs a{mesh_pts, mesh_off, n_cls, poses, poses_f64, present, order, s, k, cam_scale};
  const dim3 grid(static_cast<unsigned>(ceil_div(max_pts, kMarkThreads)), static_cast<unsigned>(s),
                  static_cast<unsigned>(b));
  vis_mark_poses_kernel<<<grid, kMarkThreads, 0, st>>>(a, h, w, r, stamp);
  if ((rc = check_launch("vis_mark_poses_kernel")) != PVN3D_OK) return rc;
  return paint(img, stamp, b, h, w, order, s, colors, 0u, st);
}

extern "C" int pvn3d_vis_draw_p2ds(uint8_t *img, int h, int w, int *p2ds, int n, int r, unsigned color,
                                   void *workspace, size_t workspace_bytes, pvn3d_stream_t stream) {
  int rc = check_image(img, 1, h, w, r);
  if (rc != PVN3D_OK) return rc;
  if (n < 0 || (n > 0 && !p2ds) || color > 0xffffffu) return PVN3D_ERR_INVALID_ARG;
  if (n == 0) return PVN3D_OK;
  if ((rc = check_workspace(workspace, workspace_bytes, 1, h, w)) != PVN3D_OK) return rc;
  int *stamp = static_cast<int *>(workspace);
  const cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(stamp, 0, static_cast<size_t>(h) * w * sizeof(int), st), "vis stamp memset");
  vis_mark_p2ds_kernel<<<static_cast<unsigned>(ceil_div(n, kMarkThreads)), kMarkThreads, 0, st>>>(p2ds, n, h, w, r,
                                                                                                   stamp);
  if ((rc = check_launch("vis_mark_p2ds_kernel")) != PVN3D_OK) return rc;
  return paint(img, stamp, 1, h, w, nullptr, 0, nullptr, color, st);
}
