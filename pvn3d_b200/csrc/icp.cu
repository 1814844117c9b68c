// icp.cu -- my_icp (reference lib/utils/icp/icp.py:141-192) on device, batched over (frame, class),
// as pvn3d/eval_icp.py:94-185 runs it after the pose solver.
//
// Reference semantics: src = init * A; per iteration, every SCENE point B_j finds its nearest point
// of the current src (distances d_j, indices idx_j), T = best_fit_transform(src[idx], B), src = T src,
// stop when |prev_error - mean(d)| < tol (prev_error starts at 0); return best_fit_transform(A, src),
// the last distances and the last loop index.
//
// Here the accumulated pose P_k (src_k = P_k A) is kept instead of src, and P_{k+1} = T_k P_k with
// T_k = Kabsch(P_k A[idx], B), as the reference composes it.  Nearest neighbours are searched in the
// MODEL frame: q_j = P_k^-1 B_j against the fixed object-frame points A, so the model's grid is built
// once.  Candidates are compared by the camera-frame distance |B_j - P_k a|, the reference's metric;
// model-frame lower bounds are scaled by a bound on P_k's smallest singular value squared, so the
// match stays exact when P_k carries a float32 init's last-bit skew.  (For a rigid init the
// composition equals P_{k+1} = Kabsch(A[idx], B); composing keeps that skew exactly where the
// reference keeps it.)  The two differ only in rounding.
//
// One CTA per fit, every iteration inside the kernel (no host round trip, no cooperative launch).
// All arithmetic of the fit is float64; the per-iteration sums (distances, matched-model centroid,
// centred cross-covariance) are reduced in a fixed order, so results are reproducible bit for bit.
//
// Model structure (private to this file): per model, a uniform grid over the bounding box
// (<= kMaxCells cells, ~4 cells per point; a power-of-two cell edge on a grid origin that is a
// multiple of it, so cell faces are exact), the points sorted by cell as double4 (x, y, z, original
// index), cell ranges, and a per-cell Chebyshev distance (in cells) to the nearest non-empty cell.
// The search is exact: it visits shells of cells around the query's (clamped) cell and stops only when
// a lower bound on the distance to every unvisited cell -- kept conservative by a margin far above
// the rounding of the bound itself -- exceeds the best squared distance found; ties go to the lowest
// original index, so the result equals a float64 brute-force scan of |B_j - P_k a| over the model.
#include <cmath>

#include "common.cuh"
#include "kabsch.cuh"

namespace pvn3d {

int class_compact_launch(const int *mask, int b, int n, int n_cls, int *perm, int *cls_off,
                         uint8_t *present, cudaStream_t st);

namespace {

constexpr int kMaxCells = 16384;  // grid cells per model
constexpr int kBuildThreads = 1024;
constexpr int kFitThreads = 512;
constexpr int kFitWarps = kFitThreads / 32;
constexpr int kMaxIcpCls = 64;  // class_compact_launch limit
constexpr unsigned kModelsMagic = 0x49435031u;

struct ModelHdr {  // 64 bytes
  double lo[3];
  double h;       // cell edge
  double margin;  // absolute slack of every lower bound (covers cell-assignment rounding)
  int dims[3];
  int n_pts;
  int pt_off;  // first point of the model in the sorted-point and input tables
};

// directory at offset 0 of the models buffer: the kernels find every array from it
struct ModelsDir {
  unsigned magic;
  int n_models;
  int total_pts;
  int pad;
  size_t hdr, cell_start, cursor, dt, cell_of, pts, orig, total;
};

ModelsDir models_layout(int n_models, int total_pts) {
  ModelsDir L{};
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t at = off;
    off = align_up(off + (bytes ? bytes : 1), 256);
    return at;
  };
  const size_t nm = static_cast<size_t>(n_models), np = static_cast<size_t>(total_pts);
  take(sizeof(ModelsDir));
  L.magic = kModelsMagic;
  L.n_models = n_models;
  L.total_pts = total_pts;
  L.hdr = take(nm * sizeof(ModelHdr));
  L.cell_start = take(nm * (kMaxCells + 1) * 4);  // relative to the model's first point
  L.cursor = take(nm * kMaxCells * 4);            // build scratch
  L.dt = take(nm * kMaxCells);
  L.cell_of = take(np * 4);                       // build scratch
  L.pts = take(np * 32);
  L.orig = take(np * 12);                         // the input points, in input order
  L.total = off;
  return L;
}

struct ModelsView {
  const ModelHdr *hdr;
  const int *cell_start;
  const uint8_t *dt;
  const double4 *pts;
  const float *orig;
  int n_models;
};

__device__ __forceinline__ ModelsView models_view(const unsigned char *buf) {
  const ModelsDir *d = reinterpret_cast<const ModelsDir *>(buf);
  ModelsView v;
  v.hdr = reinterpret_cast<const ModelHdr *>(buf + d->hdr);
  v.cell_start = reinterpret_cast<const int *>(buf + d->cell_start);
  v.dt = buf + d->dt;
  v.pts = reinterpret_cast<const double4 *>(buf + d->pts);
  v.orig = reinterpret_cast<const float *>(buf + d->orig);
  v.n_models = d->n_models;
  return v;
}

// ------------------------------------------------------------------------------------------------
// model preparation: one CTA per model
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBuildThreads)
icp_build_kernel(const float *__restrict__ pts, const int *__restrict__ model_off,
                 unsigned char *__restrict__ buf) {
  const ModelsDir *dir = reinterpret_cast<const ModelsDir *>(buf);
  ModelHdr *hdrs = reinterpret_cast<ModelHdr *>(buf + dir->hdr);
  const int m = blockIdx.x, t = threadIdx.x;
  const unsigned lane = t & 31u, warp = t >> 5;
  int *cell_start = reinterpret_cast<int *>(buf + dir->cell_start) + static_cast<size_t>(m) * (kMaxCells + 1);
  int *cursor = reinterpret_cast<int *>(buf + dir->cursor) + static_cast<size_t>(m) * kMaxCells;
  uint8_t *dt = buf + dir->dt + static_cast<size_t>(m) * kMaxCells;
  const int p0 = model_off[m], np = model_off[m + 1] - p0;
  int *cell_of = reinterpret_cast<int *>(buf + dir->cell_of) + p0;
  double4 *spts = reinterpret_cast<double4 *>(buf + dir->pts) + p0;

  __shared__ double s_red[6][kBuildThreads / 32];
  __shared__ ModelHdr s_h;
  __shared__ int s_scan[kBuildThreads / 32];

  // bounding box
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = t; i < np; i += kBuildThreads)
    for (int d = 0; d < 3; ++d) {
      const double v = pts[static_cast<size_t>(p0 + i) * 3 + d];
      mn[d] = fmin(mn[d], v);
      mx[d] = fmax(mx[d], v);
    }
  for (int d = 0; d < 3; ++d)
    for (int o = 16; o > 0; o >>= 1) {
      mn[d] = fmin(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      mx[d] = fmax(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
    }
  if (lane == 0)
    for (int d = 0; d < 3; ++d) {
      s_red[d][warp] = mn[d];
      s_red[3 + d][warp] = mx[d];
    }
  __syncthreads();
  if (t == 0) {
    ModelHdr h{};
    h.n_pts = np;
    h.pt_off = p0;
    if (np == 0) {
      for (int d = 0; d < 3; ++d) {
        h.lo[d] = 0.0;
        h.dims[d] = 1;
      }
      h.h = 1.0;
      h.margin = 0.0;
    } else {
      double lo[3], hi[3], ext[3], e[3], emax = 0.0;
      for (int d = 0; d < 3; ++d) {
        lo[d] = INFINITY;
        hi[d] = -INFINITY;
        for (int w = 0; w < kBuildThreads / 32; ++w) {
          lo[d] = fmin(lo[d], s_red[d][w]);
          hi[d] = fmax(hi[d], s_red[3 + d][w]);
        }
        ext[d] = hi[d] - lo[d];
        emax = fmax(emax, ext[d]);
      }
      // cell-size heuristic: flat, collinear and one-point models count zero-width axes as thin slabs
      const double floor_e = 1e-3 * emax + 1e-9;
      for (int d = 0; d < 3; ++d) e[d] = fmax(ext[d], floor_e);
      const double target = fmin(static_cast<double>(kMaxCells), 4.0 * np);
      // The cell edge is a power of two and the origin a multiple of it, so every cell face
      // lo + k*h is exactly representable and a point or query on a face lands in a known cell.
      double cell = exp2(rint(log2(cbrt(e[0] * e[1] * e[2] / target))));
      double glo[3], gdim[3];
      for (;;) {
        double prod = 1.0;
        for (int d = 0; d < 3; ++d) {
          glo[d] = floor(lo[d] / cell) * cell;
          gdim[d] = floor((hi[d] - glo[d]) / cell) + 1.0;
          prod *= gdim[d];
        }
        if (prod <= kMaxCells) break;
        cell *= 2.0;
      }
      double cmax = 0.0;
      for (int d = 0; d < 3; ++d) {
        h.dims[d] = static_cast<int>(gdim[d]);
        h.lo[d] = glo[d];
        cmax = fmax(cmax, fmax(fabs(h.lo[d]), fabs(h.lo[d] + h.dims[d] * cell)));
      }
      h.h = cell;
      h.margin = 1e-6 * cell + 1e-13 * cmax;
    }
    s_h = h;
    hdrs[m] = h;
  }
  __syncthreads();
  const ModelHdr h = s_h;
  const int ncell = h.dims[0] * h.dims[1] * h.dims[2];
  for (int c = t; c < ncell; c += kBuildThreads) cursor[c] = 0;
  __syncthreads();
  for (int i = t; i < np; i += kBuildThreads) {
    int ci[3];
    for (int d = 0; d < 3; ++d) {
      const double f = floor((static_cast<double>(pts[static_cast<size_t>(p0 + i) * 3 + d]) - h.lo[d]) / h.h);
      ci[d] = f >= h.dims[d] - 1 ? h.dims[d] - 1 : (f > 0.0 ? static_cast<int>(f) : 0);
    }
    const int c = (ci[2] * h.dims[1] + ci[1]) * h.dims[0] + ci[0];
    cell_of[i] = c;
    atomicAdd(&cursor[c], 1);
  }
  __syncthreads();
  // exclusive scan of the counts: each thread owns a run of consecutive cells
  const int per = (ncell + kBuildThreads - 1) / kBuildThreads;
  const int c0 = min(t * per, ncell), c1 = min(c0 + per, ncell);
  int local = 0;
  for (int c = c0; c < c1; ++c) local += cursor[c];
  int incl = local;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) s_scan[warp] = incl;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int w = 0; w < kBuildThreads / 32; ++w) {
      const int v = s_scan[w];
      s_scan[w] = run;
      run += v;
    }
  }
  __syncthreads();
  int run = s_scan[warp] + incl - local;
  for (int c = c0; c < c1; ++c) {
    const int cnt = cursor[c];
    cell_start[c] = run;
    cursor[c] = run;
    run += cnt;
  }
  if (t == 0) cell_start[ncell] = np;
  __syncthreads();
  // order inside a cell is irrelevant: the search takes the minimum of (distance, original index)
  for (int i = t; i < np; i += kBuildThreads) {
    const int pos = atomicAdd(&cursor[cell_of[i]], 1);
    const float *p = pts + static_cast<size_t>(p0 + i) * 3;
    spts[pos] = make_double4(p[0], p[1], p[2], static_cast<double>(i));
  }
  float *orig = reinterpret_cast<float *>(buf + dir->orig) + static_cast<size_t>(p0) * 3;
  for (int i = t; i < np * 3; i += kBuildThreads) orig[i] = pts[static_cast<size_t>(p0) * 3 + i];
  // Chebyshev distance transform (in cells) to the nearest non-empty cell, capped at 255: the search
  // skips the shells below it.  In-place relaxation; values only decrease and never drop below the
  // true distance, so the fixed point is the transform.
  for (int c = t; c < ncell; c += kBuildThreads) dt[c] = (cell_start[c + 1] > cell_start[c]) ? 0 : 255;
  __syncthreads();
  if (np == 0) return;
  for (;;) {
    int changed = 0;
    for (int c = t; c < ncell; c += kBuildThreads) {
      const int cur = dt[c];
      if (cur == 0) continue;
      const int x = c % h.dims[0], y = (c / h.dims[0]) % h.dims[1], z = c / (h.dims[0] * h.dims[1]);
      int best = cur;
      for (int dz = -1; dz <= 1; ++dz)
        for (int dy = -1; dy <= 1; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx, yy = y + dy, zz = z + dz;
            if (xx < 0 || yy < 0 || zz < 0 || xx >= h.dims[0] || yy >= h.dims[1] || zz >= h.dims[2]) continue;
            best = min(best, dt[(zz * h.dims[1] + yy) * h.dims[0] + xx] + 1);
          }
      if (best < cur) {
        dt[c] = static_cast<uint8_t>(best);
        changed = 1;
      }
    }
    if (!__syncthreads_or(changed)) break;
  }
}

// ------------------------------------------------------------------------------------------------
// exact nearest neighbour of q among one model's points
// ------------------------------------------------------------------------------------------------
// squared distance as numpy evaluates ((q - p)**2).sum(-1): no fused multiply-add
__device__ __forceinline__ double sqdist64(double ax, double ay, double az, double bx, double by,
                                           double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// lower bounds are compared as lb * (1 - kRel) > best: the relative slack covers their own rounding
constexpr double kRel = 1e-9;

// src = P a for one model point (one fixed evaluation order wherever src points are formed)
__device__ __forceinline__ void apply_pose(const double *m, double x, double y, double z, double o[3]) {
  for (int r = 0; r < 3; ++r) o[r] = fma(m[r * 4 + 0], x, fma(m[r * 4 + 1], y, fma(m[r * 4 + 2], z, m[r * 4 + 3])));
}

// Lower bound on the smallest eigenvalue of M^T M (M = the pose's 3x3 block): 1 - ||M^T M - I||_F.
// Distances between model-frame points, scaled by it, bound camera-frame distances from below;
// it is 1 to rounding for a Kabsch pose and ~1 - 1e-7 for a float32 rotation promoted to float64.
__device__ double metric_shrink(const double p[12]) {
  double e = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double g = (i == j) ? -1.0 : 0.0;
      for (int k = 0; k < 3; ++k) g += p[k * 4 + i] * p[k * 4 + j];
      e += g * g;
    }
  return fmax(0.0, 1.0 - sqrt(e) - 1e-12);
}

// Nearest model point of the scene point b under the pose P_k, by the CAMERA-frame distance
// |b - P_k a| (the reference's metric, also when P_k is not exactly rigid).  The grid is walked
// around q = P_k^-1 b; a model-frame lower bound lb on |q - a|^2 bounds the camera-frame squared
// distance from below by lb * shrink, which is what every pruning test compares.
__device__ void nn_search(const ModelHdr &H, const int *__restrict__ cs, const uint8_t *__restrict__ dt,
                          const double4 *__restrict__ P, const double *pose, double shrink,
                          const double b[3], const double q[3], int &best_pos, double &best_d2,
                          unsigned &tests) {
  const double scale = shrink * (1.0 - kRel);
  int c0[3];
  double g0[3];
  for (int d = 0; d < 3; ++d) {
    const double f = floor((q[d] - H.lo[d]) / H.h);
    c0[d] = f >= H.dims[d] - 1 ? H.dims[d] - 1 : (f > 0.0 ? static_cast<int>(f) : 0);
    const double slo = H.lo[d] + c0[d] * H.h;
    g0[d] = fmax(0.0, fmax(slo - q[d], q[d] - (slo + H.h)) - H.margin);
  }
  best_d2 = INFINITY;
  best_pos = -1;
  int best_idx = 0x7fffffff;
  const int dimx = H.dims[0], dimy = H.dims[1], dimz = H.dims[2];
  for (int r = dt[(c0[2] * dimy + c0[1]) * dimx + c0[0]];; ++r) {
    if (r > 0) {
      // every cell of shells >= r lies at index distance >= r along some axis
      double lb = INFINITY;
      bool any = false;
      for (int d = 0; d < 3; ++d) {
        double base = 0.0;
        for (int e = 0; e < 3; ++e)
          if (e != d) base += g0[e] * g0[e];
        if (c0[d] - r >= 0) {
          const double gap = fmax(0.0, q[d] - (H.lo[d] + (c0[d] - r + 1) * H.h) - H.margin);
          lb = fmin(lb, base + gap * gap);
          any = true;
        }
        if (c0[d] + r < H.dims[d]) {
          const double gap = fmax(0.0, (H.lo[d] + (c0[d] + r) * H.h) - q[d] - H.margin);
          lb = fmin(lb, base + gap * gap);
          any = true;
        }
      }
      if (!any || lb * scale > best_d2) break;
    }
    const int z0 = max(c0[2] - r, 0), z1 = min(c0[2] + r, dimz - 1);
    const int y0 = max(c0[1] - r, 0), y1 = min(c0[1] + r, dimy - 1);
    for (int z = z0; z <= z1; ++z) {
      const double gz = fmax(0.0, fmax(H.lo[2] + z * H.h - q[2], q[2] - (H.lo[2] + (z + 1) * H.h)) - H.margin);
      const bool ez = (z == c0[2] - r) || (z == c0[2] + r);
      for (int y = y0; y <= y1; ++y) {
        const double gy = fmax(0.0, fmax(H.lo[1] + y * H.h - q[1], q[1] - (H.lo[1] + (y + 1) * H.h)) - H.margin);
        const bool full = ez || (y == c0[1] - r) || (y == c0[1] + r);
        const int step = full ? 1 : 2 * r;  // interior rows of the shell: only its two end cells
        for (int x = c0[0] - r; x <= c0[0] + r; x += step) {
          if (x < 0 || x >= dimx) continue;
          const double gx = fmax(0.0, fmax(H.lo[0] + x * H.h - q[0], q[0] - (H.lo[0] + (x + 1) * H.h)) - H.margin);
          if ((gx * gx + gy * gy + gz * gz) * scale > best_d2) continue;
          const int c = (z * dimy + y) * dimx + x;
          const int e = cs[c + 1];
          tests += static_cast<unsigned>(e - cs[c]);
          for (int k = cs[c]; k < e; ++k) {
            const double4 p = P[k];
            // the pose is re-read from shared memory per candidate: holding it in registers spills
            const volatile double *m = pose;
            double sp[3];
            for (int r2 = 0; r2 < 3; ++r2)
              sp[r2] = fma(m[r2 * 4 + 0], p.x, fma(m[r2 * 4 + 1], p.y, fma(m[r2 * 4 + 2], p.z, m[r2 * 4 + 3])));
            const double d2 = sqdist64(b[0], b[1], b[2], sp[0], sp[1], sp[2]);
            const int idx = static_cast<int>(p.w);
            if (d2 < best_d2 || (d2 == best_d2 && idx < best_idx)) {
              best_d2 = d2;
              best_idx = idx;
              best_pos = k;
            }
          }
          if (r == 0) break;
        }
      }
    }
  }
  if (best_pos < 0) {  // only for a NaN query
    best_pos = 0;
    best_d2 = NAN;
  }
}

// ------------------------------------------------------------------------------------------------
// the fit: one CTA per (frame, class) of a batch, or one CTA for an explicit scene set
// ------------------------------------------------------------------------------------------------
struct FitParams {
  const unsigned char *models;
  // batched selection (pcld != nullptr)
  const float *pcld;
  const int *perm, *cls_off;
  const float *init_f32;
  const uint8_t *present;
  int n, n_cls, max_pts, min_pts;
  // single fit
  const float *scene;
  const double *init_f64;
  int n_scene, model;
  int max_iter;
  double tol;
  double *pose_out;
  int *iters_out;
  double *err_out;
  uint8_t *refined_out;
  double *dist_out;
  int *match;  // [fits][match_stride] sorted model positions of the current matches
  int match_stride;
  unsigned long long *tests_out;
};

// Kabsch A -> B from the centred cross-covariance h (reference best_fit_transform).  The third
// singular vectors are taken as u1 x u2 and v1 x v2: R = V U^T is then the proper rotation the
// reference's reflection fix produces, and it stays accurate when H is nearly rank 2 (a flat face).
__device__ void kabsch_from_h(const double h[3][3], const double ca[3], const double cb[3], double pose[12]) {
  double u[3][3], s[3], v[3][3];
  svd3_jacobi(h, u, s, v);
  u[0][2] = u[1][0] * u[2][1] - u[2][0] * u[1][1];
  u[1][2] = u[2][0] * u[0][1] - u[0][0] * u[2][1];
  u[2][2] = u[0][0] * u[1][1] - u[1][0] * u[0][1];
  v[0][2] = v[1][0] * v[2][1] - v[2][0] * v[1][1];
  v[1][2] = v[2][0] * v[0][1] - v[0][0] * v[2][1];
  v[2][2] = v[0][0] * v[1][1] - v[1][0] * v[0][1];
  for (int r = 0; r < 3; ++r) {
    double tr = cb[r];
    for (int c = 0; c < 3; ++c) {
      double acc = 0;
      for (int k = 0; k < 3; ++k) acc += v[r][k] * u[c][k];  // R = Vt^T U^T
      pose[r * 4 + c] = acc;
      tr -= acc * ca[c];  // t = centroid_B - R centroid_A
    }
    pose[r * 4 + 3] = tr;
  }
}

// inverse of the affine map x -> M x + t (general 3x3 inverse: the init pose may be a float32 rotation)
__device__ void affine_inverse(const double p[12], double inv[12]) {
  const double a = p[0], b = p[1], c = p[2], d = p[4], e = p[5], f = p[6], g = p[8], hh = p[9], i = p[10];
  const double A = e * i - f * hh, B = -(d * i - f * g), C = d * hh - e * g;
  const double det = a * A + b * B + c * C;
  const double id = 1.0 / det;
  const double m[9] = {A * id, -(b * i - c * hh) * id, (b * f - c * e) * id,
                       B * id, (a * i - c * g) * id, -(a * f - c * d) * id,
                       C * id, -(a * hh - b * g) * id, (a * e - b * d) * id};
  for (int r = 0; r < 3; ++r) {
    inv[r * 4 + 0] = m[r * 3 + 0];
    inv[r * 4 + 1] = m[r * 3 + 1];
    inv[r * 4 + 2] = m[r * 3 + 2];
    inv[r * 4 + 3] = -(m[r * 3 + 0] * p[3] + m[r * 3 + 1] * p[7] + m[r * 3 + 2] * p[11]);
  }
}

// fixed-order block sum of K doubles per thread; the result is valid in thread 0
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double (*s_red)[9]) {
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) s_red[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double acc = 0.0;
      for (int w = 0; w < kFitWarps; ++w) acc += s_red[w][k];
      v[k] = acc;
    }
}

__global__ void __launch_bounds__(kFitThreads, 1) icp_fit_kernel(const FitParams p) {
  const ModelsView mv = models_view(p.models);
  const int f = blockIdx.x, t = threadIdx.x;
  __shared__ double s_pose[12], s_inv[12], s_ca[3], s_cb[3], s_shrink;
  __shared__ double s_red[kFitWarps][9];
  __shared__ float s_ca32[3];
  __shared__ int s_cnt, s_nsel, s_start, s_frame, s_model, s_skip, s_done;

  if (t == 0) {
    int cnt, model, skip, start = 0, frame = 0;
    if (p.pcld) {
      const int b = f / p.n_cls, c = f % p.n_cls;
      const int *off = p.cls_off + static_cast<size_t>(b) * (p.n_cls + 1);
      cnt = c > 0 ? off[c + 1] - off[c] : 0;
      start = off[c];
      frame = b;
      model = c;
      for (int k = 0; k < 12; ++k) s_pose[k] = static_cast<double>(p.init_f32[static_cast<size_t>(f) * 12 + k]);
      skip = c == 0 || !p.present[f] || cnt < p.min_pts || c >= mv.n_models;
    } else {
      cnt = p.n_scene;
      model = p.model;
      for (int k = 0; k < 12; ++k) s_pose[k] = p.init_f64[k];
      skip = model < 0 || model >= mv.n_models;
    }
    skip = skip || cnt < 1 || mv.hdr[model].n_pts < 1;
    s_cnt = cnt;
    s_nsel = p.pcld ? min(cnt, p.max_pts) : cnt;
    s_start = start;
    s_frame = frame;
    s_model = skip ? 0 : model;
    s_skip = skip;
    s_done = 0;
    if (!skip) {
      affine_inverse(s_pose, s_inv);
      s_shrink = metric_shrink(s_pose);
    }
  }
  __syncthreads();
  if (s_skip) {
    if (t < 12) p.pose_out[static_cast<size_t>(f) * 12 + t] = s_pose[t];
    if (t == 0) {
      p.iters_out[f] = p.pcld ? 0 : -1;
      p.err_out[f] = 0.0;
      if (p.refined_out) p.refined_out[f] = 0;
    }
    return;
  }
  const int cnt = s_cnt, nsel = s_nsel;
  const ModelHdr H = mv.hdr[s_model];
  const int *cs = mv.cell_start + static_cast<size_t>(s_model) * (kMaxCells + 1);
  const uint8_t *dtm = mv.dt + static_cast<size_t>(s_model) * kMaxCells;
  const double4 *P = mv.pts + H.pt_off;
  int *match = p.match + static_cast<size_t>(f) * p.match_stride;
  // scene point j of the fit: the class's points in ascending index, strided when cnt > max_pts
  auto scene_pt = [&](int j, double b[3]) {
    const float *src;
    if (p.pcld) {
      const int qpos = static_cast<int>(static_cast<long long>(j) * cnt / nsel);
      const int i = p.perm[static_cast<size_t>(s_frame) * p.n + s_start + qpos];
      src = p.pcld + (static_cast<size_t>(s_frame) * p.n + i) * 3;
    } else {
      src = p.scene + static_cast<size_t>(j) * 3;
    }
    b[0] = src[0];
    b[1] = src[1];
    b[2] = src[2];
  };
  // scene centroid (constant over the iterations)
  {
    double acc[3] = {0, 0, 0};
    for (int j = t; j < nsel; j += kFitThreads) {
      double b[3];
      scene_pt(j, b);
      acc[0] += b[0];
      acc[1] += b[1];
      acc[2] += b[2];
    }
    block_sum<3>(acc, s_red);
    if (t == 0)
      for (int d = 0; d < 3; ++d) s_cb[d] = acc[d] / nsel;
  }
  __syncthreads();
  unsigned tests = 0;
  double prev = 0.0, mean = 0.0;
  int it = 0;
  for (it = 0; it < p.max_iter; ++it) {
    // P_k and P_k^-1 are read from shared memory (stable until the barrier after pass 2)
    const double *inv = s_inv, *cur = s_pose;
    // src_k = P_k A: the matched source point and its distance are evaluated in the camera frame as
    // the reference does, so a non-rigid init (a float32 rotation) is carried exactly like its src
    auto src_pt = [&](const double4 &a, double o[3]) { apply_pose(cur, a.x, a.y, a.z, o); };
    const double shrink = s_shrink;
    // pass 1: nearest model point of every scene point, searched in the model frame
    double acc[4] = {0, 0, 0, 0};
    for (int j = t; j < nsel; j += kFitThreads) {
      double b[3], q[3];
      scene_pt(j, b);
      for (int r = 0; r < 3; ++r) q[r] = inv[r * 4 + 0] * b[0] + inv[r * 4 + 1] * b[1] + inv[r * 4 + 2] * b[2] + inv[r * 4 + 3];
      int pos;
      double d2;
      nn_search(H, cs, dtm, P, cur, shrink, b, q, pos, d2, tests);
      match[j] = pos;
      double s[3];
      src_pt(P[pos], s);
      const double d = sqrt(d2);
      if (p.dist_out) p.dist_out[j] = d;
      acc[0] += d;
      acc[1] += s[0];
      acc[2] += s[1];
      acc[3] += s[2];
    }
    block_sum<4>(acc, s_red);
    if (t == 0) {
      mean = acc[0] / nsel;
      for (int d = 0; d < 3; ++d) s_ca[d] = acc[1 + d] / nsel;
    }
    __syncthreads();
    // pass 2: centred cross-covariance of (src[idx], B)
    double hh[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const double ca[3] = {s_ca[0], s_ca[1], s_ca[2]}, cb[3] = {s_cb[0], s_cb[1], s_cb[2]};
    for (int j = t; j < nsel; j += kFitThreads) {
      double b[3];
      scene_pt(j, b);
      double s[3];
      src_pt(P[match[j]], s);
      const double ax = s[0] - ca[0], ay = s[1] - ca[1], az = s[2] - ca[2];
      const double bx = b[0] - cb[0], by = b[1] - cb[1], bz = b[2] - cb[2];
      hh[0] += ax * bx; hh[1] += ax * by; hh[2] += ax * bz;
      hh[3] += ay * bx; hh[4] += ay * by; hh[5] += ay * bz;
      hh[6] += az * bx; hh[7] += az * by; hh[8] += az * bz;
    }
    block_sum<9>(hh, s_red);
    if (t == 0) {
      const double h3[3][3] = {{hh[0], hh[1], hh[2]}, {hh[3], hh[4], hh[5]}, {hh[6], hh[7], hh[8]}};
      double tk[12], pose[12];
      kabsch_from_h(h3, ca, cb, tk);
      // P_{k+1} = T_k P_k  (the reference's src = T src)
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c)
          pose[r * 4 + c] = tk[r * 4 + 0] * cur[0 * 4 + c] + tk[r * 4 + 1] * cur[1 * 4 + c] +
                            tk[r * 4 + 2] * cur[2 * 4 + c] + (c == 3 ? tk[r * 4 + 3] : 0.0);
      for (int k = 0; k < 12; ++k) s_pose[k] = pose[k];
      affine_inverse(pose, s_inv);
      s_shrink = metric_shrink(pose);
      s_done = fabs(prev - mean) < p.tol;
      prev = mean;
    }
    __syncthreads();
    if (s_done) break;  // thread 0 rewrites s_done only after the next iteration's barriers
  }
  if (it == p.max_iter) it = p.max_iter - 1;

  // The reference returns best_fit_transform(A, src), src = P A, with A float32 as eval_icp passes it:
  // numpy then takes A's centroid as a sequential float32 sum / P and centres A in float32.  That
  // shifts t by up to a float32 ulp of the centroid; it is reproduced here so that T matches.
  {
    const float *a32 = mv.orig + static_cast<size_t>(H.pt_off) * 3;
    const int np = H.n_pts;
    double pose[12];
    for (int k = 0; k < 12; ++k) pose[k] = s_pose[k];
    if (t == 0) {
      float s0 = 0.f, s1 = 0.f, s2 = 0.f;
      for (int i = 0; i < np; ++i) {
        s0 = __fadd_rn(s0, a32[i * 3 + 0]);
        s1 = __fadd_rn(s1, a32[i * 3 + 1]);
        s2 = __fadd_rn(s2, a32[i * 3 + 2]);
      }
      const float fn = static_cast<float>(np);
      s_ca32[0] = __fdiv_rn(s0, fn);
      s_ca32[1] = __fdiv_rn(s1, fn);
      s_ca32[2] = __fdiv_rn(s2, fn);
    }
    double acc[3] = {0, 0, 0};
    for (int i = t; i < np; i += kFitThreads) {
      const double ax = a32[i * 3 + 0], ay = a32[i * 3 + 1], az = a32[i * 3 + 2];
      for (int r = 0; r < 3; ++r) acc[r] += pose[r * 4 + 0] * ax + pose[r * 4 + 1] * ay + pose[r * 4 + 2] * az + pose[r * 4 + 3];
    }
    block_sum<3>(acc, s_red);
    if (t == 0)
      for (int d = 0; d < 3; ++d) s_cb[d] = acc[d] / np;
    __syncthreads();
    const float c32[3] = {s_ca32[0], s_ca32[1], s_ca32[2]};
    const double cb[3] = {s_cb[0], s_cb[1], s_cb[2]};
    double hh[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = t; i < np; i += kFitThreads) {
      double aa[3], bb[3];
      for (int d = 0; d < 3; ++d) aa[d] = __fsub_rn(a32[i * 3 + d], c32[d]);
      const double ax = a32[i * 3 + 0], ay = a32[i * 3 + 1], az = a32[i * 3 + 2];
      for (int r = 0; r < 3; ++r)
        bb[r] = pose[r * 4 + 0] * ax + pose[r * 4 + 1] * ay + pose[r * 4 + 2] * az + pose[r * 4 + 3] - cb[r];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) hh[r * 3 + c] += aa[r] * bb[c];
    }
    block_sum<9>(hh, s_red);
    if (t == 0) {
      const double h3[3][3] = {{hh[0], hh[1], hh[2]}, {hh[3], hh[4], hh[5]}, {hh[6], hh[7], hh[8]}};
      const double ca[3] = {c32[0], c32[1], c32[2]};
      kabsch_from_h(h3, ca, cb, pose);
      for (int k = 0; k < 12; ++k) s_pose[k] = pose[k];
    }
    __syncthreads();
  }
  if (t < 12) p.pose_out[static_cast<size_t>(f) * 12 + t] = s_pose[t];
  if (t == 0) {
    p.iters_out[f] = it;
    p.err_out[f] = mean;
    if (p.refined_out) p.refined_out[f] = 1;
  }
  if (p.tests_out) {
    unsigned long long v = tests;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((t & 31) == 0) atomicAdd(p.tests_out, v);
  }
}

struct IcpWsLayout {
  size_t stats, perm, cls_off, match, total;
};
IcpWsLayout icp_ws_layout(int b, int n, int n_cls, int max_pts) {
  IcpWsLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t at = off;
    off = align_up(off + (bytes ? bytes : 1), 256);
    return at;
  };
  L.stats = take(8);
  L.perm = take(static_cast<size_t>(b) * n * 4);
  L.cls_off = take(static_cast<size_t>(b) * (n_cls + 1) * 4);
  L.match = take(static_cast<size_t>(b) * n_cls * max_pts * 4);
  L.total = off;
  return L;
}

bool models_ok(const void *models) {
  return models && (reinterpret_cast<uintptr_t>(models) & 255u) == 0;
}

}  // namespace
}  // namespace pvn3d

using namespace pvn3d;

extern "C" size_t pvn3d_icp_models_bytes(int n_models, int total_pts) {
  if (n_models < 1 || total_pts < 0) return 0;
  return models_layout(n_models, total_pts).total;
}

extern "C" int pvn3d_icp_build_models(const float *pts, const int *model_off, int n_models,
                                      int total_pts, void *buf, size_t bytes, pvn3d_stream_t stream) {
  if (!model_off || !models_ok(buf) || n_models < 1 || total_pts < 0 || (total_pts > 0 && !pts))
    return PVN3D_ERR_INVALID_ARG;
  if (n_models > 65535) return PVN3D_ERR_UNSUPPORTED;
  const ModelsDir L = models_layout(n_models, total_pts);
  if (bytes < L.total) return PVN3D_ERR_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemcpyAsync(buf, &L, sizeof(L), cudaMemcpyHostToDevice, st), "icp models directory");
  icp_build_kernel<<<n_models, kBuildThreads, 0, st>>>(pts, model_off, static_cast<unsigned char *>(buf));
  return check_launch("icp_build_kernel");
}

extern "C" size_t pvn3d_icp_workspace_bytes(int b, int n, int n_cls, int max_pts) {
  if (b < 1 || n < 1 || n_cls < 1 || max_pts < 1) return 0;
  if (static_cast<long long>(b) * n_cls * max_pts > 0x7fffffffll || static_cast<long long>(b) * n > 0x7fffffffll)
    return 0;
  return icp_ws_layout(b, n, n_cls, max_pts).total;
}

extern "C" int pvn3d_icp_refine_batch(const void *models, const float *pcld, const int *mask, int b,
                                      int n, int n_cls, const float *init_poses, const uint8_t *present,
                                      int max_pts, int min_pts, int max_iter, double tol,
                                      double *poses_out, int *iters_out, double *err_out,
                                      uint8_t *refined_out, void *workspace, size_t workspace_bytes,
                                      pvn3d_stream_t stream) {
  if (!models_ok(models) || !pcld || !mask || !init_poses || !present || !poses_out || !iters_out ||
      !err_out || !refined_out || !workspace || b < 0 || n < 1 || n_cls < 2 || max_pts < 1 ||
      min_pts < 0 || max_iter < 1 || !(tol >= 0.0))
    return PVN3D_ERR_INVALID_ARG;
  if (b == 0) return PVN3D_OK;
  if (n_cls > kMaxIcpCls) return PVN3D_ERR_UNSUPPORTED;
  if (static_cast<long long>(b) * n_cls * max_pts > 0x7fffffffll || static_cast<long long>(b) * n > 0x7fffffffll)
    return PVN3D_ERR_UNSUPPORTED;
  const IcpWsLayout L = icp_ws_layout(b, n, n_cls, max_pts);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(ws + L.stats, 0, 8, st), "icp stats reset");
  int *perm = reinterpret_cast<int *>(ws + L.perm), *cls_off = reinterpret_cast<int *>(ws + L.cls_off);
  int rc = class_compact_launch(mask, b, n, n_cls, perm, cls_off, nullptr, st);
  if (rc != PVN3D_OK) return rc;
  FitParams p{};
  p.models = static_cast<const unsigned char *>(models);
  p.pcld = pcld;
  p.perm = perm;
  p.cls_off = cls_off;
  p.init_f32 = init_poses;
  p.present = present;
  p.n = n;
  p.n_cls = n_cls;
  p.max_pts = max_pts;
  p.min_pts = min_pts;
  p.max_iter = max_iter;
  p.tol = tol;
  p.pose_out = poses_out;
  p.iters_out = iters_out;
  p.err_out = err_out;
  p.refined_out = refined_out;
  p.match = reinterpret_cast<int *>(ws + L.match);
  p.match_stride = max_pts;
  p.tests_out = reinterpret_cast<unsigned long long *>(ws + L.stats);
  icp_fit_kernel<<<b * n_cls, kFitThreads, 0, st>>>(p);
  return check_launch("icp_fit_kernel");
}

extern "C" int pvn3d_icp_fit(const void *models, int model, const float *scene, int n,
                             const double *init_pose, int max_iter, double tol, double *pose_out,
                             double *dist_out, int *iter_out, double *err_out, void *workspace,
                             size_t workspace_bytes, pvn3d_stream_t stream) {
  if (!models_ok(models) || !scene || !init_pose || !pose_out || !iter_out || !err_out || !workspace ||
      n < 1 || model < 0 || max_iter < 1 || !(tol >= 0.0))
    return PVN3D_ERR_INVALID_ARG;
  const IcpWsLayout L = icp_ws_layout(1, n, 1, n);
  if (workspace_bytes < L.total) return PVN3D_ERR_WORKSPACE;
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return PVN3D_ERR_INVALID_ARG;
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  cudaStream_t st = as_stream(stream);
  PVN3D_CUDA_TRY(cudaMemsetAsync(ws + L.stats, 0, 8, st), "icp stats reset");
  FitParams p{};
  p.models = static_cast<const unsigned char *>(models);
  p.scene = scene;
  p.init_f64 = init_pose;
  p.n_scene = n;
  p.model = model;
  p.max_iter = max_iter;
  p.tol = tol;
  p.pose_out = pose_out;
  p.iters_out = iter_out;
  p.err_out = err_out;
  p.dist_out = dist_out;
  p.match = reinterpret_cast<int *>(ws + L.match);
  p.match_stride = n;
  p.tests_out = reinterpret_cast<unsigned long long *>(ws + L.stats);
  icp_fit_kernel<<<1, kFitThreads, 0, st>>>(p);
  return check_launch("icp_fit_kernel");
}
