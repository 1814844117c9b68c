/*
 * pn2_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, OpenMP over the batch) of the reference's PointNet++ CUDA ops, used
 * only as the parity checker by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs.  Nothing under pvn3d_b200/ may call it.
 *
 * Every function follows the reference kernel cited above it LITERALLY (same loop order, same
 * strict comparisons, same tree reduction), and evaluates squared distances with the FMA
 * contraction nvcc chose for the reference (checked in the SASS of oracle/_ref/_ext.so):
 *     d2 = fma(dz,dz, fma(dx,dx, dy*dy))
 * Build: see oracle/Makefile (-ffp-contract=off so that only the explicit fmaf() calls fuse).
 *
 * Pinning: the reference has no CPU path (ball_query.cpp:28 "CPU not supported") and no golden
 * vectors, so this restatement is pinned on the GPU box against oracle/_ref/_ext.so (the reference
 * sources compiled unmodified) by tests/test_oracle_vs_reference_gpu.py, and through the committed
 * fixtures tests/golden/pn2_ref_*.npz that the same reference build produced.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline float ref_sqdist(float dx, float dy, float dz) {
  return fmaf(dz, dz, fmaf(dx, dx, dy * dy));
}

/* out[i * n + k] = the squared distance every op below evaluates between q[i] and pts[k] (q - pts, the operand
 * order of ball_query and three_nn; the square is symmetric).  Lets the tests place points within one ulp of a
 * radius and restate single rows of an op in numpy without re-deriving the contraction. */
void oracle_sqdist(const float *q, int nq, const float *pts, int n, float *out) {
  for (int i = 0; i < nq; ++i)
    for (int k = 0; k < n; ++k)
      out[(size_t)i * n + k] = ref_sqdist(q[i * 3 + 0] - pts[k * 3 + 0], q[i * 3 + 1] - pts[k * 3 + 1],
                                          q[i * 3 + 2] - pts[k * 3 + 2]);
}

/* cuda_utils.h:15-19 */
int oracle_opt_n_threads(int work_size) {
  const int pow_2 = (int)(log((double)work_size) / log(2.0));
  int v = 1 << pow_2;
  if (v > 512) v = 512;
  if (v < 1) v = 1;
  return v;
}

/* sampling_gpu.cu:69-173 (+ sampling.cpp:73-75: temp filled with 1e10).
 * Emulates the CUDA block: `bs` threads, thread tid owns k = tid, tid+bs, ...; then the
 * shared-memory tree of __update() calls (sampling_gpu.cu:59-65). */
void oracle_furthest_point_sampling(const float *xyz, int b, int n, int m, int *idxs) {
  if (m <= 0) return;
  const int bs = oracle_opt_n_threads(n);
#pragma omp parallel for schedule(dynamic)
  for (int bi = 0; bi < b; ++bi) {
    const float *dataset = xyz + (size_t)bi * n * 3;
    int *out = idxs + (size_t)bi * m;
    float *temp = (float *)malloc(sizeof(float) * (size_t)n);
    float *dists = (float *)malloc(sizeof(float) * (size_t)bs);
    int *dists_i = (int *)malloc(sizeof(int) * (size_t)bs);
    for (int k = 0; k < n; ++k) temp[k] = 1e10f;
    int old = 0;
    out[0] = old;
    for (int j = 1; j < m; ++j) {
      const float x1 = dataset[old * 3 + 0], y1 = dataset[old * 3 + 1], z1 = dataset[old * 3 + 2];
      for (int tid = 0; tid < bs; ++tid) {
        int besti = 0;
        float best = -1;
        for (int k = tid; k < n; k += bs) {
          const float x2 = dataset[k * 3 + 0], y2 = dataset[k * 3 + 1], z2 = dataset[k * 3 + 2];
          const float mag = fmaf(z2, z2, fmaf(x2, x2, y2 * y2));
          if ((double)mag <= 1e-3) continue; /* :100-101, double literal */
          const float d = ref_sqdist(x2 - x1, y2 - y1, z2 - z1);
          const float d2 = fminf(d, temp[k]);
          temp[k] = d2;
          besti = d2 > best ? k : besti;
          best = d2 > best ? d2 : best;
        }
        dists[tid] = best;
        dists_i[tid] = besti;
      }
      for (int s = bs / 2; s >= 1; s >>= 1) { /* :115-168 */
        for (int tid = 0; tid < s; ++tid) {
          const float v1 = dists[tid], v2 = dists[tid + s];
          const int i1 = dists_i[tid], i2 = dists_i[tid + s];
          dists[tid] = fmaxf(v1, v2);
          dists_i[tid] = v2 > v1 ? i2 : i1;
        }
      }
      old = dists_i[0];
      out[j] = old;
    }
    free(temp);
    free(dists);
    free(dists_i);
  }
}

/* sampling_gpu.cu:8-20 */
void oracle_gather_points(const float *points, const int *idx, int b, int c, int n, int m,
                          float *out) {
#pragma omp parallel for collapse(2)
  for (int i = 0; i < b; ++i)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < m; ++j) {
        const int a = idx[(size_t)i * m + j];
        out[((size_t)i * c + l) * m + j] = points[((size_t)i * c + l) * n + a];
      }
}

/* sampling_gpu.cu:34-47 (atomicAdd order is irrelevant for the tests: tolerance compare) */
void oracle_gather_points_grad(const float *grad_out, const int *idx, int b, int c, int n, int m,
                               float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * n);
  for (int i = 0; i < b; ++i)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < m; ++j) {
        const int a = idx[(size_t)i * m + j];
        grad_points[((size_t)i * c + l) * n + a] += grad_out[((size_t)i * c + l) * m + j];
      }
}

/* ball_query_gpu.cu:9-44; idx zero-initialised by the host wrapper (ball_query.cpp:19-21) */
void oracle_ball_query(const float *new_xyz, const float *xyz, int b, int n, int m, float radius,
                       int nsample, int *idx) {
  const float radius2 = radius * radius;
  memset(idx, 0, sizeof(int) * (size_t)b * m * nsample);
#pragma omp parallel for collapse(2) schedule(dynamic, 64)
  for (int bi = 0; bi < b; ++bi)
    for (int j = 0; j < m; ++j) {
      const float *pts = xyz + (size_t)bi * n * 3;
      const float *q = new_xyz + ((size_t)bi * m + j) * 3;
      int *row = idx + ((size_t)bi * m + j) * nsample;
      const float new_x = q[0], new_y = q[1], new_z = q[2];
      for (int k = 0, cnt = 0; k < n && cnt < nsample; ++k) {
        const float d2 = ref_sqdist(new_x - pts[k * 3 + 0], new_y - pts[k * 3 + 1],
                                    new_z - pts[k * 3 + 2]);
        if (d2 < radius2) {
          if (cnt == 0)
            for (int l = 0; l < nsample; ++l) row[l] = k;
          row[cnt] = k;
          ++cnt;
        }
      }
    }
}

/* group_points_gpu.cu:8-28 */
void oracle_group_points(const float *points, const int *idx, int b, int c, int n, int npoints,
                         int nsample, float *out) {
#pragma omp parallel for collapse(2)
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < npoints; ++j)
        for (int k = 0; k < nsample; ++k) {
          const int ii = idx[((size_t)bi * npoints + j) * nsample + k];
          out[(((size_t)bi * c + l) * npoints + j) * nsample + k] =
              points[((size_t)bi * c + l) * n + ii];
        }
}

/* group_points_gpu.cu:43-64 */
void oracle_group_points_grad(const float *grad_out, const int *idx, int b, int c, int n,
                              int npoints, int nsample, float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * n);
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < npoints; ++j)
        for (int k = 0; k < nsample; ++k) {
          const int ii = idx[((size_t)bi * npoints + j) * nsample + k];
          grad_points[((size_t)bi * c + l) * n + ii] +=
              grad_out[(((size_t)bi * c + l) * npoints + j) * nsample + k];
        }
}

/* interpolate_gpu.cu:9-59: comparisons in double against bests seeded with 1e40 */
void oracle_three_nn(const float *unknown, const float *known, int b, int n, int m, float *dist2,
                     int *idx) {
#pragma omp parallel for collapse(2) schedule(dynamic, 64)
  for (int bi = 0; bi < b; ++bi)
    for (int j = 0; j < n; ++j) {
      const float *kn = known + (size_t)bi * m * 3;
      const float *u = unknown + ((size_t)bi * n + j) * 3;
      const float ux = u[0], uy = u[1], uz = u[2];
      double best1 = 1e40, best2 = 1e40, best3 = 1e40;
      int besti1 = 0, besti2 = 0, besti3 = 0;
      for (int k = 0; k < m; ++k) {
        const float d = ref_sqdist(ux - kn[k * 3 + 0], uy - kn[k * 3 + 1], uz - kn[k * 3 + 2]);
        if (d < best1) {
          best3 = best2; besti3 = besti2;
          best2 = best1; besti2 = besti1;
          best1 = d;     besti1 = k;
        } else if (d < best2) {
          best3 = best2; besti3 = besti2;
          best2 = d;     besti2 = k;
        } else if (d < best3) {
          best3 = d;     besti3 = k;
        }
      }
      float *dd = dist2 + ((size_t)bi * n + j) * 3;
      int *oo = idx + ((size_t)bi * n + j) * 3;
      dd[0] = (float)best1; dd[1] = (float)best2; dd[2] = (float)best3;
      oo[0] = besti1; oo[1] = besti2; oo[2] = besti3;
    }
}

/* interpolate_gpu.cu:72-101; contraction observed in the reference SASS (oracle/_ref build):
 * t = p2*w2 ; t = fma(p1,w1,t) ; out = fma(p3,w3,t)   (pinned on the GPU against the reference) */
void oracle_three_interpolate(const float *points, const int *idx, const float *weight, int b,
                              int c, int m, int n, float *out) {
#pragma omp parallel for collapse(2)
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < n; ++j) {
        const float *w = weight + ((size_t)bi * n + j) * 3;
        const int *ii = idx + ((size_t)bi * n + j) * 3;
        const float *row = points + ((size_t)bi * c + l) * m;
        out[((size_t)bi * c + l) * n + j] =
            fmaf(row[ii[2]], w[2], fmaf(row[ii[0]], w[0], row[ii[1]] * w[1]));
      }
}

/* interpolate_gpu.cu:116-143 -- the INTENDED gradient (the reference host wrapper never launches
 * this kernel: interpolate.cpp:89-93 calls the forward wrapper; SURVEY App. C) */
void oracle_three_interpolate_grad(const float *grad_out, const int *idx, const float *weight,
                                   int b, int c, int n, int m, float *grad_points) {
  memset(grad_points, 0, sizeof(float) * (size_t)b * c * m);
  for (int bi = 0; bi < b; ++bi)
    for (int l = 0; l < c; ++l)
      for (int j = 0; j < n; ++j) {
        const float *w = weight + ((size_t)bi * n + j) * 3;
        const int *ii = idx + ((size_t)bi * n + j) * 3;
        const float g = grad_out[((size_t)bi * c + l) * n + j];
        float *row = grad_points + ((size_t)bi * c + l) * m;
        row[ii[0]] += g * w[0];
        row[ii[1]] += g * w[1];
        row[ii[2]] += g * w[2];
      }
}

/* QueryAndGroup.forward (pointnet2_utils.py:311-321) composed from the ops above:
 * out[B,3+C,M,S] = cat(group(xyz^T) - new_xyz, group(features)) ; features channel-major [B,C,N] */
void oracle_query_and_group(const float *xyz, const float *new_xyz, const float *features, int b,
                            int n, int m, int c, float radius, int nsample, int *idx, float *out) {
  oracle_ball_query(new_xyz, xyz, b, n, m, radius, nsample, idx);
#pragma omp parallel for collapse(2)
  for (int bi = 0; bi < b; ++bi)
    for (int j = 0; j < m; ++j)
      for (int k = 0; k < nsample; ++k) {
        const int ii = idx[((size_t)bi * m + j) * nsample + k];
        const size_t plane = (size_t)m * nsample, slot = (size_t)j * nsample + k;
        float *o = out + (size_t)bi * (3 + c) * plane;
        for (int d = 0; d < 3; ++d)
          o[d * plane + slot] = xyz[((size_t)bi * n + ii) * 3 + d] - new_xyz[((size_t)bi * m + j) * 3 + d];
        for (int l = 0; l < c; ++l)
          o[(3 + l) * plane + slot] = features[((size_t)bi * c + l) * n + ii];
      }
}
