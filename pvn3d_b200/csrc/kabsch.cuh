// kabsch.cuh -- float64 3x3 SVD and determinant shared by the pose fit (poses.cu) and ICP (icp.cu)
#pragma once
#include <cmath>

namespace pvn3d {

// H = U diag(s) V^T with s descending (numpy convention; the reflection fix flips the LAST one)
__device__ inline void svd3_jacobi(const double h[3][3], double u[3][3], double s[3], double v[3][3]) {
  double a[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      a[i][j] = h[i][j];
      v[i][j] = (i == j) ? 1.0 : 0.0;
    }
  // one-sided (Hestenes) Jacobi: rotate column pairs of A until they are orthogonal; A = U S, H = U S V^T
  for (int sweep = 0; sweep < 60; ++sweep) {
    double offd = 0.0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; ++i) {
          alpha += a[i][p] * a[i][p];
          beta += a[i][q] * a[i][q];
          gamma += a[i][p] * a[i][q];
        }
        // purely relative: an absolute floor would leave small columns (|a_p||a_q| below it, e.g. the second and
        // third of a nearly collinear H at a 1e-4 m scale) unrotated, and U far from orthonormal
        const double lim = 1e-16 * sqrt(alpha * beta);
        if (fabs(gamma) <= lim) continue;
        offd = fmax(offd, fabs(gamma) / (sqrt(alpha * beta) + 1e-300));
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + tt * tt), sn = c * tt;
        for (int i = 0; i < 3; ++i) {
          const double ap = a[i][p], aq = a[i][q];
          a[i][p] = c * ap - sn * aq;
          a[i][q] = sn * ap + c * aq;
          const double vp = v[i][p], vq = v[i][q];
          v[i][p] = c * vp - sn * vq;
          v[i][q] = sn * vp + c * vq;
        }
      }
    if (offd < 1e-15) break;
  }
  for (int j = 0; j < 3; ++j) s[j] = sqrt(a[0][j] * a[0][j] + a[1][j] * a[1][j] + a[2][j] * a[2][j]);
  // sort singular values descending (numpy convention; the reflection fix flips the LAST one)
  int ord[3] = {0, 1, 2};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2 - i; ++j)
      if (s[ord[j]] < s[ord[j + 1]]) {
        const int tmp = ord[j];
        ord[j] = ord[j + 1];
        ord[j + 1] = tmp;
      }
  double ss[3], vv[3][3], aa[3][3];
  for (int j = 0; j < 3; ++j) {
    ss[j] = s[ord[j]];
    for (int i = 0; i < 3; ++i) {
      vv[i][j] = v[i][ord[j]];
      aa[i][j] = a[i][ord[j]];
    }
  }
  const double tiny = 1e-12 * (ss[0] > 0 ? ss[0] : 1.0);
  for (int j = 0; j < 3; ++j) {
    s[j] = ss[j];
    for (int i = 0; i < 3; ++i) {
      v[i][j] = vv[i][j];
      u[i][j] = ss[j] > tiny ? aa[i][j] / ss[j] : 0.0;
    }
  }
  // complete a rank-deficient U to an orthonormal basis (rotation is then not unique anyway)
  if (!(s[0] > tiny)) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) u[i][j] = (i == j) ? 1.0 : 0.0;
    return;
  }
  if (!(s[1] > tiny)) {
    // any unit vector orthogonal to u0
    int m = 0;
    if (fabs(u[1][0]) < fabs(u[m][0])) m = 1;
    if (fabs(u[2][0]) < fabs(u[m][0])) m = 2;
    double e[3] = {0, 0, 0};
    e[m] = 1.0;
    const double dot = u[m][0];
    double w[3], nrm = 0;
    for (int i = 0; i < 3; ++i) {
      w[i] = e[i] - dot * u[i][0];
      nrm += w[i] * w[i];
    }
    nrm = sqrt(nrm);
    for (int i = 0; i < 3; ++i) u[i][1] = w[i] / nrm;
  }
  if (!(s[2] > tiny)) {
    u[0][2] = u[1][0] * u[2][1] - u[2][0] * u[1][1];
    u[1][2] = u[2][0] * u[0][1] - u[0][0] * u[2][1];
    u[2][2] = u[0][0] * u[1][1] - u[1][0] * u[0][1];
  }
}

__device__ __forceinline__ double det3(const double r[3][3]) {
  return r[0][0] * (r[1][1] * r[2][2] - r[1][2] * r[2][1]) -
         r[0][1] * (r[1][0] * r[2][2] - r[1][2] * r[2][0]) +
         r[0][2] * (r[1][0] * r[2][1] - r[1][1] * r[2][0]);
}

}  // namespace pvn3d
