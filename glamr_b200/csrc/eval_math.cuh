// Per-frame similarity Procrustes (lib/utils/torch_transform.py:282-345) -- shared by eval_kernels.cu and the host test harness.
#pragma once
#include "glamr_math.cuh"

namespace glamr {

// 3x3 SVD K = U diag(s) V^T by one-sided Jacobi on the columns (fp64).  U's columns are normalised; a zero singular
// value leaves the corresponding column of U completed by a cross product so that det(U V^T) stays well defined.
GLAMR_HD void svd3(const double K[9], double U[9], double s[3], double Vm[9]) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; ++i) A[i] = K[i];
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; ++i) { alpha += A[i * 3 + p] * A[i * 3 + p]; beta += A[i * 3 + q] * A[i * 3 + q]; gamma += A[i * 3 + p] * A[i * 3 + q]; }
        off = fmax(off, fabs(gamma) / fmax(sqrt(alpha * beta), 1e-300));
        if (fabs(gamma) < 1e-300) continue;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
        for (int i = 0; i < 3; ++i) {
          const double ap = A[i * 3 + p], aq = A[i * 3 + q];
          A[i * 3 + p] = cs * ap - sn * aq;
          A[i * 3 + q] = sn * ap + cs * aq;
          const double vp = V[i * 3 + p], vq = V[i * 3 + q];
          V[i * 3 + p] = cs * vp - sn * vq;
          V[i * 3 + q] = sn * vp + cs * vq;
        }
      }
    if (off < 1e-15) break;
  }
  for (int j = 0; j < 3; ++j) s[j] = sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
  // sort descending (torch.svd convention)
  int idx[3] = {0, 1, 2};
  for (int a = 0; a < 2; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (s[idx[b]] > s[idx[a]]) { const int t = idx[a]; idx[a] = idx[b]; idx[b] = t; }
  double ss[3];
  for (int j = 0; j < 3; ++j) {
    const int k = idx[j];
    ss[j] = s[k];
    for (int i = 0; i < 3; ++i) { Vm[i * 3 + j] = V[i * 3 + k]; U[i * 3 + j] = s[k] > 1e-300 ? A[i * 3 + k] / s[k] : 0.0; }
  }
  for (int j = 0; j < 3; ++j) s[j] = ss[j];
  if (s[1] <= 1e-12 * fmax(s[0], 1e-300)) {
    // rank <= 1 (collinear points): the second column of A is rounding noise, and normalising it gives a U column that need
    // not be orthogonal to the first, which would leak into R a.  Take the unit vector orthogonal to U[:,0] built from the
    // axis least aligned with it.
    int k = 0;
    for (int i = 1; i < 3; ++i)
      if (fabs(U[i * 3]) < fabs(U[k * 3])) k = i;
    double e[3] = {0, 0, 0};
    e[k] = 1.0;
    const double d = U[k * 3];
    double nrm = 0.0;
    for (int i = 0; i < 3; ++i) { e[i] -= d * U[i * 3]; nrm += e[i] * e[i]; }
    nrm = sqrt(nrm);
    for (int i = 0; i < 3; ++i) U[i * 3 + 1] = e[i] / nrm;
  }
  if (s[2] <= 1e-12 * fmax(s[0], 1e-300)) {   // rank deficient: complete U with the cross product of the first two columns
    U[2] = U[3] * U[7] - U[6] * U[4];
    U[5] = U[6] * U[1] - U[0] * U[7];
    U[8] = U[0] * U[4] - U[3] * U[1];
  }
}

// S1_hat = scale * R a + t closest to b (torch_transform.py:302-345).  a, b, o: [J][3] of one frame.
GLAMR_HD void procrustes_frame(int J, const float* a, const float* b, float* o) {
  double mu1[3] = {0, 0, 0}, mu2[3] = {0, 0, 0};
  for (int j = 0; j < J; ++j)
    for (int c = 0; c < 3; ++c) { mu1[c] += a[j * 3 + c]; mu2[c] += b[j * 3 + c]; }
  for (int c = 0; c < 3; ++c) { mu1[c] /= J; mu2[c] /= J; }
  double var1 = 0.0, K[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < J; ++j) {
    double x1[3], x2[3];
    for (int c = 0; c < 3; ++c) { x1[c] = a[j * 3 + c] - mu1[c]; x2[c] = b[j * 3 + c] - mu2[c]; var1 += x1[c] * x1[c]; }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) K[r * 3 + c] += x1[r] * x2[c];        // K = X1 X2^T
  }
  double U[9], s[3], V[9];
  svd3(K, U, s, V);
  // R = V Z U^T with Z = diag(1, 1, sign(det(U V^T)))
  double UVt[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) UVt[r * 3 + c] = U[r * 3] * V[c * 3] + U[r * 3 + 1] * V[c * 3 + 1] + U[r * 3 + 2] * V[c * 3 + 2];
  const double det = UVt[0] * (UVt[4] * UVt[8] - UVt[5] * UVt[7]) - UVt[1] * (UVt[3] * UVt[8] - UVt[5] * UVt[6]) + UVt[2] * (UVt[3] * UVt[7] - UVt[4] * UVt[6]);
  const double z = det > 0 ? 1.0 : (det < 0 ? -1.0 : 0.0);
  double R[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = V[r * 3] * U[c * 3] + V[r * 3 + 1] * U[c * 3 + 1] + z * V[r * 3 + 2] * U[c * 3 + 2];
  double tr = 0.0;                                                          // trace(R K)
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) tr += R[r * 3 + k] * K[k * 3 + r];
  const double scale = tr / var1;
  double t[3];
  for (int r = 0; r < 3; ++r) t[r] = mu2[r] - scale * (R[r * 3] * mu1[0] + R[r * 3 + 1] * mu1[1] + R[r * 3 + 2] * mu1[2]);
  for (int j = 0; j < J; ++j)
    for (int r = 0; r < 3; ++r)
      o[j * 3 + r] = (float)(scale * (R[r * 3] * a[j * 3] + R[r * 3 + 1] * a[j * 3 + 1] + R[r * 3 + 2] * a[j * 3 + 2]) + t[r]);
}

}  // namespace glamr
