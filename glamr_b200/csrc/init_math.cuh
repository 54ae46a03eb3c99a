// Per-row arithmetic of init_data (glamr_b200/recon.py) shared by init_kernels.cu and the host test harness.  Every
// product, sum and quotient is spelled out with round-to-nearest intrinsics on the device, so nvcc cannot contract them
// into FMAs and the values are those numpy / SciPy compute on the host (g++ builds the harness with -ffp-contract=off).
#pragma once
#include <math.h>

#include "glamr_math.cuh"

namespace glamr {

#if defined(__CUDA_ARCH__)
GLAMR_HD double rn_mul(double a, double b) { return __dmul_rn(a, b); }
GLAMR_HD double rn_add(double a, double b) { return __dadd_rn(a, b); }
GLAMR_HD double rn_sub(double a, double b) { return __dsub_rn(a, b); }
GLAMR_HD double rn_div(double a, double b) { return __ddiv_rn(a, b); }
GLAMR_HD double rn_sqrt(double a) { return __dsqrt_rn(a); }
GLAMR_HD float rn_mul(float a, float b) { return __fmul_rn(a, b); }
GLAMR_HD float rn_add(float a, float b) { return __fadd_rn(a, b); }
GLAMR_HD float rn_sub(float a, float b) { return __fsub_rn(a, b); }
GLAMR_HD float rn_div(float a, float b) { return __fdiv_rn(a, b); }
GLAMR_HD float to_f32(double a) { return __double2float_rn(a); }
#else
GLAMR_HD double rn_mul(double a, double b) { return a * b; }
GLAMR_HD double rn_add(double a, double b) { return a + b; }
GLAMR_HD double rn_sub(double a, double b) { return a - b; }
GLAMR_HD double rn_div(double a, double b) { return a / b; }
GLAMR_HD double rn_sqrt(double a) { return sqrt(a); }
GLAMR_HD float rn_mul(float a, float b) { return a * b; }
GLAMR_HD float rn_add(float a, float b) { return a + b; }
GLAMR_HD float rn_sub(float a, float b) { return a - b; }
GLAMR_HD float rn_div(float a, float b) { return a / b; }
GLAMR_HD float to_f32(double a) { return (float)a; }
#endif

// recon.rotmats_to_rotvec for one matrix (row-major R0[9]) -> float32 rotation vector, in its operation order: two
// cofactor Newton steps towards the polar factor, the largest-diagonal quaternion branch (ties to the first index, as
// argmax), normalisation, sign flip, 2 atan2 and the series below 1e-3 rad.  Returns false (out untouched) when the
// Newton steps do not reach a proper rotation (det <= 0, orthogonality residual >= 1e-9, or non-finite): the caller
// sends that row through SciPy's SVD projection as rotmats_to_rotvec does.
GLAMR_HD bool rotmat_to_rotvec_f64(const double* R0, float* out) {
  double r[9];
  for (int k = 0; k < 9; ++k) r[k] = R0[k];
  double det = 0.0;
  for (int it = 0; it < 2; ++it) {
    const double a0 = r[0], a1 = r[1], a2 = r[2], b0 = r[3], b1 = r[4], b2 = r[5], c0 = r[6], c1 = r[7], c2 = r[8];
    double cof[9];
    cof[0] = rn_sub(rn_mul(b1, c2), rn_mul(b2, c1));
    cof[1] = rn_sub(rn_mul(b2, c0), rn_mul(b0, c2));
    cof[2] = rn_sub(rn_mul(b0, c1), rn_mul(b1, c0));
    cof[3] = rn_sub(rn_mul(c1, a2), rn_mul(c2, a1));
    cof[4] = rn_sub(rn_mul(c2, a0), rn_mul(c0, a2));
    cof[5] = rn_sub(rn_mul(c0, a1), rn_mul(c1, a0));
    cof[6] = rn_sub(rn_mul(a1, b2), rn_mul(a2, b1));
    cof[7] = rn_sub(rn_mul(a2, b0), rn_mul(a0, b2));
    cof[8] = rn_sub(rn_mul(a0, b1), rn_mul(a1, b0));
    det = rn_add(rn_add(rn_mul(a0, cof[0]), rn_mul(a1, cof[1])), rn_mul(a2, cof[2]));
    for (int k = 0; k < 9; ++k) r[k] = rn_mul(0.5, rn_add(r[k], rn_div(cof[k], det)));
  }
  const double a0 = r[0], a1 = r[1], a2 = r[2], b0 = r[3], b1 = r[4], b2 = r[5], c0 = r[6], c1 = r[7], c2 = r[8];
  const double e[6] = {fabs(rn_sub(rn_add(rn_add(rn_mul(a0, a0), rn_mul(a1, a1)), rn_mul(a2, a2)), 1.0)),
                       fabs(rn_sub(rn_add(rn_add(rn_mul(b0, b0), rn_mul(b1, b1)), rn_mul(b2, b2)), 1.0)),
                       fabs(rn_sub(rn_add(rn_add(rn_mul(c0, c0), rn_mul(c1, c1)), rn_mul(c2, c2)), 1.0)),
                       fabs(rn_add(rn_add(rn_mul(a0, b0), rn_mul(a1, b1)), rn_mul(a2, b2))),
                       fabs(rn_add(rn_add(rn_mul(a0, c0), rn_mul(a1, c1)), rn_mul(a2, c2))),
                       fabs(rn_add(rn_add(rn_mul(b0, c0), rn_mul(b1, c1)), rn_mul(b2, c2)))};
  bool ok = det > 0.0;
  for (int k = 0; k < 6; ++k) ok = ok && (e[k] < 1e-9);          // a NaN anywhere fails, as the maximum does
  if (!ok) return false;
  const double tr = rn_add(rn_add(a0, b1), c2);
  const double dg[4] = {a0, b1, c2, tr};
  int choice = 0;
  for (int i = 1; i < 4; ++i)
    if (dg[i] > dg[choice]) choice = i;
  double q[4];
  if (choice < 3) {
    const int i = choice, j = (i + 1) % 3, k = (i + 2) % 3;
    q[i] = rn_add(rn_sub(1.0, tr), rn_mul(2.0, r[3 * i + i]));
    q[j] = rn_add(r[3 * j + i], r[3 * i + j]);
    q[k] = rn_add(r[3 * k + i], r[3 * i + k]);
    q[3] = rn_sub(r[3 * k + j], r[3 * j + k]);
  } else {
    q[0] = rn_sub(r[7], r[5]);
    q[1] = rn_sub(r[2], r[6]);
    q[2] = rn_sub(r[3], r[1]);
    q[3] = rn_add(1.0, tr);
  }
  const double nrm = rn_sqrt(rn_add(rn_add(rn_add(rn_mul(q[0], q[0]), rn_mul(q[1], q[1])), rn_mul(q[2], q[2])), rn_mul(q[3], q[3])));
  for (int k = 0; k < 4; ++k) q[k] = rn_div(q[k], nrm);
  if (q[3] < 0.0)
    for (int k = 0; k < 4; ++k) q[k] = -q[k];
  const double angle = rn_mul(2.0, atan2(rn_sqrt(rn_add(rn_add(rn_mul(q[0], q[0]), rn_mul(q[1], q[1])), rn_mul(q[2], q[2]))), q[3]));
  double scale;
  if (angle <= 1e-3) {
    const double a2_ = rn_mul(angle, angle);
    scale = rn_add(rn_add(2.0, rn_div(a2_, 12.0)), rn_div(rn_mul(rn_mul(7.0, a2_), a2_), 2880.0));
  } else {
    scale = rn_div(angle, sin(rn_div(angle, 2.0)));
  }
  for (int k = 0; k < 3; ++k) out[k] = to_f32(rn_mul(scale, q[k]));
  return true;
}

// scipy.interpolate.interp1d(kind='linear', fill_value='extrapolate', assume_sorted=True) at frame t, SciPy 1.18
// (_call_linear): the bracket is searchsorted(x, t) clipped to [1, n-1], so frames before the first or after the last
// sample extrapolate from the first or last two; `before` = number of samples at frames < t.
// n >= 2 (interp1d rejects fewer samples).
GLAMR_HD void interp_bracket(int before, int n, int& lo, int& hi) {
  hi = before < 1 ? 1 : (before > n - 1 ? n - 1 : before);
  lo = hi - 1;
}
// weights w_hi = (t - x_lo) / (x_hi - x_lo), w_lo = (x_hi - t) / (x_hi - x_lo) in the abscissa's dtype W
template <typename W>
GLAMR_HD void interp_weights(W t, W x_lo, W x_hi, W& w_hi, W& w_lo) {
  const W dx = rn_sub(x_hi, x_lo);
  w_hi = rn_div(rn_sub(t, x_lo), dx);
  w_lo = rn_div(rn_sub(x_hi, t), dx);
}
// w_hi * y_hi + w_lo * y_lo in the promoted dtype Y
template <typename Y>
GLAMR_HD Y interp_value(Y w_hi, Y w_lo, Y y_hi, Y y_lo) { return rn_add(rn_mul(w_hi, y_hi), rn_mul(w_lo, y_lo)); }

// recon.filter_pose's orientation jump between consecutive frames: acos(clamp(2 w^2 - 1, -1 + 1e-6, 1 - 1e-6)) of
// q_cur (x) conj(q_prev), with q from the float32 angle-axis (the row-ops' aa_to_quat / quat_mul).  NaN stays NaN.
GLAMR_HD float orient_jump(const float* aa_prev, const float* aa_cur) {
  float qp[4], qc[4], q[4];
  aa_to_quat(aa_prev, qp);
  aa_to_quat(aa_cur, qc);
  qp[1] = -qp[1]; qp[2] = -qp[2]; qp[3] = -qp[3];
  quat_mul(qc, qp, q);
  float v = rn_sub(rn_mul(2.0f, rn_mul(q[0], q[0])), 1.0f);
  const float lo = (float)(-1.0 + 1e-6), hi = (float)(1.0 - 1e-6);
  v = v < lo ? lo : (v > hi ? hi : v);
  return acosf(v);
}

// recon.filter_pose's walk over one person's frames.  jump[i] (i >= 1): frame i was visible and jumped more than pi/3
// before the walk (the reference's `ind`, which `(i + 1) not in ind` also reads); vis: the live visibility.
GLAMR_HD void filter_pose_walk(int T, const unsigned char* jump, float* vis) {
  for (int i = 1; i < T; ++i) {
    if (!jump[i] || vis[i - 1] == 0.0f) continue;
    if (i + 1 < T && vis[i + 1] != 0.0f && !jump[i + 1])
      vis[i - 1] = 0.0f;
    else
      vis[i] = 0.0f;
  }
}

// flag_make_invis_with_keypoint: a visible frame (vis == 1) with fewer than min_num of its 26 scores above min_score
// becomes invisible
GLAMR_HD bool keypoints_too_few(const double* score26, double min_score, double min_num) {
  int n = 0;
  for (int k = 0; k < 26; ++k) n += score26[k] > min_score;
  return (double)n < min_num;
}

}  // namespace glamr
