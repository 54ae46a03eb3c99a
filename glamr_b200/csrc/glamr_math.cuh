// Rotation / rigid-transform primitives of the GLAMR global-reconstruction path: forward value AND the
// vector-Jacobian product autograd would produce for the reference's formula (selected branch only, zero
// gradient through inactive clamps).  Every function cites the reference lines it reproduces
// (paths relative to /root/reference).  Quaternions are WXYZ, matrices row-major float[9].
//
// The header is plain C++ (no CUDA intrinsics) so that tests/host_harness can compile the very same code with
// g++ and check each primitive against torch autograd on the CPU-only build box; the product only ever runs it
// inside the sm_90a kernels of this directory.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define GLAMR_HD __host__ __device__ __forceinline__
#else
#define GLAMR_HD inline
#endif

namespace glamr {

constexpr float kEps6 = 1e-6f;

// ------------------------------------------------------------------------------------------------ small helpers
GLAMR_HD float dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
GLAMR_HD void cross3(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
// o = A(3x3) * B(3x3)
GLAMR_HD void mat3_mul(const float* A, const float* B, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}
// o = A^T * B
GLAMR_HD void mat3_tmul(const float* A, const float* B, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[i * 3 + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
// o = A * B^T
GLAMR_HD void mat3_mult(const float* A, const float* B, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o[i * 3 + j] = A[i * 3] * B[j * 3] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}
GLAMR_HD void mat3_vec(const float* A, const float* v, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = A[i * 3] * v[0] + A[i * 3 + 1] * v[1] + A[i * 3 + 2] * v[2];
}
GLAMR_HD void mat3_tvec(const float* A, const float* v, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = A[i] * v[0] + A[3 + i] * v[1] + A[6 + i] * v[2];
}

// lib/utils/torch_transform.py:63-67 (and konia_transform.py:44-47): y nudged by eps when both args are tiny.
GLAMR_HD float safe_atan2(float y, float x) {
  if (fabsf(y) < kEps6 && fabsf(x) < kEps6) y += kEps6;
  return atan2f(y, x);
}
GLAMR_HD void safe_atan2_vjp(float y, float x, float g, float& gy, float& gx) {
  if (fabsf(y) < kEps6 && fabsf(x) < kEps6) y += kEps6;
  const float inv = 1.0f / (x * x + y * y);
  gy = g * x * inv;
  gx = -g * y * inv;
}

// ------------------------------------------------------------------------------------------------ quaternions
// lib/utils/torch_transform.py:10-28 (same 8-multiplication operation order)
GLAMR_HD void quat_mul(const float* a, const float* b, float* o) {
  const float w1 = a[0], x1 = a[1], y1 = a[2], z1 = a[3];
  const float w2 = b[0], x2 = b[1], y2 = b[2], z2 = b[3];
  const float ww = (z1 + x1) * (x2 + y2);
  const float yy = (w1 - y1) * (w2 + z2);
  const float zz = (w1 + y1) * (w2 - z2);
  const float xx = ww + yy + zz;
  const float qq = 0.5f * (xx + (z1 - x1) * (x2 - y2));
  o[0] = qq - ww + (z1 - y1) * (y2 - z2);
  o[1] = qq - xx + (x1 + w1) * (x2 + w2);
  o[2] = qq - yy + (w1 - x1) * (y2 + z2);
  o[3] = qq - zz + (z1 + y1) * (w2 - x2);
}
GLAMR_HD void quat_mul_plain(const float* a, const float* b, float* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}
// out = a (x) b is bilinear: g_a = g (x) conj(b), g_b = conj(a) (x) g
GLAMR_HD void quat_mul_vjp(const float* a, const float* b, const float* g, float* ga, float* gb) {
  const float bc[4] = {b[0], -b[1], -b[2], -b[3]};
  const float ac[4] = {a[0], -a[1], -a[2], -a[3]};
  if (ga) quat_mul_plain(g, bc, ga);
  if (gb) quat_mul_plain(ac, g, gb);
}

// ------------------------------------------------------------------------------------------------ axis-angle -> R
// lib/utils/konia_transform.py:234-313: theta = sqrt(clamp_min(theta^2, 1e-6)), w = r / (theta + 1e-6);
// Taylor matrix when theta^2 <= 1e-6; mask blend => gradient of the selected branch only.
GLAMR_HD void aa_to_rotmat(const float* r, float* R) {
  const float th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  if (th2 > kEps6) {
    const float th = sqrtf(th2);
    const float inv = 1.0f / (th + kEps6);
    const float wx = r[0] * inv, wy = r[1] * inv, wz = r[2] * inv;
    const float c = cosf(th), s = sinf(th), k = 1.0f - c;
    R[0] = c + wx * wx * k;
    R[1] = wx * wy * k - wz * s;
    R[2] = wy * s + wx * wz * k;
    R[3] = wz * s + wx * wy * k;
    R[4] = c + wy * wy * k;
    R[5] = -wx * s + wy * wz * k;
    R[6] = -wy * s + wx * wz * k;
    R[7] = wx * s + wy * wz * k;
    R[8] = c + wz * wz * k;
  } else {
    R[0] = 1.0f; R[1] = -r[2]; R[2] = r[1];
    R[3] = r[2]; R[4] = 1.0f;  R[5] = -r[0];
    R[6] = -r[1]; R[7] = r[0]; R[8] = 1.0f;
  }
}
GLAMR_HD void aa_to_rotmat_vjp(const float* r, const float* gR, float* gr) {
  const float th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  if (th2 > kEps6) {
    const float th = sqrtf(th2);
    const float inv = 1.0f / (th + kEps6);
    const float wx = r[0] * inv, wy = r[1] * inv, wz = r[2] * inv;
    const float c = cosf(th), s = sinf(th), k = 1.0f - c;
    const float s01 = gR[1] + gR[3], s02 = gR[2] + gR[6], s12 = gR[5] + gR[7];
    const float gk = gR[0] * wx * wx + gR[4] * wy * wy + gR[8] * wz * wz + s01 * wx * wy + s02 * wx * wz + s12 * wy * wz;
    const float gs = (gR[3] - gR[1]) * wz + (gR[2] - gR[6]) * wy + (gR[7] - gR[5]) * wx;
    const float gc = gR[0] + gR[4] + gR[8] - gk;
    const float gwx = 2.0f * gR[0] * wx * k + s01 * wy * k + s02 * wz * k + (gR[7] - gR[5]) * s;
    const float gwy = 2.0f * gR[4] * wy * k + s01 * wx * k + s12 * wz * k + (gR[2] - gR[6]) * s;
    const float gwz = 2.0f * gR[8] * wz * k + s02 * wx * k + s12 * wy * k + (gR[3] - gR[1]) * s;
    float gth = -s * gc + c * gs;
    gth -= (gwx * r[0] + gwy * r[1] + gwz * r[2]) * inv * inv;
    const float gth2 = gth / (2.0f * th);
    gr[0] = gwx * inv + 2.0f * r[0] * gth2;
    gr[1] = gwy * inv + 2.0f * r[1] * gth2;
    gr[2] = gwz * inv + 2.0f * r[2] * gth2;
  } else {
    gr[0] = gR[7] - gR[5];
    gr[1] = gR[2] - gR[6];
    gr[2] = gR[3] - gR[1];
  }
}

// smplx batch_rodrigues, in-tree statement HybrIK/hybrik/models/layers/smpl/lbs.py:446-477:
// angle = |r + 1e-8| (eps per component), no small-angle branch.
GLAMR_HD void rodrigues_smplx(const float* r, float* R) {
  const float e0 = r[0] + 1e-8f, e1 = r[1] + 1e-8f, e2 = r[2] + 1e-8f;
  const float angle = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
  const float inv = 1.0f / angle;
  const float x = r[0] * inv, y = r[1] * inv, z = r[2] * inv;
  const float s = sinf(angle), m = 1.0f - cosf(angle);
  R[0] = 1.0f + m * (-z * z - y * y);
  R[1] = -s * z + m * (x * y);
  R[2] = s * y + m * (x * z);
  R[3] = s * z + m * (x * y);
  R[4] = 1.0f + m * (-z * z - x * x);
  R[5] = -s * x + m * (y * z);
  R[6] = -s * y + m * (x * z);
  R[7] = s * x + m * (y * z);
  R[8] = 1.0f + m * (-y * y - x * x);
}
GLAMR_HD void rodrigues_smplx_vjp(const float* r, const float* gR, float* gr) {
  const float e0 = r[0] + 1e-8f, e1 = r[1] + 1e-8f, e2 = r[2] + 1e-8f;
  const float angle = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
  const float inv = 1.0f / angle;
  const float x = r[0] * inv, y = r[1] * inv, z = r[2] * inv;
  const float s = sinf(angle), c = cosf(angle), m = 1.0f - c;
  const float s01 = gR[1] + gR[3], s02 = gR[2] + gR[6], s12 = gR[5] + gR[7];
  const float gs = (gR[3] - gR[1]) * z + (gR[2] - gR[6]) * y + (gR[7] - gR[5]) * x;
  const float gm = gR[0] * (-z * z - y * y) + gR[4] * (-z * z - x * x) + gR[8] * (-y * y - x * x) + s01 * x * y + s02 * x * z + s12 * y * z;
  const float gx = s * (gR[7] - gR[5]) + m * (-2.0f * x * (gR[4] + gR[8]) + s01 * y + s02 * z);
  const float gy = s * (gR[2] - gR[6]) + m * (-2.0f * y * (gR[0] + gR[8]) + s01 * x + s12 * z);
  const float gz = s * (gR[3] - gR[1]) + m * (-2.0f * z * (gR[0] + gR[4]) + s02 * x + s12 * y);
  float gangle = c * gs + s * gm;
  gangle -= (gx * r[0] + gy * r[1] + gz * r[2]) * inv * inv;
  gr[0] = gx * inv + gangle * e0 * inv;
  gr[1] = gy * inv + gangle * e1 * inv;
  gr[2] = gz * inv + gangle * e2 * inv;
}

// ------------------------------------------------------------------------------------------------ 6d <-> R
// lib/utils/torch_transform.py:214-227: Gram-Schmidt with normalize(x) = x / max(|x|, 1e-9); R columns (b1,b2,b1xb2)
GLAMR_HD void rot6d_to_rotmat(const float* d, float* R) {
  const float n1 = fmaxf(sqrtf(dot3(d, d)), 1e-9f);
  const float b1[3] = {d[0] / n1, d[1] / n1, d[2] / n1};
  const float dp = dot3(b1, d + 3);
  const float u[3] = {d[3] - dp * b1[0], d[4] - dp * b1[1], d[5] - dp * b1[2]};
  const float n2 = fmaxf(sqrtf(dot3(u, u)), 1e-9f);
  const float b2[3] = {u[0] / n2, u[1] / n2, u[2] / n2};
  float b3[3];
  cross3(b1, b2, b3);
#pragma unroll
  for (int i = 0; i < 3; ++i) { R[i * 3] = b1[i]; R[i * 3 + 1] = b2[i]; R[i * 3 + 2] = b3[i]; }
}
GLAMR_HD void rot6d_to_rotmat_vjp(const float* d, const float* gR, float* gd) {
  const float n1r = sqrtf(dot3(d, d));
  const float n1 = fmaxf(n1r, 1e-9f);
  const float b1[3] = {d[0] / n1, d[1] / n1, d[2] / n1};
  const float dp = dot3(b1, d + 3);
  const float u[3] = {d[3] - dp * b1[0], d[4] - dp * b1[1], d[5] - dp * b1[2]};
  const float n2r = sqrtf(dot3(u, u));
  const float n2 = fmaxf(n2r, 1e-9f);
  const float b2[3] = {u[0] / n2, u[1] / n2, u[2] / n2};
  float gb1[3] = {gR[0], gR[3], gR[6]}, gb2[3] = {gR[1], gR[4], gR[7]};
  const float gb3[3] = {gR[2], gR[5], gR[8]};
  float t[3];
  cross3(b2, gb3, t);   // d(b1 x b2)/db1
  gb1[0] += t[0]; gb1[1] += t[1]; gb1[2] += t[2];
  cross3(gb3, b1, t);   // d(b1 x b2)/db2
  gb2[0] += t[0]; gb2[1] += t[1]; gb2[2] += t[2];
  float gu[3];
  {
    const float proj = (n2r >= 1e-9f) ? dot3(b2, gb2) : 0.0f;
#pragma unroll
    for (int i = 0; i < 3; ++i) gu[i] = (gb2[i] - b2[i] * proj) / n2;
  }
  const float gdp = -dot3(gu, b1);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    gd[3 + i] = gu[i] + gdp * b1[i];
    gb1[i] += -dp * gu[i] + gdp * d[3 + i];
  }
  {
    const float proj = (n1r >= 1e-9f) ? dot3(b1, gb1) : 0.0f;
#pragma unroll
    for (int i = 0; i < 3; ++i) gd[i] = (gb1[i] - b1[i] * proj) / n1;
  }
}
// lib/utils/torch_transform.py:214-217: first two COLUMNS
GLAMR_HD void rotmat_to_rot6d(const float* R, float* d) {
  d[0] = R[0]; d[1] = R[3]; d[2] = R[6]; d[3] = R[1]; d[4] = R[4]; d[5] = R[7];
}
GLAMR_HD void rotmat_to_rot6d_vjp(const float* gd, float* gR) {
  gR[0] = gd[0]; gR[3] = gd[1]; gR[6] = gd[2]; gR[1] = gd[3]; gR[4] = gd[4]; gR[7] = gd[5];
  gR[2] = 0.0f; gR[5] = 0.0f; gR[8] = 0.0f;
}

// ------------------------------------------------------------------------------------------------ R -> quaternion
// lib/utils/konia_transform.py:349-443.  Branch: 0 trace>0, 1 m00 largest, 2 m11>m22, 3 otherwise.
GLAMR_HD int rotmat_quat_branch(const float* m) {
  const float tr = m[0] + m[4] + m[8];
  if (tr > 0.0f) return 0;
  if (m[0] > m[4] && m[0] > m[8]) return 1;
  return (m[4] > m[8]) ? 2 : 3;
}
GLAMR_HD void rotmat_to_quat(const float* m, float* q) {
  const int br = rotmat_quat_branch(m);
  if (br == 0) {
    const float sq = sqrtf(fmaxf(m[0] + m[4] + m[8] + 1.0f, kEps6)) * 2.0f;
    q[0] = 0.25f * sq; q[1] = (m[7] - m[5]) / sq; q[2] = (m[2] - m[6]) / sq; q[3] = (m[3] - m[1]) / sq;
  } else if (br == 1) {
    const float sq = sqrtf(fmaxf(1.0f + m[0] - m[4] - m[8], kEps6)) * 2.0f;
    q[0] = (m[7] - m[5]) / sq; q[1] = 0.25f * sq; q[2] = (m[1] + m[3]) / sq; q[3] = (m[2] + m[6]) / sq;
  } else if (br == 2) {
    const float sq = sqrtf(fmaxf(1.0f + m[4] - m[0] - m[8], kEps6)) * 2.0f;
    q[0] = (m[2] - m[6]) / sq; q[1] = (m[1] + m[3]) / sq; q[2] = 0.25f * sq; q[3] = (m[5] + m[7]) / sq;
  } else {
    const float sq = sqrtf(fmaxf(1.0f + m[8] - m[0] - m[4], kEps6)) * 2.0f;
    q[0] = (m[3] - m[1]) / sq; q[1] = (m[2] + m[6]) / sq; q[2] = (m[5] + m[7]) / sq; q[3] = 0.25f * sq;
  }
}
// One branch of the VJP with compile-time indices (keeps everything in registers): D = 1 + sd0 m[d0] + sd1 m[d1] + sd2 m[d2]
// (trace branch: all +), slot IS holds 0.25*sq, slots IA/IB/IC hold (m[P] + S m[N]) / sq.
template <int IS, int IA, int PA, int NA, int SA, int IB, int PB, int NB, int SB, int IC, int PC, int NC, int SC, int D0, int D1, int D2, int S1, int S2>
GLAMR_HD void rotmat_to_quat_vjp_branch(const float* m, const float* gq, float* gm) {
  const float D = 1.0f + m[D0] + (float)S1 * m[D1] + (float)S2 * m[D2];
  const float Dc = fmaxf(D, kEps6);
  const float rs = sqrtf(Dc);
  const float sq = rs * 2.0f, isq = 1.0f / sq;
  const float na = m[PA] + (float)SA * m[NA], nb = m[PB] + (float)SB * m[NB], nc = m[PC] + (float)SC * m[NC];
  const float gsq = 0.25f * gq[IS] - (gq[IA] * na + gq[IB] * nb + gq[IC] * nc) * isq * isq;
  gm[PA] += gq[IA] * isq; gm[NA] += (float)SA * gq[IA] * isq;
  gm[PB] += gq[IB] * isq; gm[NB] += (float)SB * gq[IB] * isq;
  gm[PC] += gq[IC] * isq; gm[NC] += (float)SC * gq[IC] * isq;
  const float gD = (D >= kEps6) ? gsq / rs : 0.0f;   // d(2 sqrt D)/dD = 1/sqrt(D); clamp_min passes the gradient when D >= eps
  gm[D0] += gD; gm[D1] += (float)S1 * gD; gm[D2] += (float)S2 * gD;
}
GLAMR_HD void rotmat_to_quat_vjp(const float* m, const float* gq, float* gm) {
#pragma unroll
  for (int i = 0; i < 9; ++i) gm[i] = 0.0f;
  const int br = rotmat_quat_branch(m);
  if (br == 0) rotmat_to_quat_vjp_branch<0, 1, 7, 5, -1, 2, 2, 6, -1, 3, 3, 1, -1, 0, 4, 8, 1, 1>(m, gq, gm);
  else if (br == 1) rotmat_to_quat_vjp_branch<1, 0, 7, 5, -1, 2, 1, 3, 1, 3, 2, 6, 1, 0, 4, 8, -1, -1>(m, gq, gm);
  else if (br == 2) rotmat_to_quat_vjp_branch<2, 0, 2, 6, -1, 1, 1, 3, 1, 3, 5, 7, 1, 4, 0, 8, -1, -1>(m, gq, gm);
  else rotmat_to_quat_vjp_branch<3, 0, 3, 1, -1, 1, 2, 6, 1, 2, 5, 7, 1, 8, 0, 4, -1, -1>(m, gq, gm);
}

// ------------------------------------------------------------------------------------------------ q <-> axis-angle
// lib/utils/konia_transform.py:560-630
GLAMR_HD void quat_to_aa(const float* q, float* aa) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  const float s2 = x * x + y * y + z * z;
  const float s = sqrtf(fmaxf(s2, kEps6));
  const float tt = 2.0f * ((w < 0.0f) ? safe_atan2(-s, -w) : safe_atan2(s, w));
  const float k = (s2 > 0.0f) ? tt / s : 2.0f;
  aa[0] = x * k; aa[1] = y * k; aa[2] = z * k;
}
GLAMR_HD void quat_to_aa_vjp(const float* q, const float* g, float* gq) {
  const float w = q[0], x = q[1], y = q[2], z = q[3];
  const float s2 = x * x + y * y + z * z;
  const float s = sqrtf(fmaxf(s2, kEps6));
  const bool neg = w < 0.0f;
  const float tt = 2.0f * (neg ? safe_atan2(-s, -w) : safe_atan2(s, w));
  const float k = (s2 > 0.0f) ? tt / s : 2.0f;
  gq[1] = k * g[0]; gq[2] = k * g[1]; gq[3] = k * g[2];
  gq[0] = 0.0f;
  if (s2 > 0.0f) {
    const float gk = g[0] * x + g[1] * y + g[2] * z;
    const float gtt = gk / s;
    float gs = -gk * tt / (s * s);
    float gY, gX;
    safe_atan2_vjp(neg ? -s : s, neg ? -w : w, 2.0f * gtt, gY, gX);
    gs += neg ? -gY : gY;
    gq[0] = neg ? -gX : gX;
    const float gs2 = (s2 >= kEps6) ? gs / (2.0f * s) : 0.0f;
    gq[1] += 2.0f * x * gs2; gq[2] += 2.0f * y * gs2; gq[3] += 2.0f * z * gs2;
  }
}
// lib/utils/konia_transform.py:753-822
GLAMR_HD void aa_to_quat(const float* a, float* q) {
  const float th2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
  const float th = sqrtf(fmaxf(th2, kEps6));
  const float half = 0.5f * th;
  const bool pos = th2 > 0.0f;
  const float k = pos ? sinf(half) / th : 0.5f;
  q[0] = pos ? cosf(half) : 1.0f;
  q[1] = a[0] * k; q[2] = a[1] * k; q[3] = a[2] * k;
}
GLAMR_HD void aa_to_quat_vjp(const float* a, const float* gq, float* ga) {
  const float th2 = a[0] * a[0] + a[1] * a[1] + a[2] * a[2];
  const float th = sqrtf(fmaxf(th2, kEps6));
  const float half = 0.5f * th;
  const bool pos = th2 > 0.0f;
  const float sh = sinf(half), ch = cosf(half);
  const float k = pos ? sh / th : 0.5f;
  ga[0] = k * gq[1]; ga[1] = k * gq[2]; ga[2] = k * gq[3];
  if (pos) {
    const float gk = gq[1] * a[0] + gq[2] * a[1] + gq[3] * a[2];
    const float gth = gk * (0.5f * ch / th - sh / (th * th)) - 0.5f * sh * gq[0];
    const float gth2 = (th2 >= kEps6) ? gth / (2.0f * th) : 0.0f;
    ga[0] += 2.0f * a[0] * gth2; ga[1] += 2.0f * a[1] * gth2; ga[2] += 2.0f * a[2] * gth2;
  }
}
// lib/utils/konia_transform.py:477-557 (normalises with eps 1e-12 first)
GLAMR_HD void quat_to_rotmat(const float* qi, float* R) {
  const float n = fmaxf(sqrtf(qi[0] * qi[0] + qi[1] * qi[1] + qi[2] * qi[2] + qi[3] * qi[3]), 1e-12f);
  const float w = qi[0] / n, x = qi[1] / n, y = qi[2] / n, z = qi[3] / n;
  const float tx = 2.0f * x, ty = 2.0f * y, tz = 2.0f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1.0f - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1.0f - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0f - (txx + tyy);
}

// rotation_matrix_to_angle_axis = quat_to_aa o rotmat_to_quat (konia_transform.py:316-339)
GLAMR_HD void rotmat_to_aa(const float* R, float* aa) {
  float q[4];
  rotmat_to_quat(R, q);
  quat_to_aa(q, aa);
}
GLAMR_HD void rotmat_to_aa_vjp(const float* R, const float* gaa, float* gR) {
  float q[4], gq[4];
  rotmat_to_quat(R, q);
  quat_to_aa_vjp(q, gaa, gq);
  rotmat_to_quat_vjp(R, gq, gR);
}

// ------------------------------------------------------------------------------------------------ projection
// lib/utils/geometry.py:23-25  uv = (K X)_xy / ((K X)_z + 1e-8)
GLAMR_HD void project(const float* K, const float* X, float* uv) {
  float p[3];
  mat3_vec(K, X, p);
  const float iz = 1.0f / (p[2] + 1e-8f);
  uv[0] = p[0] * iz; uv[1] = p[1] * iz;
}
GLAMR_HD void project_vjp(const float* K, const float* X, const float* guv, float* gX) {
  float p[3];
  mat3_vec(K, X, p);
  const float iz = 1.0f / (p[2] + 1e-8f);
  const float gp[3] = {guv[0] * iz, guv[1] * iz, -(guv[0] * p[0] + guv[1] * p[1]) * iz * iz};
  mat3_tvec(K, gp, gX);
}
// global_recon/models/loss_func.py:6-12 Geman-McClure, sigma = 100
GLAMR_HD float gmof(float d) { const float d2 = d * d; return (10000.0f * d2) / (10000.0f + d2); }
GLAMR_HD float gmof_grad(float d) { const float t = 10000.0f + d * d; return 2.0f * 1.0e8f * d / (t * t); }

}  // namespace glamr
