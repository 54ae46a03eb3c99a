// TEST INFRASTRUCTURE ONLY.  g++ build of init_math.cuh (the per-row math of glamr_b200/csrc/init_kernels.cu) so that the
// rotation vectors, the gap fill and filter_pose can be checked against numpy / SciPy / the Python loop without a GPU.
#include <stdint.h>

#include <vector>

#include "../../include/glamr_b200.h"
#include "../../glamr_b200/csrc/init_math.cuh"

template <typename W, typename Y, typename O>
static void fill_all(int n, const int* frames, int T, int C, const Y* src, O* dst) {
  int before = 0;
  for (int t = 0; t < T; ++t) {
    while (before < n && frames[before] < t) ++before;
    int lo, hi;
    glamr::interp_bracket(before, n, lo, hi);
    W w_hi, w_lo;
    glamr::interp_weights<W>((W)t, (W)frames[lo], (W)frames[hi], w_hi, w_lo);
    using Cm = decltype(W() * Y());
    for (int c = 0; c < C; ++c)
      dst[(size_t)t * C + c] = (O)glamr::interp_value<Cm>((Cm)w_hi, (Cm)w_lo, (Cm)src[(size_t)hi * C + c], (Cm)src[(size_t)lo * C + c]);
  }
}

extern "C" {

int glamr_host_init_rotvec(int n, const double* mats, float* out, uint8_t* flags) {
  for (int i = 0; i < n; ++i) flags[i] = glamr::rotmat_to_rotvec_f64(mats + (size_t)i * 9, out + (size_t)i * 3) ? 0 : 1;
  return 0;
}

// kind: GLAMR_FILL_* of include/glamr_b200.h; src [n, C] samples at `frames`, dst [T, C]
int glamr_host_init_interp(int n, const int* frames, int T, int C, int kind, const void* src, void* dst) {
  if (n < 2) return 1;
  switch (kind) {
    case GLAMR_FILL_F32: fill_all<float, float, float>(n, frames, T, C, (const float*)src, (float*)dst); break;
    case GLAMR_FILL_F64: fill_all<float, double, double>(n, frames, T, C, (const double*)src, (double*)dst); break;
    case GLAMR_FILL_F32_W64: fill_all<double, float, float>(n, frames, T, C, (const float*)src, (float*)dst); break;
    default: return 1;
  }
  return 0;
}

// one person: orient [T,3] float32, vis [T] in/out, score [T,26] or NULL
int glamr_host_init_filter_pose(int T, const float* orient, float* vis, const double* score, double min_score, double min_num) {
  std::vector<unsigned char> jump(T, 0);
  const float thr = (float)(3.14159265358979323846 / 3.0);
  for (int t = 1; t < T; ++t) jump[t] = vis[t] != 0.0f && glamr::orient_jump(orient + (size_t)(t - 1) * 3, orient + (size_t)t * 3) > thr;
  glamr::filter_pose_walk(T, jump.data(), vis);
  if (score)
    for (int t = 0; t < T; ++t)
      if (vis[t] == 1.0f && glamr::keypoints_too_few(score + (size_t)t * 26, min_score, min_num)) vis[t] = 0.0f;
  return 0;
}
}
