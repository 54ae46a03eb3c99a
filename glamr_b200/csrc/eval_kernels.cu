// Evaluation kernels (global_recon/utils/evaluator.py:202-327): sparse joint regression from the skinned vertices
// (evaluator.py:263,306  joint_h36m = J_regressor @ vertices) and the per-frame similarity Procrustes alignment
// (lib/utils/torch_transform.py:282-345 batch_compute_similarity_transform_torch).  sm_90a.
#include <math.h>

#include "common.cuh"
#include "eval_math.cuh"

namespace glamr {

// out[f][r][c] = sum_e w[e] * vertices[f][ci[e]][c] over the CSR row r.  One thread per (frame, row, coordinate).
__global__ void __launch_bounds__(256) sparse_regress_kernel(int n, int V, int rows, const int32_t* __restrict__ ptr, const int32_t* __restrict__ ci,
                                                             const float* __restrict__ w, const float* __restrict__ vertices,
                                                             float* __restrict__ out) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)n * rows * 3) return;
  const int c = (int)(e % 3);
  const int r = (int)((e / 3) % rows);
  const size_t f = e / ((size_t)3 * rows);
  const float* v = vertices + f * V * 3;
  float acc = 0.0f;
  for (int k = ptr[r]; k < ptr[r + 1]; ++k) acc = fmaf(w[k], v[(size_t)ci[k] * 3 + c], acc);
  out[e] = acc;
}

// One thread per frame.  S1, S2, out: [n][J][3].
__global__ void __launch_bounds__(128) procrustes_kernel(int n, int J, const float* __restrict__ S1, const float* __restrict__ S2, float* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  procrustes_frame(J, S1 + (size_t)f * J * 3, S2 + (size_t)f * J * 3, out + (size_t)f * J * 3);
}

}  // namespace glamr

using namespace glamr;

extern "C" int glamr_sparse_regress(int n, int V, int rows, const int32_t* row_ptr, const int32_t* col_idx, const float* weights,
                                    const float* vertices, float* out, void* stream) {
  if (n < 0 || V <= 0 || rows <= 0 || !row_ptr || !col_idx || !weights || !vertices || !out) return GLAMR_EINVAL;
  if (n == 0) return GLAMR_OK;
  const size_t total = (size_t)n * rows * 3;
  sparse_regress_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n, V, rows, row_ptr, col_idx, weights, vertices, out);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_procrustes_align(int n, int J, const float* S1, const float* S2, float* out, void* stream) {
  if (n < 0 || J <= 0 || !S1 || !S2 || !out) return GLAMR_EINVAL;
  if (n == 0) return GLAMR_OK;
  procrustes_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, J, S1, S2, out);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
