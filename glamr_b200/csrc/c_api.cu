// Row-wise rotation algebra and the trajectory codec as stand-alone C-ABI entry points (used by the host-side
// init_data mirror and by the parity tests).  See include/glamr_b200.h.
#include "block_scan.cuh"
#include "rowops.cuh"

namespace glamr {

__global__ void rowop_fwd_kernel(int op, int n, int d0, int d1, int dout, const float* __restrict__ in0, const float* __restrict__ in1,
                                 float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[9], b[9], o[9];
  for (int k = 0; k < d0; ++k) a[k] = in0[(size_t)i * d0 + k];
  for (int k = 0; k < d1; ++k) b[k] = in1[(size_t)i * d1 + k];
  rowop_fwd(op, a, b, o);
  for (int k = 0; k < dout; ++k) out[(size_t)i * dout + k] = o[k];
}

__global__ void rowop_vjp_kernel(int op, int n, int d0, int d1, int dout, const float* __restrict__ in0, const float* __restrict__ in1,
                                 const float* __restrict__ gout, float* __restrict__ gin0, float* __restrict__ gin1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[9], b[9], g[9], ga[9], gb[9];
  for (int k = 0; k < 9; ++k) { ga[k] = 0.0f; gb[k] = 0.0f; }
  for (int k = 0; k < d0; ++k) a[k] = in0[(size_t)i * d0 + k];
  for (int k = 0; k < d1; ++k) b[k] = in1[(size_t)i * d1 + k];
  for (int k = 0; k < dout; ++k) g[k] = gout[(size_t)i * dout + k];
  rowop_vjp(op, a, b, g, ga, (gin1 != nullptr) ? gb : nullptr);
  if (gin0) for (int k = 0; k < d0; ++k) gin0[(size_t)i * d0 + k] = ga[k];
  if (gin1) for (int k = 0; k < d1; ++k) gin1[(size_t)i * d1 + k] = gb[k];
}

// traj_pred/utils/traj_utils.py:65-88 for one sequence of T frames whose frame t sits at row t * ld (local, trans, orient_q
// already offset to the sequence); head [T] and xy [2T] are its scratch.  One CTA.
__device__ __forceinline__ void traj_local2global_seq(int T, int ld, const float* __restrict__ local, int local_heading,
                                                      float* __restrict__ trans, float* __restrict__ orient_q, float* __restrict__ head,
                                                      float* __restrict__ xy, float* sm) {
  for (int t = threadIdx.x; t < T; t += kScanThreads) {
    const float* l = local + (size_t)t * ld * 11;
    head[t] = safe_atan2(l[10], l[9]);
  }
  __syncthreads();
  if (local_heading) block_scan_inplace(head, T, 1, false, sm);
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += kScanThreads) {
    const float* l = local + (size_t)t * ld * 11;
    float x = l[0], y = l[1];
    if (t > 0) {
      const float h = head[t - 1];
      const float c = cosf(h), s = sinf(h);
      const float rx = x * c - y * s, ry = x * s + y * c;
      x = rx; y = ry;
    }
    xy[2 * t] = x; xy[2 * t + 1] = y;
  }
  __syncthreads();
  block_scan_inplace(xy, T, 2, false, sm);
  block_scan_inplace(xy + 1, T, 2, false, sm);
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += kScanThreads) {
    const float* l = local + (size_t)t * ld * 11;
    float R[9], lq[4], hq[4], q1[4], q[4];
    rot6d_to_rotmat(l + 3, R);
    rotmat_to_quat(R, lq);
    const float ha[3] = {0.0f, 0.0f, head[t]};
    aa_to_quat(ha, hq);
    quat_mul(hq, lq, q1);
    const float base[4] = {0.5f, 0.5f, 0.5f, 0.5f};
    quat_mul(q1, base, q);
    float* tr = trans + (size_t)t * ld * 3;
    tr[0] = xy[2 * t]; tr[1] = xy[2 * t + 1]; tr[2] = l[2];
    float* oq = orient_q + (size_t)t * ld * 4;
    oq[0] = q[0]; oq[1] = q[1]; oq[2] = q[2]; oq[3] = q[3];
  }
}

// B sequences, time-major [T,B,*]; one CTA per sequence
__global__ void __launch_bounds__(kScanThreads) traj_local2global_kernel(int T, int B, const float* __restrict__ local, int local_heading,
                                                                        float* __restrict__ trans, float* __restrict__ orient_q,
                                                                        float* __restrict__ scratch /*[B][T][3]*/) {
  __shared__ float sm[kScanThreads / 32 + 1];
  const int b = blockIdx.x;
  float* head = scratch + (size_t)b * T * 3;
  traj_local2global_seq(T, B, local + (size_t)b * 11, local_heading, trans + (size_t)b * 3, orient_q + (size_t)b * 4, head, head + T, sm);
}

// B sequences of their own length, packed: sequence b holds rows offsets[b] .. offsets[b+1] - 1 of every array (scratch [rows][3]).
// Sequence b gets exactly the arithmetic of a T = offsets[b+1] - offsets[b] call: the scan's chunking follows its own length.
__global__ void __launch_bounds__(kScanThreads) traj_local2global_ragged_kernel(const int* __restrict__ offsets, const float* __restrict__ local,
                                                                               int local_heading, float* __restrict__ trans,
                                                                               float* __restrict__ orient_q, float* __restrict__ scratch) {
  __shared__ float sm[kScanThreads / 32 + 1];
  const int b = blockIdx.x, o = offsets[b], T = offsets[b + 1] - o;
  float* head = scratch + (size_t)o * 3;
  traj_local2global_seq(T, 1, local + (size_t)o * 11, local_heading, trans + (size_t)o * 3, orient_q + (size_t)o * 4, head, head + T, sm);
}

// Register-resident FFMA loop: what the FP32 pipe of this GPU sustains at its current clocks (bench.py quotes the LBS kernel,
// FP32-FMA bound by construction, against this measured number instead of a data-sheet peak).
__global__ void __launch_bounds__(256) fp32_probe_kernel(float* __restrict__ out, int iters, float b, float c) {
  float a[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) a[j] = (float)(threadIdx.x + j) * 1e-3f;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int j = 0; j < 16; ++j) a[j] = fmaf(a[j], b, c);
  }
  float s = 0.0f;
#pragma unroll
  for (int j = 0; j < 16; ++j) s += a[j];
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

}  // namespace glamr

using namespace glamr;

extern "C" int glamr_fp32_probe(int iters, float* scratch, size_t scratch_floats, double* flops, void* stream) {
  if (iters <= 0 || !scratch || !flops) return GLAMR_EINVAL;
  int dev = 0, sms = 0;
  GLAMR_CUDA_TRY(cudaGetDevice(&dev));
  GLAMR_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = sms * 8;                       // 8 x 256 threads = 64 warps per SM
  if (scratch_floats < (size_t)grid * 256) return GLAMR_ENOSPACE;
  fp32_probe_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(scratch, iters, 0.999f, 1e-3f);
  GLAMR_LAUNCH_CHECK();
  *flops = (double)grid * 256.0 * (double)iters * 16.0 * 2.0;
  return GLAMR_OK;
}

extern "C" int glamr_rowop_fwd(int op, int n, const float* in0, const float* in1, float* out, void* stream) {
  int d0, d1, dout;
  rowop_dims(op, d0, d1, dout);
  if (dout == 0 || n < 0 || !in0 || !out || (d1 > 0 && !in1)) return GLAMR_EINVAL;
  if (n == 0) return GLAMR_OK;
  rowop_fwd_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(op, n, d0, d1, dout, in0, in1, out);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_rowop_vjp(int op, int n, const float* in0, const float* in1, const float* gout, float* gin0, float* gin1,
                               void* stream) {
  int d0, d1, dout;
  rowop_dims(op, d0, d1, dout);
  if (dout == 0 || n < 0 || !in0 || !gout || (d1 > 0 && !in1) || op == ROP_QUAT_TO_ROTMAT) return GLAMR_EINVAL;
  if (n == 0) return GLAMR_OK;
  rowop_vjp_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(op, n, d0, d1, dout, in0, in1, gout, gin0, gin1);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_traj_local2global(int T, int B, const float* local_traj, int local_heading, float* trans, float* orient_q,
                                       float* scratch, void* stream) {
  if (T <= 0 || B <= 0 || !local_traj || !trans || !orient_q || !scratch) return GLAMR_EINVAL;
  traj_local2global_kernel<<<B, kScanThreads, 0, (cudaStream_t)stream>>>(T, B, local_traj, local_heading, trans, orient_q, scratch);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

namespace glamr {
// the codec over packed sequences of their own length (nets_kernels.cu's ragged trajectory predictor); offsets [B+1] on the device
int traj_local2global_ragged(int B, const int* offsets, const float* local_traj, float* trans, float* orient_q, float* scratch,
                             cudaStream_t stream) {
  traj_local2global_ragged_kernel<<<B, kScanThreads, 0, stream>>>(offsets, local_traj, 1, trans, orient_q, scratch);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
}  // namespace glamr
