// Learned-prior inference on sm_90a: the motion infiller (CVAE, transformer encoder/decoder over 50-frame windows,
// motion_infiller/models/motion_infiller_vae.py:22-123,252-421,564-632) and the trajectory predictor (CVAE, MLP +
// 2-layer bidirectional LSTM, traj_pred/models/traj_pred_vae.py:20-92,202-333; lib/models/{mlp,rnn,pos_encoding}.py).
// Every Linear (QKV / out-proj / FFN / MLP / LSTM input projections) runs on the tensor cores: wgmma.mma_async tf32
// with a 3xTF32 split and the accumulator in registers (gemm_tf32x3_wgmma_kernel); LayerNorm, softmax attention (S <= 64,
// shared memory) and the LSTM recurrence (W_hh resident in registers + shared memory for the whole sequence) are FP32
// SIMT kernels.  Outputs match the reference's fp32 networks to <= 1e-4 (tests/golden/nets.npz).
// Weights are addressed by their reference state-dict names so Lightning checkpoints map 1:1.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "block_scan.cuh"
#include "glamr_math.cuh"

namespace glamr {

// ------------------------------------------------------------------------------------------------ SGEMM  Y = act(X W^T + b)
// X [M,K] (row stride ldx), W [N,K], Y [M,N] (row stride ldy).  64x64x16 tiles, 256 threads, 4x4 micro-tiles.
constexpr int GT = 64, GK = 16;
template <int ACT>   // 0 none, 1 relu
__global__ void __launch_bounds__(256) gemm_bias_act_kernel(int M, int N, int K, const float* __restrict__ X, int ldx,
                                                            const float* __restrict__ W, const float* __restrict__ bias,
                                                            const float* __restrict__ bias2, float* __restrict__ Y, int ldy) {
  __shared__ float Xs[GK][GT + 4];
  __shared__ float Ws[GK][GT + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
  const int tx = tid & 15, ty = tid >> 4;       // 16 x 16 threads, each 4 (m) x 4 (n)
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  const int lr = tid >> 2, lk = (tid & 3) * 4;  // loader: row 0..63, k offset 0,4,8,12
  for (int k0 = 0; k0 < K; k0 += GK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = k0 + lk + q;
      const int m = m0 + lr, n = n0 + lr;
      Xs[lk + q][lr] = (m < M && k < K) ? X[(size_t)m * ldx + k] : 0.0f;
      Ws[lk + q][lr] = (n < N && k < K) ? W[(size_t)n * K + k] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = Xs[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Ws[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] + (bias ? bias[n] : 0.0f) + (bias2 ? bias2[n] : 0.0f);
      if (ACT == 1) v = fmaxf(v, 0.0f);
      Y[(size_t)m * ldy + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ wgmma GEMM (3xTF32)
// Y = act(X W^T + b) on the Hopper tensor cores: wgmma.mma_async tf32 with the accumulator in registers.
// FP32 accuracy is kept with the 3xTF32 split  x = hi + lo (hi = tf32(x), lo = tf32(x - hi)):
//   X W^T ~= Xhi Whi^T + Xlo Whi^T + Xhi Wlo^T     (error ~2^-21 relative per product; partial sums per K step of 32 are
//   folded in FP32, see the main loop)
// CTA = 256 threads = two warpgroups, tile 128 (M) x 128 (N), K step 32; warpgroup g computes rows 64 g .. 64 g + 63 (m64n128k8).
// Both operands are K-major (X [M,K] and W [N,K] row-major), written by the CTA into shared memory in the canonical no-swizzle
// layout (8-row x 16-byte core matrices: element (r,k) at ((k/4)*128 + r)*16 + (k%4)*4 bytes => LBO = 2048 B between K groups,
// SBO = 128 B between 8-row groups) and made visible to the async proxy with fence.proxy.async; the epilogue adds the bias to the
// accumulator fragment, applies the activation and stores.
constexpr int TCM = 128, TCN = 128, TCK = 32;
constexpr int kTcATileFloats = TCM * TCK;                       // 4096 floats = 16 KB (hi or lo of the X tile)
constexpr int kTcBTileFloats = TCN * TCK;                       // 4096 floats = 16 KB (hi or lo of the W tile)

__device__ __forceinline__ float4 split_tf32_4(const float4 v, float4& lo) {
  float4 hi;
  split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y); split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
  return hi;
}

constexpr int kTcThreads = 256;
constexpr int kTcStages = 2;
constexpr int kTcStageFloats = 2 * kTcATileFloats + 2 * kTcBTileFloats;                  // Xhi | Xlo | Whi | Wlo
constexpr int kTcXVec = (TCM * TCK / 4) / kTcThreads;                                    // 16-byte loads per thread and K step
constexpr int kTcWVec = (TCN * TCK / 4) / kTcThreads;
constexpr size_t kTcSmemBytes = (size_t)kTcStages * kTcStageFloats * sizeof(float);

// one K step (32 columns) of the 128-row X tile and the 128-row W tile, in flight in registers
struct TcRegs {
  float4 x[kTcXVec], w[kTcWVec];
};
template <bool VEC>
__device__ __forceinline__ float4 tc_load_row4(const float* __restrict__ P, int ld, int row, int nrows, int k, int K) {
  if (VEC) {
    if (row < nrows && k < K) return __ldg(reinterpret_cast<const float4*>(P + (size_t)row * ld + k));
    return make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float a[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) a[q] = (row < nrows && k + q < K) ? P[(size_t)row * ld + k + q] : 0.0f;
  return make_float4(a[0], a[1], a[2], a[3]);
}
template <bool VEC>
__device__ __forceinline__ void tc_load_tiles(TcRegs& r, int tid, int M, int N, int K, const float* __restrict__ X, int ldx,
                                              const float* __restrict__ W, int m0, int n0, int k0) {
#pragma unroll
  for (int i = 0; i < kTcXVec; ++i) {
    const int idx = tid + i * kTcThreads;
    r.x[i] = tc_load_row4<VEC>(X, ldx, m0 + (idx & (TCM - 1)), M, k0 + (idx / TCM) * 4, K);      // row, 16-byte K group (0..7)
  }
#pragma unroll
  for (int i = 0; i < kTcWVec; ++i) {
    const int idx = tid + i * kTcThreads;
    r.w[i] = tc_load_row4<VEC>(W, K, n0 + (idx & (TCN - 1)), N, k0 + (idx / TCN) * 4, K);
  }
}
// split into tf32 hi / lo and store as K-major 8x16-byte core matrices (the layout wgmma_desc_kmajor_noswizzle describes)
__device__ __forceinline__ void tc_store_tiles(float* st, int tid, const TcRegs& r) {
  float* Ahi = st;
  float* Alo = st + kTcATileFloats;
  float* Bhi = st + 2 * kTcATileFloats;
  float* Blo = Bhi + kTcBTileFloats;
#pragma unroll
  for (int i = 0; i < kTcXVec; ++i) {
    const int idx = tid + i * kTcThreads;
    const int off = ((idx / TCM) * TCM + (idx & (TCM - 1))) * 4;
    float4 lo;
    const float4 hi = split_tf32_4(r.x[i], lo);
    *reinterpret_cast<float4*>(Ahi + off) = hi;
    *reinterpret_cast<float4*>(Alo + off) = lo;
  }
#pragma unroll
  for (int i = 0; i < kTcWVec; ++i) {
    const int idx = tid + i * kTcThreads;
    const int off = ((idx / TCN) * TCN + (idx & (TCN - 1))) * 4;
    float4 lo;
    const float4 hi = split_tf32_4(r.w[i], lo);
    *reinterpret_cast<float4*>(Bhi + off) = hi;
    *reinterpret_cast<float4*>(Blo + off) = lo;
  }
}

// 256 threads; two shared-memory stages: while the tensor core works on stage s (12 wgmma per K step and warpgroup, one commit
// group) all threads split and store K step it+1 into stage s^1 and already have the global loads of step it+2 in flight in
// registers, so the L2 latency never sits on the critical path of these small GEMMs.
template <int ACT, bool VEC>
__global__ void __launch_bounds__(kTcThreads) gemm_tf32x3_wgmma_kernel(int M, int N, int K, const float* __restrict__ X, int ldx,
                                                                       const float* __restrict__ W, const float* __restrict__ bias,
                                                                       const float* __restrict__ bias2, float* __restrict__ Y, int ldy) {
  extern __shared__ __align__(128) unsigned char tc_smem[];
  float* stage0 = reinterpret_cast<float*>(tc_smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = warp >> 2;                                                                // warpgroup: rows 64 g .. 64 g + 63
  const int m0 = blockIdx.y * TCM, n0 = blockIdx.x * TCN;

  const int nk = (K + TCK - 1) / TCK;
  TcRegs regs;
  tc_load_tiles<VEC>(regs, tid, M, N, K, X, ldx, W, m0, n0, 0);
  tc_store_tiles(stage0, tid, regs);
  if (nk > 1) tc_load_tiles<VEC>(regs, tid, M, N, K, X, ldx, W, m0, n0, TCK);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy smem writes -> visible to the tensor core
  __syncthreads();

  // Each K step accumulates into `part` on the tensor core, and `part` is folded into `acc` with an FP32 add.  The tensor core's
  // accumulation does not round to nearest, so a 3xTF32 sum kept in its accumulator over all of K drifts with K (a Linear missed a
  // float64 product by 4.6x, the infiller's output a float64 oracle by ~20x, what the FP32 kernels miss by); 32-wide partial sums
  // bound that drift to one K step.
  float acc[TCN / 2], part[TCN / 2];
#pragma unroll
  for (int i = 0; i < TCN / 2; ++i) acc[i] = 0.0f;
  for (int it = 0; it < nk; ++it) {
    const int s = it & 1;
    float* st = stage0 + s * kTcStageFloats;
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < TCK / 8; ++k8) {                               // one tf32 wgmma consumes K = 8 (two 16-byte K groups)
      const size_t koa = (size_t)k8 * 2 * TCM * 4 + g * 64 * 4, kob = (size_t)k8 * 2 * TCN * 4;   // floats
      const uint64_t dah = wgmma_desc_kmajor_noswizzle(st + koa, TCM), dal = wgmma_desc_kmajor_noswizzle(st + kTcATileFloats + koa, TCM);
      const uint64_t dbh = wgmma_desc_kmajor_noswizzle(st + 2 * kTcATileFloats + kob, TCN);
      const uint64_t dbl = wgmma_desc_kmajor_noswizzle(st + 2 * kTcATileFloats + kTcBTileFloats + kob, TCN);
      wgmma_m64n128k8_tf32(part, dal, dbh, k8 > 0 ? 1u : 0u);            // the small cross terms first
      wgmma_m64n128k8_tf32(part, dah, dbl, 1u);
      wgmma_m64n128k8_tf32(part, dah, dbh, 1u);
    }
    wgmma_commit();
    if (it + 1 < nk) {
      // stage s^1 was last read by step it-1, which every warpgroup retired before the barrier that ended that step: refill it
      // while step `it` computes
      tc_store_tiles(stage0 + (s ^ 1) * kTcStageFloats, tid, regs);
      if (it + 2 < nk) tc_load_tiles<VEC>(regs, tid, M, N, K, X, ldx, W, m0, n0, (it + 2) * TCK);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    wgmma_wait<0>();
    wgmma_fence_acc(part);
#pragma unroll
    for (int i = 0; i < TCN / 2; ++i) acc[i] += part[i];
    if (it + 1 < nk) __syncthreads();
  }

  // ---- epilogue: acc[4 i + 2 h + e] = Y[m0 + 64 g + 16 (warp % 4) + lane / 4 + 8 h][n0 + 8 i + 2 (lane % 4) + e]
  const bool yvec = (ldy & 1) == 0 && (reinterpret_cast<uintptr_t>(Y) & 7) == 0;
#pragma unroll
  for (int i = 0; i < TCN / 8; ++i) {
    const int n = n0 + 8 * i + 2 * (lane & 3);
    if (n >= N) continue;
    const bool pair = n + 1 < N;
    float b0 = 0.0f, b1 = 0.0f;
    if (bias) { b0 += __ldg(bias + n); if (pair) b1 += __ldg(bias + n + 1); }
    if (bias2) { b0 += __ldg(bias2 + n); if (pair) b1 += __ldg(bias2 + n + 1); }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (m >= M) continue;
      float o0 = acc[4 * i + 2 * h] + b0, o1 = acc[4 * i + 2 * h + 1] + b1;
      if (ACT == 1) { o0 = fmaxf(o0, 0.0f); o1 = fmaxf(o1, 0.0f); }
      float* y = Y + (size_t)m * ldy + n;
      if (pair && yvec) {
        *reinterpret_cast<float2*>(y) = make_float2(o0, o1);
      } else {
        y[0] = o0;
        if (pair) y[1] = o1;
      }
    }
  }
}

static int gemm_tc_launch(cudaStream_t s, int M, int N, int K, const float* X, int ldx, const float* W, const float* b, const float* b2,
                          float* Y, int ldy, int act) {
  static bool attr = false;
  if (!attr) {
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(gemm_tf32x3_wgmma_kernel<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(gemm_tf32x3_wgmma_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(gemm_tf32x3_wgmma_kernel<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(gemm_tf32x3_wgmma_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes));
    attr = true;
  }
  const dim3 grid((N + TCN - 1) / TCN, (M + TCM - 1) / TCM);
  const bool vec = (K % 4 == 0) && (ldx % 4 == 0) && (((uintptr_t)X | (uintptr_t)W) % 16 == 0);
  auto go = [&](auto kernel) { kernel<<<grid, kTcThreads, kTcSmemBytes, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy); };
  if (vec) {
    if (act == 1) go(gemm_tf32x3_wgmma_kernel<1, true>); else go(gemm_tf32x3_wgmma_kernel<0, true>);
  } else {
    if (act == 1) go(gemm_tf32x3_wgmma_kernel<1, false>); else go(gemm_tf32x3_wgmma_kernel<0, false>);
  }
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}


// ------------------------------------------------------------------------------------------------ skinny GEMM (M <= 256)
// The prior runs at batch 1-4: its linear layers are [50 B x K] x [K x N] with K, N <= 512 -- a few MFLOP each, ~450 of them
// in dependent order per sequence, so the figure of merit is the LATENCY of one launch, not its throughput.  One warp owns an
// 8 x 4 output tile and splits K across its lanes: every lane issues all its 16-byte loads of the 8 X rows and 4 W rows at once
// (no shared memory, no block barrier, one global round trip), accumulates 32 partial dot products in FP32 and the warp folds
// them with a 31-shuffle transpose-reduction that leaves output (r, c) on lane 4 r + c: one launch of a few us instead of the
// one-tile tensor-core kernel's staged pipeline, exact FP32 FMA arithmetic.
constexpr int kSkinnyMaxM = 256;
template <int ACT, bool VEC>
__global__ void __launch_bounds__(128) gemm_skinny_kernel(int M, int N, int K, const float* __restrict__ X, int ldx, const float* __restrict__ W,
                                                          const float* __restrict__ bias, const float* __restrict__ bias2, float* __restrict__ Y, int ldy) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int m0 = blockIdx.y * 8, n0 = (blockIdx.x * 4 + wid) * 4;
  if (n0 >= N) return;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
  const float* xr[8];
  const float* wr[4];
#pragma unroll
  for (int r = 0; r < 8; ++r) xr[r] = X + (size_t)min(m0 + r, M - 1) * ldx;      // rows / columns past the edge are clamped, never stored
#pragma unroll
  for (int c = 0; c < 4; ++c) wr[c] = W + (size_t)min(n0 + c, N - 1) * K;
  if (VEC) {
#pragma unroll 2
    for (int k = 4 * lane; k < K; k += 128) {
      float4 xv[8], wv[4];
#pragma unroll
      for (int r = 0; r < 8; ++r) xv[r] = *reinterpret_cast<const float4*>(xr[r] + k);
#pragma unroll
      for (int c = 0; c < 4; ++c) wv[c] = *reinterpret_cast<const float4*>(wr[c] + k);
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          acc[r * 4 + c] = fmaf(xv[r].w, wv[c].w, fmaf(xv[r].z, wv[c].z, fmaf(xv[r].y, wv[c].y, fmaf(xv[r].x, wv[c].x, acc[r * 4 + c]))));
    }
  } else {
#pragma unroll 4
    for (int k = lane; k < K; k += 32) {
      float xv[8], wv[4];
#pragma unroll
      for (int r = 0; r < 8; ++r) xv[r] = xr[r][k];
#pragma unroll
      for (int c = 0; c < 4; ++c) wv[c] = wr[c][k];
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r * 4 + c] = fmaf(xv[r], wv[c], acc[r * 4 + c]);
    }
  }
  // transpose-reduce: after the step with offset o a lane keeps the half of its values whose index has bit o equal to its own lane bit
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float keep = up ? acc[i + o] : acc[i];
      const float send = up ? acc[i] : acc[i + o];
      acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  const int m = m0 + (lane >> 2), n = n0 + (lane & 3);
  if (m < M && n < N) {
    float v = acc[0] + (bias ? bias[n] : 0.0f) + (bias2 ? bias2[n] : 0.0f);
    if (ACT == 1) v = fmaxf(v, 0.0f);
    Y[(size_t)m * ldy + n] = v;
  }
}

static int gemm_skinny_launch(cudaStream_t s, int M, int N, int K, const float* X, int ldx, const float* W, const float* b, const float* b2,
                              float* Y, int ldy, int act) {
  const dim3 grid((N + 15) / 16, (M + 7) / 8);
  const bool vec = (K % 4 == 0) && (ldx % 4 == 0) && (((uintptr_t)X | (uintptr_t)W) % 16 == 0);
  if (vec) {
    if (act == 1) gemm_skinny_kernel<1, true><<<grid, 128, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
    else gemm_skinny_kernel<0, true><<<grid, 128, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
  } else {
    if (act == 1) gemm_skinny_kernel<1, false><<<grid, 128, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
    else gemm_skinny_kernel<0, false><<<grid, 128, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
  }
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// Arithmetic of a Linear with more than kSkinnyMaxM rows; smaller ones run the exact FP32 skinny kernel either way.
enum GemmPrec { kTf32x3, kFp32 };
static int gemm_large(cudaStream_t s, GemmPrec prec, int M, int N, int K, const float* X, int ldx, const float* W, const float* b,
                      const float* b2, float* Y, int ldy, int act) {
  if (prec == kTf32x3) return gemm_tc_launch(s, M, N, K, X, ldx, W, b, b2, Y, ldy, act);
  dim3 grid((N + GT - 1) / GT, (M + GT - 1) / GT);
  if (act == 1)
    gemm_bias_act_kernel<1><<<grid, 256, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
  else
    gemm_bias_act_kernel<0><<<grid, 256, 0, s>>>(M, N, K, X, ldx, W, b, b2, Y, ldy);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
static int gemm(cudaStream_t s, GemmPrec prec, int M, int N, int K, const float* X, int ldx, const float* W, const float* b, const float* b2,
                float* Y, int ldy, int act) {
  if (M <= kSkinnyMaxM) return gemm_skinny_launch(s, M, N, K, X, ldx, W, b, b2, Y, ldy, act);
  return gemm_large(s, prec, M, N, K, X, ldx, W, b, b2, Y, ldy, act);
}
// The ragged entry points: rows [0, split) run on the kernel a call of at most kSkinnyMaxM rows selects, rows [split, M) on the one a
// larger call selects, so that each row gets the arithmetic of the single-track call it reproduces (every kernel computes an output row
// from its X row and W alone).  X + split * ldx keeps the 16-byte alignment the vector paths test whenever ldx % 4 == 0, and with
// ldx % 4 != 0 both the sub-range and the full call take the scalar path.
static int gemm_split(cudaStream_t s, GemmPrec prec, int split, int M, int N, int K, const float* X, int ldx, const float* W, const float* b,
                      const float* b2, float* Y, int ldy, int act) {
  int rc;
  if (split > 0 && (rc = gemm_skinny_launch(s, split, N, K, X, ldx, W, b, b2, Y, ldy, act))) return rc;
  if (split < M) return gemm_large(s, prec, M - split, N, K, X + (size_t)split * ldx, ldx, W, b, b2, Y + (size_t)split * ldy, ldy, act);
  return GLAMR_OK;
}

// ------------------------------------------------------------------------------------------------ LayerNorm(x + r), D = 256
__global__ void __launch_bounds__(128) add_layernorm_kernel(int M, const float* __restrict__ X, const float* __restrict__ R,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            float* __restrict__ Y) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M) return;
  float v[8];
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    v[i] = X[(size_t)row * 256 + c] + R[(size_t)row * 256 + c];
    s += v[i];
  }
  const float mean = warp_sum(s) * (1.0f / 256.0f);
  float q = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float d = v[i] - mean; q += d * d; }
  const float rstd = 1.0f / sqrtf(warp_sum(q) * (1.0f / 256.0f) + 1e-5f);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    Y[(size_t)row * 256 + c] = (v[i] - mean) * rstd * gamma[c] + beta[c];
  }
}

// ------------------------------------------------------------------------------------------------ attention, head dim 32
// Q rows (tq * B + b), K/V rows (tk * B + b) -- or batch-major (BM) rows b * Sq + tq, b * Sk + tk; row strides ldq / ldkv; 8 heads of
// 32.  key_mask [B,Sk] (1 = ignore) or NULL.
// grid (B, 8 heads, ceil(Sq / 8)): a CTA stages the head's K / V once and its 4 warps take 2 queries each, so that the kernel is
// one short dependent chain deep at the batch sizes of the inference (B = 1-4) instead of Sq / 4 of them.
constexpr int kAttnQChunk = 8;
template <bool BM>
__global__ void __launch_bounds__(128) attention_kernel(int B, int Sq, int Sk, const float* __restrict__ Q, int ldq,
                                                        const float* __restrict__ K, const float* __restrict__ V, int ldkv,
                                                        const uint8_t* __restrict__ key_mask, float* __restrict__ O, int ldo) {
  __shared__ float Ks[64][33];
  __shared__ float Vs[64][33];
  __shared__ float Ps[4][64];
  const int b = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int e = tid; e < Sk * 32; e += 128) {
    const int j = e >> 5, d = e & 31;
    const size_t kr = BM ? (size_t)b * Sk + j : (size_t)j * B + b;
    Ks[j][d] = K[kr * ldkv + h * 32 + d];
    Vs[j][d] = V[kr * ldkv + h * 32 + d];
  }
  __syncthreads();
  const float scale = 0.17677669529663687f;   // 1/sqrt(32)
  const int q_end = min(Sq, ((int)blockIdx.z + 1) * kAttnQChunk);
  for (int q = blockIdx.z * kAttnQChunk + w; q < q_end; q += 4) {
    const size_t qr = BM ? (size_t)b * Sq + q : (size_t)q * B + b;
    const float qd = Q[qr * ldq + h * 32 + lane] * scale;   // torch scales q before q k^T
    float sc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int j = lane + 32 * r;
      float a = 0.0f;
#pragma unroll
      for (int d = 0; d < 32; ++d) a = fmaf(__shfl_sync(0xffffffffu, qd, d), (j < Sk) ? Ks[j][d] : 0.0f, a);
      const bool dead = (j >= Sk) || (key_mask && key_mask[(size_t)b * Sk + j]);
      sc[r] = dead ? -INFINITY : a;
    }
    float mx = fmaxf(sc[0], sc[1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e0 = (sc[0] == -INFINITY) ? 0.0f : expf(sc[0] - mx), e1 = (sc[1] == -INFINITY) ? 0.0f : expf(sc[1] - mx);
    const float den = warp_sum(e0 + e1);
    Ps[w][lane] = e0 / den;
    Ps[w][lane + 32] = e1 / den;
    __syncwarp();
    float o = 0.0f;
    for (int j = 0; j < Sk; ++j) o = fmaf(Ps[w][j], Vs[j][lane], o);      // in key order (the reference's softmax(QK^T) V row sum)
    O[qr * ldo + h * 32 + lane] = o;
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------ positional encoding
// out[row] = [ src_row (in_dim) | PE(pos) (256) ] with the 'original' sinusoid (lib/models/pos_encoding.py:27-32);
// row = t * B + b (or, batch-major, row = b * S + t with per = S; else per = B), pos = t + pos_offset; src row = (src_bcast_t ? b : row)
// -> lets z be repeated over time.
template <bool BM>
__global__ void pe_concat_kernel(int rows, int per, int in_dim, const float* __restrict__ src, int src_ld, int src_bcast_t,
                                 int token_mode, int pos_offset, float* __restrict__ out) {
  const int row = blockIdx.x;
  if (row >= rows) return;
  const int q = row / per, r = row - q * per;
  const int t = BM ? r : q, b = BM ? q : r;
  const int od = in_dim + 256;
  const float* s = token_mode ? (src + (size_t)t * src_ld) : (src + (size_t)(src_bcast_t ? b : row) * src_ld);
  for (int c = threadIdx.x; c < od; c += blockDim.x) {
    float v;
    if (c < in_dim) {
      v = s[c];
    } else {
      const int e = c - in_dim;
      const float mul = expf((float)(e & ~1) * (-9.210340371976184f / 256.0f));   // exp(2i * -ln(1e4)/256)
      const float a = (float)(t + pos_offset) * mul;
      v = (e & 1) ? cosf(a) : sinf(a);
    }
    out[(size_t)row * od + c] = v;
  }
}

// rows t*B+b of out [T2,B,D] = cat(a[:Ta], b_[:Tb]) along time
__global__ void concat_time_kernel(int Ta, int Tb, int B, int D, const float* __restrict__ a, const float* __restrict__ b_,
                                   float* __restrict__ out) {
  const size_t total = (size_t)(Ta + Tb) * B * D;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / D;
    const int t = (int)(row / B);
    out[e] = (t < Ta) ? a[e] : b_[e - (size_t)Ta * B * D];
  }
}

// rows 0 .. B-1 of out [*,256] := tok_a, rows B .. 2B-1 := tok_b (the posterior's two query tokens at time 0 and 1, time-major)
__global__ void token_rows_kernel(int B, const float* __restrict__ tok_a, const float* __restrict__ tok_b, float* __restrict__ out) {
  const int row = blockIdx.x, c = threadIdx.x;
  out[(size_t)row * 256 + c] = (row < B ? tok_a : tok_b)[c];
}

// z = mu + eps * exp(0.5 logvar)  (lib/utils/dist.py:8-26); eps may be NULL (-> mu) or broadcast over the batch
__global__ void sample_z_kernel(int B, int nz, const float* __restrict__ mu, int ld_mu, const float* __restrict__ logvar, int ld_lv,
                                const float* __restrict__ eps, int eps_ld, float* __restrict__ z) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * nz) return;
  const int b = e / nz, k = e - b * nz;
  const float ep = eps ? eps[(size_t)b * eps_ld + k] : 0.0f;
  z[e] = mu[(size_t)b * ld_mu + k] + ep * expf(0.5f * logvar[(size_t)b * ld_lv + k]);
}

__global__ void mean_time_kernel(int T, int B, int D, const float* __restrict__ X, float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * D) return;
  float s = 0.0f;
  for (int t = 0; t < T; ++t) s += X[(size_t)t * B * D + e];
  out[e] = s / (float)T;
}

// ---- packed sequences of their own length: sequence b holds rows off[b] .. off[b+1] - 1 (off == NULL: every sequence has T rows)
__device__ __forceinline__ int seq_off(const int* off, int T, int b) { return off ? off[b] : b * T; }
// the sequence that packed row `row` belongs to
__device__ __forceinline__ int seq_of_row(const int* __restrict__ off, int B, int row) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}
// mean_time_kernel of each sequence over its own frames, in the same order
__global__ void mean_time_ragged_kernel(int B, int T, const int* __restrict__ off, int D, const float* __restrict__ X, float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * D) return;
  const int b = e / D, k = e - b * D;
  const int o = seq_off(off, T, b), n = seq_off(off, T, b + 1) - o;
  float s = 0.0f;
  for (int t = 0; t < n; ++t) s += X[((size_t)o + t) * D + k];
  out[e] = s / (float)n;
}
// concat_z_kernel with each packed row's own sequence
__global__ void concat_z_ragged_kernel(int rows, int B, int T, const int* __restrict__ off, int nz, int D, const float* __restrict__ z,
                                       const float* __restrict__ ctx, float* __restrict__ out) {
  const size_t total = (size_t)rows * (nz + D);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / (nz + D);
    const int c = (int)(e - row * (nz + D));
    const int b = off ? seq_of_row(off, B, (int)row) : (int)(row / T);
    out[e] = (c < nz) ? z[(size_t)b * nz + c] : ctx[row * D + (c - nz)];
  }
}

// [z (nz, per batch) | context row] -> rows of width nz + D
__global__ void concat_z_kernel(int rows, int B, int nz, int D, const float* __restrict__ z, const float* __restrict__ ctx,
                                float* __restrict__ out) {
  const size_t total = (size_t)rows * (nz + D);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / (nz + D);
    const int c = (int)(e - row * (nz + D));
    const int b = (int)(row % B);
    out[e] = (c < nz) ? z[(size_t)b * nz + c] : ctx[row * D + (c - nz)];
  }
}

// frame 0 of the predicted local trajectory: xy := init_xy (or 0), heading vec := init (or (0,1))
// (traj_pred_vae.py:319-329)
__global__ void traj_first_frame_kernel(int B, float* __restrict__ local /*[T,B,11]*/, const float* __restrict__ init_xy,
                                        const float* __restrict__ init_heading) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float* l = local + (size_t)b * 11;
  l[0] = init_xy ? init_xy[b * 2] : 0.0f;
  l[1] = init_xy ? init_xy[b * 2 + 1] : 0.0f;
  l[9] = init_heading ? cosf(init_heading[b]) : 0.0f;
  l[10] = init_heading ? sinf(init_heading[b]) : 1.0f;
}

// traj_first_frame_kernel on frame 0 of each packed sequence
__global__ void traj_first_frame_ragged_kernel(int B, const int* __restrict__ off, float* __restrict__ local /*[rows,11]*/,
                                               const float* __restrict__ init_xy, const float* __restrict__ init_heading) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float* l = local + (size_t)off[b] * 11;
  l[0] = init_xy ? init_xy[b * 2] : 0.0f;
  l[1] = init_xy ? init_xy[b * 2 + 1] : 0.0f;
  l[9] = init_heading ? cosf(init_heading[b]) : 0.0f;
  l[10] = init_heading ? sinf(init_heading[b]) : 1.0f;
}

__global__ void quat_rows_to_aa_kernel(int n, const float* __restrict__ q, float* __restrict__ aa) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float qq[4] = {q[i * 4], q[i * 4 + 1], q[i * 4 + 2], q[i * 4 + 3]}, a[3];
  quat_to_aa(qq, a);
  aa[i * 3] = a[0]; aa[i * 3 + 1] = a[1]; aa[i * 3 + 2] = a[2];
}

// ------------------------------------------------------------------------------------------------ LSTM recurrence
// nn.LSTMCell loop of lib/models/rnn.py:45-61 for one direction of one layer, hidden 128, gate order i,f,g,o.
// grid (B, 2 directions), 512 threads = one gate row each.  The recurrent matrix W_hh [512,128] lives on chip for the
// whole sequence: columns 0..63 of a thread's row in registers, columns 64..127 in shared memory ([k][row], conflict
// free).  xproj [T,B,2,512] already holds W_ih x_t + b_ih + b_hh.  out [T,B,256] = [h_fwd | h_bwd].
// PACKED: sequence b is rows seq_off(off, T, b) .. of its own length (xproj [rows,2,512], out [rows,256]); the backward direction starts
// at its own last frame.
constexpr int LH = 128, LG = 4 * LH, LREG = 64;
template <bool PACKED>
__global__ void __launch_bounds__(LG, 1) lstm_recurrence_kernel(int T, int B, const int* __restrict__ off, const float* __restrict__ xproj,
                                                                const float* __restrict__ whh_f, const float* __restrict__ whh_b,
                                                                float* __restrict__ out) {
  extern __shared__ float smem[];
  float* Wsm = smem;                       // [LH - LREG][LG]
  float* hs = Wsm + (LH - LREG) * LG;      // [LH]
  float* gs = hs + LH;                     // [LG]
  const int b = blockIdx.x, dir = blockIdx.y, r = threadIdx.x;
  const int o = PACKED ? seq_off(off, T, b) : 0;
  const int n = PACKED ? seq_off(off, T, b + 1) - o : T;
  const float* W = (dir == 0 ? whh_f : whh_b) + (size_t)r * LH;
  float wreg[LREG];
#pragma unroll
  for (int k = 0; k < LREG; ++k) wreg[k] = W[k];
  for (int k = 0; k < LH - LREG; ++k) Wsm[k * LG + r] = W[LREG + k];
  float c = 0.0f;
  if (r < LH) hs[r] = 0.0f;
  __syncthreads();
  for (int step = 0; step < n; ++step) {
    const int t = dir == 0 ? step : n - 1 - step;
    const size_t row = PACKED ? (size_t)o + t : (size_t)t * B + b;
    float a = xproj[(row * 2 + dir) * LG + r];
#pragma unroll
    for (int k4 = 0; k4 < LREG / 4; ++k4) {
      const float4 h4 = *reinterpret_cast<const float4*>(hs + 4 * k4);
      a = fmaf(wreg[4 * k4], h4.x, a);
      a = fmaf(wreg[4 * k4 + 1], h4.y, a);
      a = fmaf(wreg[4 * k4 + 2], h4.z, a);
      a = fmaf(wreg[4 * k4 + 3], h4.w, a);
    }
#pragma unroll 8
    for (int k = 0; k < LH - LREG; ++k) a = fmaf(Wsm[k * LG + r], hs[LREG + k], a);
    gs[r] = a;
    __syncthreads();
    if (r < LH) {
      const float ig = 1.0f / (1.0f + expf(-gs[r]));
      const float fg = 1.0f / (1.0f + expf(-gs[LH + r]));
      const float gg = tanhf(gs[2 * LH + r]);
      const float og = 1.0f / (1.0f + expf(-gs[3 * LH + r]));
      c = fg * c + ig * gg;
      const float h = og * tanhf(c);
      hs[r] = h;
      out[row * (2 * LH) + dir * LH + r] = h;
    }
    __syncthreads();
  }
}

}  // namespace glamr

// =================================================================================================== C ABI
using namespace glamr;

struct glamr_net {
  std::map<std::string, std::pair<float*, size_t>> t;
  std::vector<void*> allocs;
};

namespace {
const float* W(const glamr_net* n, const std::string& name, size_t expect, int* err) {
  auto it = n->t.find(name);
  if (it == n->t.end() || (expect && it->second.second != expect)) { *err = 1; return nullptr; }
  return it->second.first;
}

struct AttnW { const float *in_w, *in_b, *out_w, *out_b; };
struct EncLayer { AttnW sa; const float *l1w, *l1b, *l2w, *l2b, *n1g, *n1b, *n2g, *n2b; };
struct DecLayer { AttnW sa, ca; const float *l1w, *l1b, *l2w, *l2b, *n1g, *n1b, *n2g, *n2b, *n3g, *n3b; };

AttnW attn_w(const glamr_net* n, const std::string& p, int* e) {
  return {W(n, p + ".in_proj_weight", 768 * 256, e), W(n, p + ".in_proj_bias", 768, e), W(n, p + ".out_proj.weight", 256 * 256, e),
          W(n, p + ".out_proj.bias", 256, e)};
}
EncLayer enc_layer(const glamr_net* n, const std::string& p, int* e) {
  EncLayer L;
  L.sa = attn_w(n, p + ".self_attn", e);
  L.l1w = W(n, p + ".linear1.weight", 512 * 256, e); L.l1b = W(n, p + ".linear1.bias", 512, e);
  L.l2w = W(n, p + ".linear2.weight", 256 * 512, e); L.l2b = W(n, p + ".linear2.bias", 256, e);
  L.n1g = W(n, p + ".norm1.weight", 256, e); L.n1b = W(n, p + ".norm1.bias", 256, e);
  L.n2g = W(n, p + ".norm2.weight", 256, e); L.n2b = W(n, p + ".norm2.bias", 256, e);
  return L;
}
DecLayer dec_layer(const glamr_net* n, const std::string& p, int* e) {
  DecLayer L;
  L.sa = attn_w(n, p + ".self_attn", e);
  L.ca = attn_w(n, p + ".multihead_attn", e);
  L.l1w = W(n, p + ".linear1.weight", 512 * 256, e); L.l1b = W(n, p + ".linear1.bias", 512, e);
  L.l2w = W(n, p + ".linear2.weight", 256 * 512, e); L.l2b = W(n, p + ".linear2.bias", 256, e);
  L.n1g = W(n, p + ".norm1.weight", 256, e); L.n1b = W(n, p + ".norm1.bias", 256, e);
  L.n2g = W(n, p + ".norm2.weight", 256, e); L.n2b = W(n, p + ".norm2.bias", 256, e);
  L.n3g = W(n, p + ".norm3.weight", 256, e); L.n3b = W(n, p + ".norm3.bias", 256, e);
  return L;
}

struct Arena {
  float* base; size_t cap, used;
  float* take(size_t n) { size_t o = used; used += (n + 63) & ~(size_t)63; return used <= cap ? base + o : nullptr; }
};

// How the Linears of an infiller window choose their kernel.  rb == NULL: by the launch's own M (B sequences, time-major rows t * B + b).
// Otherwise the rows are batch-major (b * S + t) and slot b reproduces a call of rb[b] sequences (host array); the slots are ordered so
// that S * rb[b] > kSkinnyMaxM holds on a suffix of them for every S, and a Linear over S rows per slot runs as two row ranges.
struct WinDisp {
  int B;
  const int* rb;
};
int lin(cudaStream_t s, const WinDisp& d, int S, int N, int K, const float* X, int ldx, const float* W, const float* b, float* Y, int ldy,
        int act) {
  if (!d.rb) return gemm(s, kTf32x3, S * d.B, N, K, X, ldx, W, b, nullptr, Y, ldy, act);
  int j = 0;
  while (j < d.B && S * d.rb[j] <= kSkinnyMaxM) ++j;
  return gemm_split(s, kTf32x3, j * S, S * d.B, N, K, X, ldx, W, b, nullptr, Y, ldy, act);
}

int layernorm(cudaStream_t s, int M, const float* X, const float* R, const float* g, const float* b, float* Y) {
  add_layernorm_kernel<<<(M + 3) / 4, 128, 0, s>>>(M, X, R, g, b, Y);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// multi-head attention block: out = out_proj(attn(q_src, kv_src)); q_src [Sq*B,256], kv_src [Sk*B,256]
int mha(cudaStream_t s, Arena& A, const WinDisp& d, const AttnW& w, int Sq, int Sk, const float* q_src, const float* kv_src,
        const uint8_t* mask, float* out) {
  if (Sk > 64) return GLAMR_EUNSUPPORTED;
  const int B = d.B, Mq = Sq * B, Mk = Sk * B;
  const size_t mark = A.used;
  float* q = A.take((size_t)Mq * 256);
  float* kv = A.take((size_t)Mk * 512);
  float* att = A.take((size_t)Mq * 256);
  if (!q || !kv || !att) return GLAMR_ENOSPACE;
  int rc;
  if ((rc = lin(s, d, Sq, 256, 256, q_src, 256, w.in_w, w.in_b, q, 256, 0))) return rc;
  if ((rc = lin(s, d, Sk, 512, 256, kv_src, 256, w.in_w + 256 * 256, w.in_b + 256, kv, 512, 0))) return rc;
  const dim3 grid(B, 8, (Sq + kAttnQChunk - 1) / kAttnQChunk);
  if (d.rb) attention_kernel<true><<<grid, 128, 0, s>>>(B, Sq, Sk, q, 256, kv, kv + 256, 512, mask, att, 256);
  else attention_kernel<false><<<grid, 128, 0, s>>>(B, Sq, Sk, q, 256, kv, kv + 256, 512, mask, att, 256);
  GLAMR_LAUNCH_CHECK();
  if ((rc = lin(s, d, Sq, 256, 256, att, 256, w.out_w, w.out_b, out, 256, 0))) return rc;
  A.used = mark;
  return GLAMR_OK;
}

int ffn(cudaStream_t s, Arena& A, const WinDisp& d, int S, const float* x, const float* l1w, const float* l1b, const float* l2w,
        const float* l2b, float* out) {
  const size_t mark = A.used;
  float* h = A.take((size_t)S * d.B * 512);
  if (!h) return GLAMR_ENOSPACE;
  int rc;
  if ((rc = lin(s, d, S, 512, 256, x, 256, l1w, l1b, h, 512, 1))) return rc;
  if ((rc = lin(s, d, S, 256, 512, h, 512, l2w, l2b, out, 256, 0))) return rc;
  A.used = mark;
  return GLAMR_OK;
}

// nn.TransformerEncoderLayer, post-norm, relu, eval mode (dropout = identity); x updated in place
int encoder_layer(cudaStream_t s, Arena& A, const WinDisp& d, const EncLayer& L, int S, float* x, const uint8_t* mask) {
  const int M = S * d.B;
  const size_t mark = A.used;
  float* t = A.take((size_t)M * 256);
  if (!t) return GLAMR_ENOSPACE;
  int rc;
  if ((rc = mha(s, A, d, L.sa, S, S, x, x, mask, t))) return rc;
  if ((rc = layernorm(s, M, x, t, L.n1g, L.n1b, x))) return rc;
  if ((rc = ffn(s, A, d, S, x, L.l1w, L.l1b, L.l2w, L.l2b, t))) return rc;
  if ((rc = layernorm(s, M, x, t, L.n2g, L.n2b, x))) return rc;
  A.used = mark;
  return GLAMR_OK;
}
// nn.TransformerDecoderLayer (no tgt mask), memory [Sm*B,256] with key padding mask
int decoder_layer(cudaStream_t s, Arena& A, const WinDisp& d, const DecLayer& L, int S, int Sm, float* x, const float* mem,
                  const uint8_t* mem_mask) {
  const int M = S * d.B;
  const size_t mark = A.used;
  float* t = A.take((size_t)M * 256);
  if (!t) return GLAMR_ENOSPACE;
  int rc;
  if ((rc = mha(s, A, d, L.sa, S, S, x, x, nullptr, t))) return rc;
  if ((rc = layernorm(s, M, x, t, L.n1g, L.n1b, x))) return rc;
  if ((rc = mha(s, A, d, L.ca, S, Sm, x, mem, mem_mask, t))) return rc;
  if ((rc = layernorm(s, M, x, t, L.n2g, L.n2b, x))) return rc;
  if ((rc = ffn(s, A, d, S, x, L.l1w, L.l1b, L.l2w, L.l2b, t))) return rc;
  if ((rc = layernorm(s, M, x, t, L.n3g, L.n3b, x))) return rc;
  A.used = mark;
  return GLAMR_OK;
}
}  // namespace

// Y[M,N] = act(X[M,K] W[N,K]^T + bias) -- stand-alone entry for the GEMM used by every Linear of the prior networks
// (nn.Linear in lib/models/mlp.py:32-41, nn.MultiheadAttention projections, FFN).  mode: 1 wgmma 3xTF32, 0 FP32 SIMT.
extern "C" int glamr_linear_forward(int M, int N, int K, const float* X, const float* W, const float* bias, int relu, float* Y, int mode,
                                    void* stream) {
  if (M <= 0 || N <= 0 || K <= 0 || !X || !W || !Y) return GLAMR_EINVAL;
  return gemm((cudaStream_t)stream, mode == 1 ? kTf32x3 : kFp32, M, N, K, X, K, W, bias, nullptr, Y, N, relu ? 1 : 0);
}

extern "C" int glamr_net_create(glamr_net** out) {
  if (!out) return GLAMR_EINVAL;
  *out = new glamr_net();
  return GLAMR_OK;
}
extern "C" int glamr_net_destroy(glamr_net* n) {
  if (!n) return GLAMR_OK;
  cudaDeviceSynchronize();
  for (void* p : n->allocs) cudaFree(p);
  delete n;
  return GLAMR_OK;
}
// upload one named parameter (HOST pointer, float32)
extern "C" int glamr_net_set_tensor(glamr_net* n, const char* name, const float* host, size_t numel) {
  if (!n || !name || !host || numel == 0) return GLAMR_EINVAL;
  void* p = nullptr;
  GLAMR_CUDA_TRY(cudaMalloc(&p, numel * sizeof(float)));
  GLAMR_CUDA_TRY(cudaMemcpy(p, host, numel * sizeof(float), cudaMemcpyHostToDevice));
  n->allocs.push_back(p);
  n->t[name] = {(float*)p, numel};
  return GLAMR_OK;
}

extern "C" size_t glamr_infiller_workspace_floats(int B) { return (size_t)B * 50 * 256 * 16 + 65536; }

// One 50-frame window of MotionInfillerVAE.inference_one_step for d.B sequences (layout and kernel choice: WinDisp) -> *dec_out, the
// 30 decoded frames [30 B, 69] (arena memory).  in_pose [50 B, 69]  key_pad_mask [B,50]  eps rows eps_ld apart (0: one row for all) or NULL
// gt_cur NULL: mode 'infer', z drawn from the learned prior.  Otherwise mode 'recon' (time-major rows only): gt_cur [30,B,69] is the
// ground-truth body pose of the window's 30 current frames, and z is the mean of the posterior q(z | X, C); eps is not read.
static int infiller_window(const glamr_net* n, const WinDisp& d, const float* in_pose, const uint8_t* key_pad_mask, const float* eps,
                           int eps_ld, const float* gt_cur, float** dec_out_p, Arena& A, cudaStream_t s) {
  const int B = d.B;
  const bool bm = d.rb != nullptr;
  int e = 0;
  const std::string ce = "context_encoder.", dd = "data_decoder.";
  const float* in_fc_w = W(n, ce + "in_fc.weight", 256 * 69, &e), * in_fc_b = W(n, ce + "in_fc.bias", 256, &e);
  const float* cpe_w = W(n, ce + "pos_enc.fc.weight", 256 * 512, &e), * cpe_b = W(n, ce + "pos_enc.fc.bias", 256, &e);
  EncLayer enc[2] = {enc_layer(n, ce + "temporal_net.layers.0", &e), enc_layer(n, ce + "temporal_net.layers.1", &e)};
  const float* dpe_w = W(n, dd + "pos_enc.fc.weight", 256 * 384, &e), * dpe_b = W(n, dd + "pos_enc.fc.bias", 256, &e);
  DecLayer dec[2] = {dec_layer(n, dd + "temporal_net.layers.0", &e), dec_layer(n, dd + "temporal_net.layers.1", &e)};
  const float* om0w = W(n, dd + "out_mlp.affine_layers.0.weight", 512 * 256, &e), * om0b = W(n, dd + "out_mlp.affine_layers.0.bias", 512, &e);
  const float* om1w = W(n, dd + "out_mlp.affine_layers.1.weight", 256 * 512, &e), * om1b = W(n, dd + "out_mlp.affine_layers.1.bias", 256, &e);
  const float* ofw = W(n, dd + "out_fc.weight", 69 * 256, &e), * ofb = W(n, dd + "out_fc.bias", 69, &e);
  const float* ppe_w = W(n, dd + "prior_pos_enc.fc.weight", 256 * 512, &e), * ppe_b = W(n, dd + "prior_pos_enc.fc.bias", 256, &e);
  DecLayer pri = dec_layer(n, dd + "prior_temporal_net.layers.0", &e);
  const float* mu_tok = W(n, dd + "mu_token", 256, &e), * lv_tok = W(n, dd + "logvar_token", 256, &e);
  const float* pmw = W(n, dd + "p_z_mu_net.weight", 128 * 256, &e), * pmb = W(n, dd + "p_z_mu_net.bias", 128, &e);
  const float* plw = W(n, dd + "p_z_logvar_net.weight", 128 * 256, &e), * plb = W(n, dd + "p_z_logvar_net.bias", 128, &e);
  if (e) return GLAMR_EINVAL;
  const int S = 50, Sc = 30, M = S * B, Mc = Sc * B;
  float* x = A.take((size_t)M * 256);
  float* cat = A.take((size_t)M * 512);
  float* tok = A.take(2 * 256);
  float* px = A.take((size_t)2 * B * 256);
  float* mu = A.take((size_t)B * 128);
  float* lv = A.take((size_t)B * 128);
  float* z = A.take((size_t)B * 128);
  float* dx = A.take((size_t)Mc * 256);
  float* h1 = A.take((size_t)Mc * 512);
  float* h2 = A.take((size_t)Mc * 256);
  float* dec_out = A.take((size_t)Mc * 69);
  if (!dec_out) return GLAMR_ENOSPACE;
  int rc;
  auto pe_concat = [&](int rows, int per_tm, int per_bm, int in_dim, const float* src, int src_bcast_t, int token_mode, int pos_offset) {
    if (bm) pe_concat_kernel<true><<<rows, 128, 0, s>>>(rows, per_bm, in_dim, src, in_dim, src_bcast_t, token_mode, pos_offset, cat);
    else pe_concat_kernel<false><<<rows, 128, 0, s>>>(rows, per_tm, in_dim, src, in_dim, src_bcast_t, token_mode, pos_offset, cat);
  };
  // ---- context encoder (motion_infiller_vae.py:92-123)
  if ((rc = lin(s, d, S, 256, 69, in_pose, 69, in_fc_w, in_fc_b, x, 256, 0))) return rc;
  pe_concat(M, B, S, 256, x, 0, 0, 0);
  GLAMR_LAUNCH_CHECK();
  if ((rc = lin(s, d, S, 256, 512, cat, 512, cpe_w, cpe_b, x, 256, 0))) return rc;
  for (int l = 0; l < 2; ++l)
    if ((rc = encoder_layer(s, A, d, enc[l], S, x, key_pad_mask))) return rc;
  if (gt_cur) {
    // ---- posterior (DataEncoder.forward, :204-233): [mu token | logvar token | in_fc(30 ground-truth frames)] with the PE of
    // positions 0..31, two decoder layers (self-attention unmasked, cross-attention to the context), z = q_z_mu_net(row 0) (:375-376;
    // the logvar head reaches no output of this mode)
    if (bm) return GLAMR_EINVAL;
    const std::string de = "data_encoder.";
    const float* q_in_w = W(n, de + "in_fc.weight", 256 * 69, &e), * q_in_b = W(n, de + "in_fc.bias", 256, &e);
    const float* qpe_w = W(n, de + "pos_enc.fc.weight", 256 * 512, &e), * qpe_b = W(n, de + "pos_enc.fc.bias", 256, &e);
    DecLayer qdec[2] = {dec_layer(n, de + "temporal_net.layers.0", &e), dec_layer(n, de + "temporal_net.layers.1", &e)};
    const float* q_mu_tok = W(n, de + "mu_token", 256, &e), * q_lv_tok = W(n, de + "logvar_token", 256, &e);
    const float* qmw = W(n, de + "q_z_mu_net.weight", 128 * 256, &e), * qmb = W(n, de + "q_z_mu_net.bias", 128, &e);
    if (e) return GLAMR_EINVAL;
    const int Sq = 2 + Sc;
    float* qx = A.take((size_t)Sq * B * 256);
    if (!qx) return GLAMR_ENOSPACE;
    token_rows_kernel<<<2 * B, 256, 0, s>>>(B, q_mu_tok, q_lv_tok, qx);
    GLAMR_LAUNCH_CHECK();
    if ((rc = lin(s, d, Sc, 256, 69, gt_cur, 69, q_in_w, q_in_b, qx + (size_t)2 * B * 256, 256, 0))) return rc;
    pe_concat(Sq * B, B, Sq, 256, qx, 0, 0, 0);
    GLAMR_LAUNCH_CHECK();
    if ((rc = lin(s, d, Sq, 256, 512, cat, 512, qpe_w, qpe_b, qx, 256, 0))) return rc;
    for (int l = 0; l < 2; ++l)
      if ((rc = decoder_layer(s, A, d, qdec[l], Sq, S, qx, x, key_pad_mask))) return rc;
    if ((rc = lin(s, d, 1, 128, 256, qx, 256, qmw, qmb, z, 128, 0))) return rc;
  } else {
    // ---- learned prior over z (:354-362): two tokens attend to the context
    GLAMR_CUDA_TRY(cudaMemcpyAsync(tok, mu_tok, 256 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    GLAMR_CUDA_TRY(cudaMemcpyAsync(tok + 256, lv_tok, 256 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    pe_concat(2 * B, B, 2, 256, tok, 0, 1, 0);
    GLAMR_LAUNCH_CHECK();
    if ((rc = lin(s, d, 2, 256, 512, cat, 512, ppe_w, ppe_b, px, 256, 0))) return rc;
    if ((rc = decoder_layer(s, A, d, pri, 2, S, px, x, key_pad_mask))) return rc;
    // the mu token's rows, then the logvar token's: rows 0 .. B-1 and B .. 2B-1 time-major, every other row batch-major
    const float* pmu = px;
    const float* plv = bm ? px + 256 : px + (size_t)B * 256;
    const int ldp = bm ? 512 : 256;
    if ((rc = lin(s, d, 1, 128, 256, pmu, ldp, pmw, pmb, mu, 128, 0))) return rc;
    if ((rc = lin(s, d, 1, 128, 256, plv, ldp, plw, plb, lv, 128, 0))) return rc;
    sample_z_kernel<<<(B * 128 + 127) / 128, 128, 0, s>>>(B, 128, mu, 128, lv, 128, eps, eps_ld, z);
    GLAMR_LAUNCH_CHECK();
  }
  // ---- decoder (:383-395): z repeated over the 30 current frames, PE offset 10
  pe_concat(Mc, B, Sc, 128, z, 1, 0, 10);
  GLAMR_LAUNCH_CHECK();
  if ((rc = lin(s, d, Sc, 256, 384, cat, 384, dpe_w, dpe_b, dx, 256, 0))) return rc;
  for (int l = 0; l < 2; ++l)
    if ((rc = decoder_layer(s, A, d, dec[l], Sc, S, dx, x, key_pad_mask))) return rc;
  if ((rc = lin(s, d, Sc, 512, 256, dx, 256, om0w, om0b, h1, 512, 1))) return rc;
  if ((rc = lin(s, d, Sc, 256, 512, h1, 512, om1w, om1b, h2, 256, 1))) return rc;
  if ((rc = lin(s, d, Sc, 69, 256, h2, 256, ofw, ofb, dec_out, 69, 0))) return rc;
  *dec_out_p = dec_out;
  return GLAMR_OK;
}

// One 50-frame window of MotionInfillerVAE.inference_one_step (mode 'infer', sample_num 1), B sequences.
//   in_pose [50,B,69]  key_pad_mask [B,50] (1 = frame not usable as key)  eps [B or 1,128] (eps_rows = B or 1) or NULL
//   out_pose [40,B,69] = [first 10 input frames | 30 decoded frames]
extern "C" int glamr_infiller_window_forward(const glamr_net* n, int B, const float* in_pose, const uint8_t* key_pad_mask,
                                             const float* eps, int eps_rows, float* out_pose, float* workspace,
                                             size_t workspace_floats, void* stream) {
  if (!n || B <= 0 || !in_pose || !key_pad_mask || !out_pose || !workspace) return GLAMR_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  Arena A{workspace, workspace_floats, 0};
  float* dec_out = nullptr;
  const int rc = infiller_window(n, WinDisp{B, nullptr}, in_pose, key_pad_mask, eps, eps_rows == 1 ? 0 : 128, nullptr, &dec_out, A, s);
  if (rc) return rc;
  concat_time_kernel<<<64, 256, 0, s>>>(10, 30, B, 69, in_pose, dec_out, out_pose);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}


// ------------------------------------------------------------------------------------------------ all windows of a sequence
// motion_infiller_vae.py:618-632: the autoregressive sweep of 50-frame windows with stride 30.  Window i reads frames
// [30 i, 30 i + 50) of the running pose (zeros past the end), masks keys that are invisible or past the end (the 10 past frames
// are always usable), and its first min(40, T - 30 i) output frames replace the running pose.  One call for the whole sweep: the
// window staging / commit are two small kernels instead of a dozen framework ops per window.
__global__ void window_prep_kernel(int T, int B, int s0, const float* __restrict__ pose, const uint8_t* __restrict__ key_pad_all,
                                   float* __restrict__ win, uint8_t* __restrict__ kp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = B * 69;
  if (i < 50 * row) {
    const int t = i / row;
    win[i] = (s0 + t < T) ? pose[(size_t)(s0 + t) * row + (i - t * row)] : 0.0f;
  }
  if (i < B * 50) {
    const int b = i / 50, t = i - b * 50;
    kp[i] = t < 10 ? 0 : ((s0 + t < T) ? key_pad_all[(size_t)b * T + s0 + t] : 1);
  }
}
__global__ void window_commit_kernel(int B, int s0, int nfr, const float* __restrict__ out, float* __restrict__ pose) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = B * 69;
  if (i < nfr * row) pose[(size_t)s0 * row + i] = out[i];
}

// the ground truth of window s0's 30 current frames: gwin [30,B,69] = frames s0 + 10 .. s0 + 39 of gt [T,B,69], zero past T
__global__ void window_gt_kernel(int T, int B, int s0, const float* __restrict__ gt, float* __restrict__ gwin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = B * 69;
  if (i >= 30 * row) return;
  const int t = s0 + 10 + i / row;
  gwin[i] = t < T ? gt[(size_t)t * row + i % row] : 0.0f;
}

extern "C" size_t glamr_infiller_sequence_workspace_floats(int B) {
  return glamr_infiller_workspace_floats(B) + (size_t)90 * B * 69 + (size_t)(B * 50 + 3) / 4 + 192;
}
extern "C" size_t glamr_infiller_recon_workspace_floats(int B) {
  if (B <= 0) return 0;
  return glamr_infiller_sequence_workspace_floats(B) + (((size_t)30 * B * 69 + 63) & ~(size_t)63);
}

// The sweep of both modes: gt NULL runs 'infer' with eps, otherwise 'recon' with the ground truth gt [T,B,69] (eps not read).
static int infiller_sweep(const glamr_net* n, int T, int B, float* pose_io, const float* gt, const uint8_t* key_pad_all, const float* eps,
                          int eps_rows, float* workspace, size_t workspace_floats, cudaStream_t s) {
  float* win = workspace;
  float* out = win + (size_t)50 * B * 69;
  uint8_t* kp = reinterpret_cast<uint8_t*>(out + (size_t)40 * B * 69);
  float* rest = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(kp + (size_t)B * 50) + 255) & ~(uintptr_t)255);
  float* gwin = nullptr;
  if (gt) {
    gwin = rest;
    rest += ((size_t)30 * B * 69 + 63) & ~(size_t)63;
  }
  const size_t rest_floats = workspace_floats - (size_t)(rest - workspace);
  const int nwin = (T - 10 + 29) / 30;
  const int prep_blocks = (50 * B * 69 + 255) / 256;
  for (int i = 0; i < nwin; ++i) {
    const int s0 = i * 30;
    window_prep_kernel<<<prep_blocks, 256, 0, s>>>(T, B, s0, pose_io, key_pad_all, win, kp);
    GLAMR_LAUNCH_CHECK();
    if (gt) {
      window_gt_kernel<<<(30 * B * 69 + 255) / 256, 256, 0, s>>>(T, B, s0, gt, gwin);
      GLAMR_LAUNCH_CHECK();
    }
    Arena A{rest, rest_floats, 0};
    float* dec = nullptr;
    const float* eps_i = gt ? nullptr : eps + (size_t)i * eps_rows * 128;
    const int rc = infiller_window(n, WinDisp{B, nullptr}, win, kp, eps_i, eps_rows == 1 ? 0 : 128, gwin, &dec, A, s);
    if (rc) return rc;
    concat_time_kernel<<<64, 256, 0, s>>>(10, 30, B, 69, win, dec, out);
    GLAMR_LAUNCH_CHECK();
    const int nfr = (s0 + 40 < T ? s0 + 40 : T) - s0;
    window_commit_kernel<<<(nfr * B * 69 + 255) / 256, 256, 0, s>>>(B, s0, nfr, out, pose_io);
    GLAMR_LAUNCH_CHECK();
  }
  return GLAMR_OK;
}

//   pose_io [T,B,69]: the input body pose, overwritten with the infilled pose   key_pad_all [B,T] uint8 (1 = frame invisible)
//   eps [n_windows][eps_rows][128] with eps_rows in {1, B}, n_windows = ceil((T - 10) / 30)
extern "C" int glamr_infiller_forward(const glamr_net* n, int T, int B, float* pose_io, const uint8_t* key_pad_all, const float* eps,
                                      int eps_rows, float* workspace, size_t workspace_floats, void* stream) {
  if (!n || T <= 10 || B <= 0 || !pose_io || !key_pad_all || !eps || !workspace || (eps_rows != 1 && eps_rows != B)) return GLAMR_EINVAL;
  if (workspace_floats < glamr_infiller_sequence_workspace_floats(B)) return GLAMR_ENOSPACE;
  return infiller_sweep(n, T, B, pose_io, nullptr, key_pad_all, eps, eps_rows, workspace, workspace_floats, (cudaStream_t)stream);
}

//   pose_io [T,B,69]: the input body pose, overwritten with the reconstructed pose   gt_body_pose [T,B,69]: the ground truth the
//   posterior encodes   key_pad_all [B,T] uint8 (1 = frame invisible)
extern "C" int glamr_infiller_recon_forward(const glamr_net* n, int T, int B, float* pose_io, const float* gt_body_pose,
                                            const uint8_t* key_pad_all, float* workspace, size_t workspace_floats, void* stream) {
  if (!n || T <= 10 || B <= 0 || !pose_io || !gt_body_pose || !key_pad_all || !workspace) return GLAMR_EINVAL;
  if (workspace_floats < glamr_infiller_recon_workspace_floats(B)) return GLAMR_ENOSPACE;
  return infiller_sweep(n, T, B, pose_io, gt_body_pose, key_pad_all, nullptr, 1, workspace, workspace_floats, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------ tracks of their own length
// The ragged entry points take B tracks packed without padding: track b is rows offsets[b] .. offsets[b+1] - 1 (offsets [B+1] on the
// device, lens [B] and row_batch [B] on the host).  Row b reproduces the single-track entry called for a batch of row_batch[b] tracks of
// its length (1 for a lone track, P for a block of P equal-length tracks): each Linear of that call picks its kernel by M, so the rows are
// ordered by the kernel each Linear runs for them, and every Linear runs as at most two launches over contiguous rows (gemm_split).

// The infiller's kernel choice for a call of rb tracks: which of its Linears (50, 30, 2 and 1 rows per track) exceed kSkinnyMaxM rows.
static int infiller_class(int rb) {
  const int S[4] = {50, 30, 2, 1};
  int c = 0;
  for (int i = 0; i < 4; ++i) c += S[i] * rb > kSkinnyMaxM;
  return c;
}
static int infiller_windows(int T) { return (T - 10 + 29) / 30; }

// Window slots -> tracks.  The tracks are ordered by infiller class and, within a class, by decreasing length, so the tracks that still
// have window i form a prefix of each class: slot j of segment g (slot0[g] <= j < slot0[g+1]) is track row0[g] + j - slot0[g].
constexpr int kMaxInfillerClasses = 5;
struct SlotMap {
  int nseg;
  int slot0[kMaxInfillerClasses + 1], row0[kMaxInfillerClasses];
};
__device__ __forceinline__ int slot_track(const SlotMap& m, int j) {
  int g = 0;
  while (g + 1 < m.nseg && j >= m.slot0[g + 1]) ++g;
  return m.row0[g] + j - m.slot0[g];
}
// window_prep_kernel for the Bi active slots (batch-major window [Bi,50,69], key mask [Bi,50]), plus each slot's eps of window `wi`
__global__ void window_prep_ragged_kernel(int Bi, SlotMap m, int wi, int s0, int eps_windows, const int* __restrict__ off,
                                          const float* __restrict__ pose, const uint8_t* __restrict__ key_pad, const float* __restrict__ eps,
                                          float* __restrict__ win, uint8_t* __restrict__ kp, float* __restrict__ epsw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Bi * 50 * 69) {
    const int j = i / (50 * 69), t = (i - j * 50 * 69) / 69, k = i - (j * 50 + t) * 69;
    const int r = slot_track(m, j), o = off[r], T = off[r + 1] - o;
    win[i] = (s0 + t < T) ? pose[((size_t)o + s0 + t) * 69 + k] : 0.0f;
  }
  if (i < Bi * 50) {
    const int j = i / 50, t = i - j * 50;
    const int r = slot_track(m, j), o = off[r], T = off[r + 1] - o;
    kp[i] = t < 10 ? 0 : ((s0 + t < T) ? key_pad[(size_t)o + s0 + t] : 1);
  }
  if (i < Bi * 128) {
    const int j = i / 128, k = i - j * 128;
    epsw[i] = eps[((size_t)slot_track(m, j) * eps_windows + wi) * 128 + k];
  }
}
// window_commit_kernel: the first min(40, T - s0) frames of [10 input frames | 30 decoded frames] replace the track's running pose
__global__ void window_commit_ragged_kernel(int Bi, SlotMap m, int s0, const int* __restrict__ off, const float* __restrict__ win,
                                            const float* __restrict__ dec, float* __restrict__ pose) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Bi * 40 * 69) return;
  const int j = i / (40 * 69), t = (i - j * 40 * 69) / 69, k = i - (j * 40 + t) * 69;
  const int r = slot_track(m, j), o = off[r], T = off[r + 1] - o;
  if (t < min(40, T - s0)) pose[((size_t)o + s0 + t) * 69 + k] = t < 10 ? win[((size_t)j * 50 + t) * 69 + k] : dec[((size_t)j * 30 + t - 10) * 69 + k];
}

extern "C" size_t glamr_infiller_ragged_workspace_floats(int B) {
  if (B <= 0) return 0;
  return glamr_infiller_workspace_floats(B) + (size_t)50 * B * 69 + (size_t)B * 128 + (size_t)(B * 50 + 3) / 4 + 256;
}

extern "C" int glamr_infiller_forward_ragged(const glamr_net* n, int B, const int* lens, const int* row_batch, const int* offsets,
                                             float* pose_io, const uint8_t* key_pad, const float* eps, int eps_windows, float* workspace,
                                             size_t workspace_floats, void* stream) {
  if (!n || B <= 0 || !lens || !row_batch || !offsets || !pose_io || !key_pad || !eps || !workspace) return GLAMR_EINVAL;
  int nmax = 0;
  for (int b = 0; b < B; ++b) {
    if (lens[b] <= 10 || row_batch[b] <= 0) return GLAMR_EINVAL;
    if (b > 0) {
      const int c0 = infiller_class(row_batch[b - 1]), c1 = infiller_class(row_batch[b]);
      if (c1 < c0 || (c1 == c0 && lens[b] > lens[b - 1])) return GLAMR_EINVAL;
    }
    nmax = max(nmax, infiller_windows(lens[b]));
  }
  if (eps_windows < nmax) return GLAMR_EINVAL;
  if (workspace_floats < glamr_infiller_ragged_workspace_floats(B)) return GLAMR_ENOSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  float* win = workspace;
  float* epsw = win + (size_t)50 * B * 69;
  uint8_t* kp = reinterpret_cast<uint8_t*>(epsw + (size_t)B * 128);
  float* rest = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(kp + (size_t)B * 50) + 255) & ~(uintptr_t)255);
  const size_t rest_floats = workspace_floats - (size_t)(rest - workspace);
  std::vector<int> rb_slot(B);
  for (int i = 0; i < nmax; ++i) {
    SlotMap m{};
    int Bi = 0;
    for (int b0 = 0; b0 < B;) {
      int b1 = b0;
      while (b1 < B && infiller_class(row_batch[b1]) == infiller_class(row_batch[b0])) ++b1;
      m.slot0[m.nseg] = Bi;
      m.row0[m.nseg++] = b0;
      for (int b = b0; b < b1 && infiller_windows(lens[b]) > i; ++b) rb_slot[Bi++] = row_batch[b];
      b0 = b1;
    }
    m.slot0[m.nseg] = Bi;
    const int s0 = i * 30;
    window_prep_ragged_kernel<<<(Bi * 50 * 69 + 255) / 256, 256, 0, s>>>(Bi, m, i, s0, eps_windows, offsets, pose_io, key_pad, eps, win, kp, epsw);
    GLAMR_LAUNCH_CHECK();
    Arena A{rest, rest_floats, 0};
    float* dec = nullptr;
    const int rc = infiller_window(n, WinDisp{Bi, rb_slot.data()}, win, kp, epsw, 128, nullptr, &dec, A, s);
    if (rc) return rc;
    window_commit_ragged_kernel<<<(Bi * 40 * 69 + 255) / 256, 256, 0, s>>>(Bi, m, s0, offsets, win, dec, pose_io);
    GLAMR_LAUNCH_CHECK();
  }
  return GLAMR_OK;
}

extern "C" size_t glamr_trajpred_workspace_floats(int T, int B) { return (size_t)T * B * (512 + 256 + 2 * 512 + 256 + 384 + 512 + 256 + 64) + (size_t)B * 2048 + 65536; }

extern "C" int glamr_traj_local2global(int T, int B, const float* local_traj, int local_heading, float* trans, float* orient_q,
                                       float* scratch, void* stream);

// The trajectory predictor's network for R independent rows of T frames (traj_pred_vae.py:72-92 context encoder, :281-297
// prior + z, :298-333 decoder up to out_fc): in [T,R,69] -> raw [T,R,11], the decoder output before any frame-0 override.
// eps [R or 1,128] (eps_rows = R or 1) or NULL (-> z = mu).  Scratch comes from A.  The single-pass and the windowed entry
// points both run the network through here.  Its Linears stay on the FP32 GEMMs: their matrices are launch-latency sized, and the
// per-frame heading error accumulates through the codec's prefix sum.
// Packed rows (the ragged entries): sequence b of the R holds frames seq_off(off, T, b) .. of its own length, M frames in all; frames
// [0, fsplit) and sequences [0, rsplit) run their Linears on the kernel a call of at most kSkinnyMaxM rows selects, the rest on the larger one.
struct Packed {
  const int* off;
  int M, fsplit, rsplit;
};
static int trajpred_network(const glamr_net* n, int T, int R, const Packed* pk, const float* in, const float* eps, int eps_rows, float* raw,
                            Arena& A, cudaStream_t s) {
  int e = 0;
  const std::string ce = "context_encoder.", dd = "data_decoder.";
  const float* im0w = W(n, ce + "in_mlp.affine_layers.0.weight", 512 * 69, &e), * im0b = W(n, ce + "in_mlp.affine_layers.0.bias", 512, &e);
  const float* im1w = W(n, ce + "in_mlp.affine_layers.1.weight", 256 * 512, &e), * im1b = W(n, ce + "in_mlp.affine_layers.1.bias", 256, &e);
  const float *wih[2][2], *whh[2][2], *bih[2][2], *bhh[2][2];
  for (int l = 0; l < 2; ++l)
    for (int d = 0; d < 2; ++d) {
      const std::string p = ce + "temporal_net." + std::to_string(l) + (d == 0 ? ".rnn_f." : ".rnn_b.");
      wih[l][d] = W(n, p + "weight_ih", 512 * 256, &e); whh[l][d] = W(n, p + "weight_hh", 512 * 128, &e);
      bih[l][d] = W(n, p + "bias_ih", 512, &e); bhh[l][d] = W(n, p + "bias_hh", 512, &e);
    }
  const float* cm0w = W(n, ce + "out_mlp.affine_layers.0.weight", 512 * 256, &e), * cm0b = W(n, ce + "out_mlp.affine_layers.0.bias", 512, &e);
  const float* cm1w = W(n, ce + "out_mlp.affine_layers.1.weight", 256 * 512, &e), * cm1b = W(n, ce + "out_mlp.affine_layers.1.bias", 256, &e);
  const float* pm0w = W(n, dd + "prior_mlp.affine_layers.0.weight", 512 * 256, &e), * pm0b = W(n, dd + "prior_mlp.affine_layers.0.bias", 512, &e);
  const float* pm1w = W(n, dd + "prior_mlp.affine_layers.1.weight", 256 * 512, &e), * pm1b = W(n, dd + "prior_mlp.affine_layers.1.bias", 256, &e);
  const float* pzw = W(n, dd + "p_z_net.weight", 256 * 256, &e), * pzb = W(n, dd + "p_z_net.bias", 256, &e);
  const float* dm0w = W(n, dd + "out_mlp.affine_layers.0.weight", 512 * 384, &e), * dm0b = W(n, dd + "out_mlp.affine_layers.0.bias", 512, &e);
  const float* dm1w = W(n, dd + "out_mlp.affine_layers.1.weight", 256 * 512, &e), * dm1b = W(n, dd + "out_mlp.affine_layers.1.bias", 256, &e);
  const float* ofw = W(n, dd + "out_fc.weight", 11 * 256, &e), * ofb = W(n, dd + "out_fc.bias", 11, &e);
  if (e) return GLAMR_EINVAL;
  const int M = pk ? pk->M : T * R;
  auto flin = [&](int N, int K, const float* X, int ldx, const float* Wt, const float* b, const float* b2, float* Y, int ldy, int act) {
    return pk ? gemm_split(s, kFp32, pk->fsplit, M, N, K, X, ldx, Wt, b, b2, Y, ldy, act) : gemm(s, kFp32, M, N, K, X, ldx, Wt, b, b2, Y, ldy, act);
  };
  auto rlin = [&](int N, int K, const float* X, int ldx, const float* Wt, const float* b, float* Y, int ldy, int act) {
    return pk ? gemm_split(s, kFp32, pk->rsplit, R, N, K, X, ldx, Wt, b, nullptr, Y, ldy, act) : gemm(s, kFp32, R, N, K, X, ldx, Wt, b, nullptr, Y, ldy, act);
  };
  float* h512 = A.take((size_t)M * 512);
  float* x = A.take((size_t)M * 256);
  float* xp = A.take((size_t)M * 2 * 512);
  float* y = A.take((size_t)M * 256);
  float* cat = A.take((size_t)M * 384);
  float* hm = A.take((size_t)R * 256);
  float* hp = A.take((size_t)R * 512);
  float* hq = A.take((size_t)R * 256);
  float* pz = A.take((size_t)R * 256);
  float* z = A.take((size_t)R * 128);
  if (!z) return GLAMR_ENOSPACE;
  int rc;
  static bool attr = false;
  const size_t lstm_smem = ((size_t)(LH - LREG) * LG + LH + LG) * sizeof(float);
  if (!attr) {
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lstm_recurrence_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lstm_smem));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lstm_recurrence_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lstm_smem));
    attr = true;
  }
  // ---- context encoder (traj_pred_vae.py:72-92)
  if ((rc = flin(512, 69, in, 69, im0w, im0b, nullptr, h512, 512, 1))) return rc;
  if ((rc = flin(256, 512, h512, 512, im1w, im1b, nullptr, x, 256, 1))) return rc;
  for (int l = 0; l < 2; ++l) {
    for (int d = 0; d < 2; ++d)   // xproj[t][b][d][:] = W_ih x + b_ih + b_hh
      if ((rc = flin(512, 256, x, 256, wih[l][d], bih[l][d], bhh[l][d], xp + d * 512, 1024, 0))) return rc;
    if (pk) lstm_recurrence_kernel<true><<<dim3(R, 2), LG, lstm_smem, s>>>(T, R, pk->off, xp, whh[l][0], whh[l][1], y);
    else lstm_recurrence_kernel<false><<<dim3(R, 2), LG, lstm_smem, s>>>(T, R, nullptr, xp, whh[l][0], whh[l][1], y);
    GLAMR_LAUNCH_CHECK();
    float* tmp = x; x = y; y = tmp;
  }
  if ((rc = flin(512, 256, x, 256, cm0w, cm0b, nullptr, h512, 512, 1))) return rc;
  if ((rc = flin(256, 512, h512, 512, cm1w, cm1b, nullptr, y, 256, 1))) return rc;      // y = context
  // ---- prior + z (:281-297)
  if (pk) mean_time_ragged_kernel<<<(R * 256 + 127) / 128, 128, 0, s>>>(R, T, pk->off, 256, y, hm);
  else mean_time_kernel<<<(R * 256 + 127) / 128, 128, 0, s>>>(T, R, 256, y, hm);
  GLAMR_LAUNCH_CHECK();
  if ((rc = rlin(512, 256, hm, 256, pm0w, pm0b, hp, 512, 1))) return rc;
  if ((rc = rlin(256, 512, hp, 512, pm1w, pm1b, hq, 256, 1))) return rc;
  if ((rc = rlin(256, 256, hq, 256, pzw, pzb, pz, 256, 0))) return rc;
  sample_z_kernel<<<(R * 128 + 127) / 128, 128, 0, s>>>(R, 128, pz, 256, pz + 128, 256, eps, eps_rows == 1 ? 0 : 128, z);
  GLAMR_LAUNCH_CHECK();
  // ---- decoder (:298-333)
  if (pk) concat_z_ragged_kernel<<<256, 256, 0, s>>>(M, R, T, pk->off, 128, 256, z, y, cat);
  else concat_z_kernel<<<256, 256, 0, s>>>(M, R, 128, 256, z, y, cat);
  GLAMR_LAUNCH_CHECK();
  if ((rc = flin(512, 384, cat, 384, dm0w, dm0b, nullptr, h512, 512, 1))) return rc;
  if ((rc = flin(256, 512, h512, 512, dm1w, dm1b, nullptr, x, 256, 1))) return rc;
  return flin(11, 256, x, 256, ofw, ofb, nullptr, raw, 11, 0);
}

// TrajPredVAE.inference (multi_step False, sample_num 1): joint positions -> local trajectory -> global trajectory.
//   in_joint_pos [T,B,69]   eps [B or 1,128] or NULL   init_xy [B,2] / init_heading [B] or NULL
//   out_local_traj [T,B,11]  out_trans [T,B,3]  out_orient_aa [T,B,3]
extern "C" int glamr_trajpred_forward(const glamr_net* n, int T, int B, const float* in_joint_pos, const float* eps, int eps_rows,
                                      const float* init_xy, const float* init_heading, float* out_local_traj, float* out_trans,
                                      float* out_orient_aa, float* workspace, size_t workspace_floats, void* stream) {
  if (!n || T <= 0 || B <= 0 || !in_joint_pos || !out_local_traj || !out_trans || !out_orient_aa || !workspace) return GLAMR_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  Arena A{workspace, workspace_floats, 0};
  const int M = T * B;
  int rc;
  if ((rc = trajpred_network(n, T, B, nullptr, in_joint_pos, eps, eps_rows, out_local_traj, A, s))) return rc;
  float* oq = A.take((size_t)M * 4);
  float* sc = A.take((size_t)M * 3);
  if (!sc) return GLAMR_ENOSPACE;
  traj_first_frame_kernel<<<(B + 127) / 128, 128, 0, s>>>(B, out_local_traj, init_xy, init_heading);
  GLAMR_LAUNCH_CHECK();
  if ((rc = glamr_traj_local2global(T, B, out_local_traj, 1, out_trans, oq, sc, stream))) return rc;
  quat_rows_to_aa_kernel<<<(M + 127) / 128, 128, 0, s>>>(M, oq, out_orient_aa);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// ------------------------------------------------------------------------------------------------ windowed trajectory prediction
// TrajPredVAE.inference_multi_step (traj_pred_vae.py:484-520, sample_num 1): the track is cut into C = ceil(T / W) windows of W
// frames, the last one zero-padded in joint-position space, and every window runs the network on its own.  A window reads no
// other window's output (the stitch below rewrites only frame 0's heading vector, from columns 3:9 that nothing rewrites), so
// all of them go through the network as R = C * B rows of one batch.  Rows are window-major: row c * B + b is window c of
// sequence b, which makes eps [C,B,128] the rows' eps as laid out.

// [T,B,69] -> [W,C*B,69]: window c, frame t of sequence b = global frame c W + t, zero past T
__global__ void traj_window_gather_kernel(int T, int B, int W, int C, const float* __restrict__ jp, float* __restrict__ win) {
  const size_t total = (size_t)W * C * B * 69;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / 69;                       // t * (C B) + c B + b
    const int k = (int)(e - row * 69);
    const int t = (int)(row / ((size_t)C * B));
    const int cb = (int)(row - (size_t)t * C * B);
    const int c = cb / B, b = cb - c * B;
    const int tg = c * W + t;
    win[e] = tg < T ? jp[((size_t)tg * B + b) * 69 + k] : 0.0f;
  }
}

// raw [W,C*B,11] -> local [T,B,11] (get_res_from_cur_data, :500-506).  Window 0 contributes its overridden output (frame 0:
// xy = 0, heading vector (0, 1): no init_xy / init_heading reaches a window, :319-327); window c >= 1 its raw output with
// frame 0's heading vector replaced by heading_to_vec(get_heading(rot6d_to_quat(.))) of global frame c W - 1's columns 3:9.
// Padded frames are dropped.  One thread per output row.
// src: the frame's raw row; prev: raw row W - 1 of window c - 1
__device__ __forceinline__ void traj_window_stitch_row(int c, int tw, const float* __restrict__ src, const float* __restrict__ prev,
                                                       float* __restrict__ dst) {
  float l[11];
#pragma unroll
  for (int k = 0; k < 11; ++k) l[k] = src[k];
  if (tw == 0) {
    if (c == 0) {
      l[0] = 0.0f; l[1] = 0.0f; l[9] = 0.0f; l[10] = 1.0f;
    } else {
      float R[9], q[4];
      rot6d_to_rotmat(prev + 3, R);
      rotmat_to_quat(R, q);
      const float h = 2.0f * safe_atan2(q[3], q[0]);
      l[9] = cosf(h); l[10] = sinf(h);
    }
  }
#pragma unroll
  for (int k = 0; k < 11; ++k) dst[k] = l[k];
}
__global__ void traj_window_stitch_kernel(int T, int B, int W, int C, const float* __restrict__ raw, float* __restrict__ local) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T * B) return;
  const int t = i / B, b = i - t * B;
  const int c = t / W, tw = t - c * W;
  traj_window_stitch_row(c, tw, raw + ((size_t)tw * C * B + (size_t)c * B + b) * 11,
                         c > 0 ? raw + ((size_t)(W - 1) * C * B + (size_t)(c - 1) * B + b) * 11 : nullptr, local + (size_t)i * 11);
}

extern "C" size_t glamr_trajpred_windows_workspace_floats(int T, int B, int W) {
  if (T <= 0 || B <= 0 || W <= 0) return 0;
  const size_t C = ((size_t)T + W - 1) / W, R = C * B;
  return (size_t)W * R * (69 + 11) + (size_t)T * B * 7 + 4 * 64 + glamr_trajpred_workspace_floats(W, (int)R);
}

//   in_joint_pos [T,B,69]   eps [C,B,128] or NULL (z = mu)   out_local_traj [T,B,11]  out_trans [T,B,3]  out_orient_aa [T,B,3]
extern "C" int glamr_trajpred_windows_forward(const glamr_net* n, int T, int B, int W, const float* in_joint_pos, const float* eps,
                                              float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                              size_t workspace_floats, void* stream) {
  if (!n || T <= 0 || B <= 0 || W <= 0 || !in_joint_pos || !out_local_traj || !out_trans || !out_orient_aa || !workspace) return GLAMR_EINVAL;
  const int C = (T + W - 1) / W;
  if ((size_t)C * B > (size_t)INT_MAX / W) return GLAMR_EINVAL;
  const int R = C * B;
  if (workspace_floats < glamr_trajpred_windows_workspace_floats(T, B, W)) return GLAMR_ENOSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  Arena A{workspace, workspace_floats, 0};
  float* win = A.take((size_t)W * R * 69);
  float* raw = A.take((size_t)W * R * 11);
  float* oq = A.take((size_t)T * B * 4);
  float* sc = A.take((size_t)T * B * 3);
  if (!sc) return GLAMR_ENOSPACE;
  traj_window_gather_kernel<<<1024, 256, 0, s>>>(T, B, W, C, in_joint_pos, win);
  GLAMR_LAUNCH_CHECK();
  int rc;
  if ((rc = trajpred_network(n, W, R, nullptr, win, eps, R, raw, A, s))) return rc;
  traj_window_stitch_kernel<<<(T * B + 127) / 128, 128, 0, s>>>(T, B, W, C, raw, out_local_traj);
  GLAMR_LAUNCH_CHECK();
  if ((rc = glamr_traj_local2global(T, B, out_local_traj, 1, out_trans, oq, sc, stream))) return rc;
  quat_rows_to_aa_kernel<<<(T * B + 127) / 128, 128, 0, s>>>(T * B, oq, out_orient_aa);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// ------------------------------------------------------------------------------------------------ ragged trajectory predictor
extern "C" int glamr_traj_local2global(int T, int B, const float* local_traj, int local_heading, float* trans, float* orient_q,
                                       float* scratch, void* stream);
namespace glamr {
int traj_local2global_ragged(int B, const int* offsets, const float* local_traj, float* trans, float* orient_q, float* scratch,
                             cudaStream_t stream);
}

// The predictor's kernel choice for a call whose Linears have `frames` rows per frame-wise layer and `rows` per sequence-wise layer
static int trajpred_class(long long frames, long long rows) { return (frames > kSkinnyMaxM) + (rows > kSkinnyMaxM); }

static int ragged_total(int B, const int* lens) {
  long long M = 0;
  for (int b = 0; b < B; ++b) {
    if (lens[b] <= 0) return -1;
    M += lens[b];
  }
  return M > INT_MAX / 1024 ? -1 : (int)M;
}

extern "C" size_t glamr_trajpred_ragged_workspace_floats(int B, const int* lens) {
  const int M = (B > 0 && lens) ? ragged_total(B, lens) : -1;
  return M < 0 ? 0 : glamr_trajpred_workspace_floats(M, 1) + (size_t)B * 2048;
}

extern "C" int glamr_trajpred_forward_ragged(const glamr_net* n, int B, const int* lens, const int* row_batch, const int* offsets,
                                             const float* in_joint_pos, const float* eps, const float* init_xy, const float* init_heading,
                                             float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                             size_t workspace_floats, void* stream) {
  if (!n || B <= 0 || !lens || !row_batch || !offsets || !in_joint_pos || !out_local_traj || !out_trans || !out_orient_aa || !workspace)
    return GLAMR_EINVAL;
  const int M = ragged_total(B, lens);
  if (M < 0) return GLAMR_EINVAL;
  Packed pk{offsets, M, 0, 0};
  for (int b = 0; b < B; ++b) {
    if (row_batch[b] <= 0) return GLAMR_EINVAL;
    const int c = trajpred_class((long long)lens[b] * row_batch[b], row_batch[b]);
    if (b > 0 && c < trajpred_class((long long)lens[b - 1] * row_batch[b - 1], row_batch[b - 1])) return GLAMR_EINVAL;
    if (c == 0) pk.fsplit += lens[b];
    if (c < 2) ++pk.rsplit;
  }
  if (workspace_floats < glamr_trajpred_ragged_workspace_floats(B, lens)) return GLAMR_ENOSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  Arena A{workspace, workspace_floats, 0};
  int rc;
  if ((rc = trajpred_network(n, 0, B, &pk, in_joint_pos, eps, B, out_local_traj, A, s))) return rc;
  float* oq = A.take((size_t)M * 4);
  float* sc = A.take((size_t)M * 3);
  if (!sc) return GLAMR_ENOSPACE;
  traj_first_frame_ragged_kernel<<<(B + 127) / 128, 128, 0, s>>>(B, offsets, out_local_traj, init_xy, init_heading);
  GLAMR_LAUNCH_CHECK();
  if ((rc = traj_local2global_ragged(B, offsets, out_local_traj, out_trans, oq, sc, s))) return rc;
  quat_rows_to_aa_kernel<<<(M + 127) / 128, 128, 0, s>>>(M, oq, out_orient_aa);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// window row w (window c of track b, w = win_offsets[b] + c), frame tw = global frame c W + tw of track b, zero past its end
__global__ void traj_window_gather_ragged_kernel(int B, int W, int Rw, const int* __restrict__ off, const int* __restrict__ woff,
                                                 const float* __restrict__ jp, float* __restrict__ win) {
  const size_t total = (size_t)Rw * W * 69;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t row = e / 69;
    const int k = (int)(e - row * 69);
    const int w = (int)(row / W), tw = (int)(row - (size_t)w * W);
    const int b = seq_of_row(woff, B, w);
    const int t = (w - woff[b]) * W + tw, o = off[b];
    win[e] = t < off[b + 1] - o ? jp[((size_t)o + t) * 69 + k] : 0.0f;
  }
}
__global__ void traj_window_stitch_ragged_kernel(int B, int W, int M, const int* __restrict__ off, const int* __restrict__ woff,
                                                 const float* __restrict__ raw, float* __restrict__ local) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int b = seq_of_row(off, B, i);
  const int t = i - off[b], c = t / W, tw = t - c * W;
  const size_t w = (size_t)woff[b] + c;
  traj_window_stitch_row(c, tw, raw + (w * W + tw) * 11, c > 0 ? raw + ((w - 1) * W + W - 1) * 11 : nullptr, local + (size_t)i * 11);
}

static long long ragged_windows(int B, const int* lens, int W) {
  long long C = 0;
  for (int b = 0; b < B; ++b) C += (lens[b] + W - 1) / W;
  return C;
}

extern "C" size_t glamr_trajpred_windows_ragged_workspace_floats(int B, const int* lens, int W) {
  const int M = (B > 0 && lens && W > 0) ? ragged_total(B, lens) : -1;
  if (M < 0) return 0;
  const long long Rw = ragged_windows(B, lens, W);
  if (Rw * W > INT_MAX / 1024) return 0;
  return (size_t)W * Rw * (69 + 11) + (size_t)M * 7 + 4 * 64 + glamr_trajpred_workspace_floats(W, (int)Rw);
}

extern "C" int glamr_trajpred_windows_forward_ragged(const glamr_net* n, int B, int W, const int* lens, const int* row_batch,
                                                     const int* offsets, const int* win_offsets, const float* in_joint_pos, const float* eps,
                                                     float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                                     size_t workspace_floats, void* stream) {
  if (!n || B <= 0 || W <= 0 || !lens || !row_batch || !offsets || !win_offsets || !in_joint_pos || !out_local_traj || !out_trans ||
      !out_orient_aa || !workspace)
    return GLAMR_EINVAL;
  const size_t need = glamr_trajpred_windows_ragged_workspace_floats(B, lens, W);
  if (need == 0) return GLAMR_EINVAL;
  const int M = ragged_total(B, lens), Rw = (int)ragged_windows(B, lens, W);
  // window rows inherit their track's class: a single-track call of rb tracks runs C rb windows of W frames as one batch
  Packed pk{nullptr, Rw * W, 0, 0};
  for (int b = 0; b < B; ++b) {
    if (row_batch[b] <= 0) return GLAMR_EINVAL;
    const long long C = (lens[b] + W - 1) / W, r = C * row_batch[b];
    const int c = trajpred_class(r * W, r);
    if (b > 0) {
      const long long rp = (long long)((lens[b - 1] + W - 1) / W) * row_batch[b - 1];
      if (c < trajpred_class(rp * W, rp)) return GLAMR_EINVAL;
    }
    if (c == 0) pk.fsplit += (int)C * W;
    if (c < 2) pk.rsplit += (int)C;
  }
  if (workspace_floats < need) return GLAMR_ENOSPACE;
  cudaStream_t s = (cudaStream_t)stream;
  Arena A{workspace, workspace_floats, 0};
  float* win = A.take((size_t)W * Rw * 69);
  float* raw = A.take((size_t)W * Rw * 11);
  float* oq = A.take((size_t)M * 4);
  float* sc = A.take((size_t)M * 3);
  if (!sc) return GLAMR_ENOSPACE;
  traj_window_gather_ragged_kernel<<<1024, 256, 0, s>>>(B, W, Rw, offsets, win_offsets, in_joint_pos, win);
  GLAMR_LAUNCH_CHECK();
  int rc;
  if ((rc = trajpred_network(n, W, Rw, &pk, win, eps, Rw, raw, A, s))) return rc;
  traj_window_stitch_ragged_kernel<<<(M + 127) / 128, 128, 0, s>>>(B, W, M, offsets, win_offsets, raw, out_local_traj);
  GLAMR_LAUNCH_CHECK();
  if ((rc = traj_local2global_ragged(B, offsets, out_local_traj, out_trans, oq, sc, s))) return rc;
  quat_rows_to_aa_kernel<<<(M + 127) / 128, 128, 0, s>>>(M, oq, out_orient_aa);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
