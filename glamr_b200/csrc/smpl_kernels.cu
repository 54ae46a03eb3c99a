// SMPL forward on sm_90a: Rodrigues + kinematic chain (pose_prep), blend shapes + pose blend + linear blend skinning
// (lbs_kernel: 1-D bulk-TMA / mbarrier double-buffered posedirs slabs, FP32 FMA, K-sparse skinning), extra joint
// regression + joint remap + re-rooting (joints_finalize).  Reference arithmetic: smplx.lbs as stated in-tree at
// HybrIK/hybrik/models/layers/smpl/lbs.py:195-288,402-548 and GLAMR's wrapper lib/models/smpl.py:289-343.
#include <math.h>
#include <algorithm>
#include <cmath>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "glamr_math.cuh"
#include "smpl_model.cuh"

namespace glamr {

// ------------------------------------------------------------------------------------------------ pose_prep
// One warp per frame-person, lane j < 24 owns joint j.
//   R_j = rodrigues(pose_j)                                   lbs.py:446-477
//   J_j = j_template + j_shapedirs . beta  (== J_regressor @ v_shaped, lbs.py:240-244, by linearity)
//   G_j = G_parent(j) * [R_j | J_j - J_parent],  A_j = G_j - [0 | G_j J_j]      lbs.py:493-548
__global__ void __launch_bounds__(128) pose_prep_kernel(SmplDev m, int n, const float* __restrict__ orient,
                                                        const float* __restrict__ body_pose,
                                                        const float* __restrict__ betas, int use_betas, SmplWorkspace w) {
  pdl_launch_dependents();
  pdl_wait();
  const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (f >= n) return;
  pose_prep_frame(m, f, orient ? orient + (size_t)f * 3 : nullptr, body_pose + (size_t)f * 69, use_betas ? betas + (size_t)f * kNB : nullptr, w,
                  threadIdx.x & 31);
}

// ------------------------------------------------------------------------------------------------ lbs_kernel
// CTA = 128 vertices x 32 frame-persons, 128 threads (4 warps).  Warp w owns frames 8w..8w+7, lane l owns vertices
// 4l..4l+3 of the tile: a 12 (columns) x 8 (frames) register tile = 96 FP32 accumulators per thread.
//   v_posed = v_template + shapedirs.beta + posedirs^T.pose_feature           lbs.py:240,256-267
//   vert    = (sum_k w_k A_k) [v_posed; 1]                                    lbs.py:273-284
// Why this shape: the kernel is shared-memory-bandwidth bound unless the register tile is large.  Per k a thread reads
// 12 posedirs values (3 LDS.128, distinct per lane) + 8 pose-feature values (2 LDS.128, warp-broadcast) = 20 wavefronts
// per warp for 96 FFMA (0.21 wavefronts/FFMA, below the 0.25 the LSU can sustain next to 4 FFMA/clk); the first
// version (3 x 16 tile) needed 19 wavefronts per 48 FFMA and stalled on the LSU.
// All operands arrive by 1-D bulk TMA (cp.async.bulk + mbarrier): the CTA's posedirs slab [207][384] in 23 chunks of
// 9 rows (13,824 B contiguous thanks to the tile-major re-layout), the matching [9][32] pose-feature chunk, and the
// A tile [24][32][12]; a 3-stage full/empty mbarrier ring replaces __syncthreads in the main loop.
constexpr int kFramesPerCta = 32;
constexpr int kFramesPerWarp = 8;
constexpr int kVertsPerThread = 4;
constexpr int kLbsThreads = 128;
constexpr int kMaxStages = 4;
constexpr int kChunkFloats = kChunkK * kTileCols;                 // 3456 posedirs floats per stage
constexpr uint32_t kChunkBytes = kChunkFloats * sizeof(float);    // 13,824
constexpr int kPfChunkFloats = kChunkK * kFramesPerCta;           // 288 pose-feature floats per stage
constexpr uint32_t kPfChunkBytes = kPfChunkFloats * sizeof(float);
constexpr int kATileFloats = kFramesPerCta * kNJ * 12;            // 9216
constexpr int kVpFloats = kVTile * 3 * kFramesPerCta;            // 12,288: v_posed tile handed from the GEMM phase to the skinning phase
__host__ __device__ constexpr int stage_region_floats(int stages) { return (stages * (kChunkFloats + kPfChunkFloats) > kVpFloats) ? stages * (kChunkFloats + kPfChunkFloats) : kVpFloats; }
constexpr size_t lbs_smem_bytes(int stages) { return (size_t)(stage_region_floats(stages) + kATileFloats + kFramesPerCta * kNB) * sizeof(float) + (2 * kMaxStages + 1) * sizeof(uint64_t); }

template <int KREG, int kStages>
__global__ void __launch_bounds__(kLbsThreads, 2)
lbs_kernel(SmplDev m, int n_begin, int n_end, const float* __restrict__ betas, SmplWorkspace w, float* __restrict__ vertices, int dbg) {
  constexpr int kStageRegionFloats = stage_region_floats(kStages);
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* PDs = reinterpret_cast<float*>(smem_raw);              // [kStages][9][384]
  float* pfs = PDs + kStages * kChunkFloats;                     // [kStages][9][32]
  float* As = PDs + kStageRegionFloats;                          // [24][32 frames][12]
  float* bs = As + kATileFloats;                                 // [32][10]
  uint64_t* full = reinterpret_cast<uint64_t*>(bs + kFramesPerCta * kNB);   // [kStages]
  uint64_t* empty = full + kStages;                              // [kStages]
  uint64_t* abar = empty + kStages;                              // A tile

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int wf = (tid >> 5) * kFramesPerWarp;                   // first frame (within the tile) of this warp
  const int vtile = blockIdx.x;
  const int f0 = n_begin + blockIdx.y * kFramesPerCta;
  const int gv0 = vtile * kVTile + lane * kVertsPerThread;      // first of this thread's 4 vertices
  const float* pd_slab = m.pd_tiles + (size_t)vtile * kPF * kTileCols;
  const float* pf_slab = w.pf + (size_t)(f0 >> 5) * kNChunks * kPfChunkFloats;

  pdl_launch_dependents();
  // issue the per-vertex constant loads first: their latency overlaps the barrier set-up and the first TMA round trip
  float sdv[kVertsPerThread][30], vt[kVertsPerThread][3];
  {
    const float4* sd4 = reinterpret_cast<const float4*>(m.shapedirs + (size_t)gv0 * 30);           // gv0 % 4 == 0 -> 480-byte aligned
    float tmp[kVertsPerThread * 30];
#pragma unroll
    for (int q = 0; q < kVertsPerThread * 30 / 4; ++q) {
      const float4 t4 = __ldg(sd4 + q);
      tmp[4 * q] = t4.x; tmp[4 * q + 1] = t4.y; tmp[4 * q + 2] = t4.z; tmp[4 * q + 3] = t4.w;
    }
#pragma unroll
    for (int v = 0; v < kVertsPerThread; ++v)
#pragma unroll
      for (int k = 0; k < 30; ++k) sdv[v][k] = tmp[v * 30 + k];
    const float4* vt4 = reinterpret_cast<const float4*>(m.v_template + (size_t)gv0 * 3);            // 12 contiguous floats
    const float4 a = __ldg(vt4), b = __ldg(vt4 + 1), c = __ldg(vt4 + 2);
    vt[0][0] = a.x; vt[0][1] = a.y; vt[0][2] = a.z; vt[1][0] = a.w; vt[1][1] = b.x; vt[1][2] = b.y;
    vt[2][0] = b.z; vt[2][1] = b.w; vt[2][2] = c.x; vt[3][0] = c.y; vt[3][1] = c.z; vt[3][2] = c.w;
  }
  float bpre[(kFramesPerCta * kNB + kLbsThreads - 1) / kLbsThreads];
#pragma unroll
  for (int i = 0; i < (kFramesPerCta * kNB + kLbsThreads - 1) / kLbsThreads; ++i) {
    const int e = tid + i * kLbsThreads;
    const int f = e / kNB, l = e - f * kNB;
    const int nn = f0 + f;
    bpre[i] = (e < kFramesPerCta * kNB && nn < n_end) ? betas[(size_t)nn * kNB + l] : 0.0f;
  }
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kLbsThreads / 32); }
    mbar_init(abar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto issue_chunk = [&](int c) {      // producer: one elected thread, two bulk copies per stage
    const int s = c % kStages;
    mbar_expect_tx(&full[s], kChunkBytes + kPfChunkBytes);
    tma_bulk_g2s(PDs + s * kChunkFloats, pd_slab + (size_t)c * kChunkFloats, kChunkBytes, &full[s]);
    tma_bulk_g2s(pfs + s * kPfChunkFloats, pf_slab + (size_t)c * kPfChunkFloats, kPfChunkBytes, &full[s]);
  };
  // posedirs is a model constant: the first stages' slabs are fetched before this grid waits for its producer
  // (pose_prep_kernel, PDL); their pose-feature halves and the A tile follow after pdl_wait().
  if (tid == 0) {
#pragma unroll
    for (int c = 0; c < kStages - 1; ++c) {
      mbar_expect_tx_only(&full[c], kChunkBytes);
      tma_bulk_g2s(PDs + c * kChunkFloats, pd_slab + (size_t)c * kChunkFloats, kChunkBytes, &full[c]);
    }
  }
#pragma unroll
  for (int i = 0; i < (kFramesPerCta * kNB + kLbsThreads - 1) / kLbsThreads; ++i) {
    const int e = tid + i * kLbsThreads;
    if (e < kFramesPerCta * kNB) bs[e] = bpre[i];
  }
  __syncthreads();

  // acc[f][c]: c = 3 * vertex + coord over the thread's 4 vertices
  float acc[kFramesPerWarp][12];
#pragma unroll
  for (int f = 0; f < kFramesPerWarp; ++f) {
    float bl[kNB];
#pragma unroll
    for (int l = 0; l < kNB; ++l) bl[l] = bs[(wf + f) * kNB + l];
#pragma unroll
    for (int v = 0; v < kVertsPerThread; ++v) {
      float a0 = vt[v][0], a1 = vt[v][1], a2 = vt[v][2];
#pragma unroll
      for (int l = 0; l < kNB; ++l) {
        a0 = fmaf(sdv[v][l], bl[l], a0);
        a1 = fmaf(sdv[v][10 + l], bl[l], a1);
        a2 = fmaf(sdv[v][20 + l], bl[l], a2);
      }
      acc[f][3 * v + 0] = a0; acc[f][3 * v + 1] = a1; acc[f][3 * v + 2] = a2;
    }
  }

  pdl_wait();                          // A and pf below are written by pose_prep_kernel
  if (tid == 0) {
    mbar_expect_tx(abar, (uint32_t)kATileFloats * sizeof(float));
    tma_bulk_g2s(As, w.A + (size_t)(f0 >> 5) * kATileFloats, (uint32_t)kATileFloats * sizeof(float), abar);
#pragma unroll
    for (int c = 0; c < kStages - 1; ++c) {
      mbar_expect_tx(&full[c], kPfChunkBytes);
      tma_bulk_g2s(pfs + c * kPfChunkFloats, pf_slab + (size_t)c * kPfChunkFloats, kPfChunkBytes, &full[c]);
    }
  }

  for (int c = 0; c < kNChunks; ++c) {
    const int s = c % kStages;
    if (tid == 0 && c + kStages - 1 < kNChunks) {
      // the stage about to be refilled was last read for chunk c-1: wait until every warp released it
      if (c >= 1) mbar_wait(&empty[(c + kStages - 1) % kStages], ((c - 1) / kStages) & 1);
      issue_chunk(c + kStages - 1);
    }
    mbar_wait(&full[s], (c / kStages) & 1);
    const float4* P = reinterpret_cast<const float4*>(PDs + s * kChunkFloats + 12 * lane);
    const float4* F = reinterpret_cast<const float4*>(pfs + s * kPfChunkFloats + wf);
    if (!(GLAMR_DBG(dbg) & 1))
#pragma unroll
    for (int k = 0; k < kChunkK; ++k) {
      const float4 p0 = P[k * (kTileCols / 4) + 0], p1 = P[k * (kTileCols / 4) + 1], p2 = P[k * (kTileCols / 4) + 2];
      const float4 q0 = F[k * (kFramesPerCta / 4) + 0], q1 = F[k * (kFramesPerCta / 4) + 1];
      const float pv[12] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, p2.x, p2.y, p2.z, p2.w};
      const float qv[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
      for (int f = 0; f < kFramesPerWarp; ++f)
#pragma unroll
        for (int cc = 0; cc < 12; ++cc) acc[f][cc] = fmaf(qv[f], pv[cc], acc[f][cc]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  // ---- hand the v_posed tile to the skinning phase through shared memory (the stage buffers are free now).
  // Layout VP[row = vertex*3 + coord][32 frames] with the 4-frame chunk index XOR-swizzled by the writing lane so that
  // both the STS.128 here (lanes = vertices) and the LDS.32 below (lanes = frames) are bank-conflict free.
  __syncthreads();
  float* VP = PDs;
#pragma unroll
  for (int v = 0; v < kVertsPerThread; ++v)
#pragma unroll
    for (int cc = 0; cc < 3; ++cc) {
      const int row = (lane * kVertsPerThread + v) * 3 + cc;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int chunk = ((wf >> 2) + h) ^ (lane & 7);
        *reinterpret_cast<float4*>(VP + row * 32 + chunk * 4) =
            make_float4(acc[4 * h + 0][3 * v + cc], acc[4 * h + 1][3 * v + cc], acc[4 * h + 2][3 * v + cc], acc[4 * h + 3][3 * v + cc]);
      }
    }
  mbar_wait(abar, 0);
  __syncthreads();

  // ---- skinning: warp w owns vertices 32w..32w+31 of the tile, lane = frame.  Joint indices / weights are
  // warp-uniform (prefetched one vertex per lane, broadcast with shuffles), a lane reads its frame's A_j with three
  // LDS.128: every LDS is conflict free.
  const int fr = lane;
  const int n = f0 + fr;
  const bool n_ok = n < n_end;
  const int vbase = (tid >> 5) * 32;
  if (!(GLAMR_DBG(dbg) & 2)) {
    if (KREG > 0) {
      const int gvl = min(vtile * kVTile + vbase + lane, kVPad - 1);
      const float4 my_w = *reinterpret_cast<const float4*>(m.skin_w + (size_t)gvl * 4);
      const unsigned int my_j = *reinterpret_cast<const unsigned int*>(m.skin_j + (size_t)gvl * 4);
      const int my_ci = m.compact_of_vertex[gvl];
#pragma unroll 4
      for (int i = 0; i < 32; ++i) {
        const int vi = vbase + i;
        const int gv = vtile * kVTile + vi;
        if (gv >= kV) break;
        const float w0 = __shfl_sync(0xffffffffu, my_w.x, i), w1 = __shfl_sync(0xffffffffu, my_w.y, i);
        const float w2 = __shfl_sync(0xffffffffu, my_w.z, i), w3 = __shfl_sync(0xffffffffu, my_w.w, i);
        const unsigned int jj = __shfl_sync(0xffffffffu, my_j, i);
        const int ci = __shfl_sync(0xffffffffu, my_ci, i);
        const int pos = ((((fr >> 2) ^ ((vi >> 2) & 7)) << 2) | (fr & 3));
        const float x = VP[(vi * 3 + 0) * 32 + pos], y = VP[(vi * 3 + 1) * 32 + pos], z = VP[(vi * 3 + 2) * 32 + pos];
        const float4* a0 = reinterpret_cast<const float4*>(As + ((jj & 0xff) * 32 + fr) * 12);
        const float4* a1 = reinterpret_cast<const float4*>(As + (((jj >> 8) & 0xff) * 32 + fr) * 12);
        const float4* a2 = reinterpret_cast<const float4*>(As + (((jj >> 16) & 0xff) * 32 + fr) * 12);
        const float4* a3 = reinterpret_cast<const float4*>(As + (((jj >> 24) & 0xff) * 32 + fr) * 12);
        float T[12];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float4 q0 = a0[r], q1 = a1[r], q2 = a2[r], q3 = a3[r];
          T[4 * r + 0] = fmaf(w3, q3.x, fmaf(w2, q2.x, fmaf(w1, q1.x, w0 * q0.x)));
          T[4 * r + 1] = fmaf(w3, q3.y, fmaf(w2, q2.y, fmaf(w1, q1.y, w0 * q0.y)));
          T[4 * r + 2] = fmaf(w3, q3.z, fmaf(w2, q2.z, fmaf(w1, q1.z, w0 * q0.z)));
          T[4 * r + 3] = fmaf(w3, q3.w, fmaf(w2, q2.w, fmaf(w1, q1.w, w0 * q0.w)));
        }
        const float ox = fmaf(T[0], x, fmaf(T[1], y, fmaf(T[2], z, T[3])));
        const float oy = fmaf(T[4], x, fmaf(T[5], y, fmaf(T[6], z, T[7])));
        const float oz = fmaf(T[8], x, fmaf(T[9], y, fmaf(T[10], z, T[11])));
        if (n_ok) {
          if (vertices) {
            float* o = vertices + ((size_t)n * kV + gv) * 3;
            o[0] = ox; o[1] = oy; o[2] = oz;
          }
          if (ci >= 0) {
            float* o = w.vcompact + ((size_t)n * m.S + ci) * 3;
            o[0] = ox; o[1] = oy; o[2] = oz;
          }
        }
      }
    } else {
      for (int vi = vbase; vi < vbase + 32; ++vi) {
        const int gv = vtile * kVTile + vi;
        if (gv >= kV) break;
        const int ci = m.compact_of_vertex[gv];
        const int pos = ((((fr >> 2) ^ ((vi >> 2) & 7)) << 2) | (fr & 3));
        const float x = VP[(vi * 3 + 0) * 32 + pos], y = VP[(vi * 3 + 1) * 32 + pos], z = VP[(vi * 3 + 2) * 32 + pos];
        float T[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) T[k] = 0.0f;
        for (int s = 0; s < m.K; ++s) {
          const int jj = m.skin_j[(size_t)gv * m.K + s];
          const float wt = m.skin_w[(size_t)gv * m.K + s];
          const float* a = As + (jj * 32 + fr) * 12;
#pragma unroll
          for (int k = 0; k < 12; ++k) T[k] = fmaf(wt, a[k], T[k]);
        }
        const float ox = fmaf(T[0], x, fmaf(T[1], y, fmaf(T[2], z, T[3])));
        const float oy = fmaf(T[4], x, fmaf(T[5], y, fmaf(T[6], z, T[7])));
        const float oz = fmaf(T[8], x, fmaf(T[9], y, fmaf(T[10], z, T[11])));
        if (n_ok) {
          if (vertices) {
            float* o = vertices + ((size_t)n * kV + gv) * 3;
            o[0] = ox; o[1] = oy; o[2] = oz;
          }
          if (ci >= 0) {
            float* o = w.vcompact + ((size_t)n * m.S + ci) * 3;
            o[0] = ox; o[1] = oy; o[2] = oz;
          }
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------ blend features
// The A operand of the blend GEMM for frame-person f: (R_j - I) of the 23 body joints (lbs.py:256-258), the betas, the constant 1
// that multiplies v_template and zero padding, as scaled fp16 hi / lo in the wgmma image (put_blend_features).  It depends on the body
// pose and the betas only -- NOT on the root orientation -- so the optimiser evaluates it (and the blend GEMM behind it) off the
// critical path of the iteration.  One warp per frame-person.
__global__ void __launch_bounds__(128) blend_features_kernel(int n, const float* __restrict__ body_pose, const float* __restrict__ betas, SmplWorkspace w) {
  const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f >= n) return;
  float R[9];
  if (lane >= 1 && lane < kNJ) {
    const float* bp = body_pose + (size_t)f * 69 + (lane - 1) * 3;
    const float rv[3] = {bp[0], bp[1], bp[2]};
    rodrigues_smplx(rv, R);
  }
  put_blend_features(w, f, lane, R, betas ? betas + (size_t)f * kNB : nullptr);
}

// ------------------------------------------------------------------------------------------------ tensor-core LBS
// The shape blend + pose blend of SMPL is one contraction  v_posed[frame, col] = sum_k feat[frame, k] basis[col, k]
// (k: 207 pose features x posedirs | 10 betas x shapedirs | 1 x v_template; lbs.py:240,256-267), i.e. a [n x 218] x [218 x 20670]
// GEMM.  lbs_blend_tc_kernel runs it on the Hopper tensor cores (wgmma) with FP32 accuracy (3xFP16: hi*hi + lo*hi + hi*lo,
// |error| ~ 2e-7 on the blended vertex): both operands are scaled by powers of two (the basis by 2^e_B, feature row f by 2^e_f) into
// FP16's normal range, where an fp16 hi / lo pair carries the 22 significant bits of a tf32 pair at twice the tensor-core rate and
// half the bytes.  They are PRE-SPLIT and pre-tiled in global memory as the K-major core-matrix image wgmma reads from shared memory
// (basis once at glamr_smpl_create, features by put_blend_features), so a pipeline stage is two 1-D bulk TMA copies (8 KB of A, 16 KB
// of B) with no SIMT work on the operand path.  Tile = 128 frames x 256 basis columns, K in 14 steps of 16; warp 8 = TMA producer,
// warpgroups 0 and 1 = consumers (64 frames each, m64n256k16, the accumulator in 128 registers per thread), which release a stage once
// the wgmma group that read it has retired and finally multiply each row by its exact unscale factor 2^-(e_f + e_B) and store the
// accumulator TRANSPOSED ([column][frame]) so that lbs_skin_kernel (lanes = frames) reads contiguous bytes per vertex coordinate; the
// store goes through a shared-memory staging chunk per warpgroup, so that it leaves as 16-byte pieces of whole frame runs instead of
// scalars that half-fill their sectors.  8 stages x 24 KB = 192 KB of shared memory per CTA (+ 21 KB of staging): with 4 stages the
// blend alone runs as fast, but the iteration of 4 x 300 frame-persons, where the blend shares the GPU with the residual and backward
// kernels, is ~5 % slower.
// Persistent: the grid has one CTA per SM (the register file holds one), and CTA b runs tiles b, b + grid, ...  The stage ring runs on
// across tiles, so the producer fetches the next tile's first stages while the consumers store the current accumulator.  Tiles are
// numbered column-tile major (frame tile fastest): the CTAs that read one 448 KB basis column tile run at the same time, and the
// 18.6 MB basis leaves HBM about once per launch instead of once per frame tile.  A last frame tile with at most 64 frames is a half
// tile: both warpgroups take its 64 rows, each for 128 of the 256 columns (m64n128k16) -- same products, same K order.
constexpr int kTcStages = 8;
constexpr int kTcThreads = 288;           // warpgroups 0-1 consume, warp 8 produces
constexpr uint32_t kTcABytes = kTcAStageHalves * sizeof(__half);     // 8,192
constexpr uint32_t kTcBBytes = kTcBStageHalves * sizeof(__half);     // 16,384
constexpr size_t kTcRingBytes = (size_t)kTcStages * (kTcABytes + kTcBBytes) + 128;   // stages, then the full / empty barriers
constexpr size_t kTcSmemBytes = kTcRingBytes + 2 * (size_t)kTcOutCols * kTcOutPitch * sizeof(float);   // + a staging chunk per warpgroup

// Phase clock of the consumer warpgroups (tools/blend_phases_exp.py), experiment build only: each consumer thread adds the clock64
// cycles since its previous stamp to a phase; lane 0 of the first warp of each warpgroup adds the sums of its CTA at the end of a launch.
#ifdef GLAMR_EXPERIMENT
constexpr int kBlendPhaseCtas = 1024;
constexpr int kBlendPhases = 5;         // wait full | wgmma issue + retire wait | epilogue | other | tiles
__device__ unsigned long long g_blend_phases[kBlendPhaseCtas][2][kBlendPhases];
#define BLEND_CLOCK_INIT() long long bl_ph[kBlendPhases] = {}; long long bl_t = clock64()
#define BLEND_CLOCK(k) do { const long long bl_now = clock64(); bl_ph[k] += bl_now - bl_t; bl_t = bl_now; } while (0)
#define BLEND_CLOCK_TILE() (++bl_ph[kBlendPhases - 1])
#define BLEND_CLOCK_STORE() do { if ((warp & 3) == 0 && lane == 0 && blockIdx.x < kBlendPhaseCtas)                                     \
      for (int k = 0; k < kBlendPhases; ++k) atomicAdd(&g_blend_phases[blockIdx.x][g][k], (unsigned long long)bl_ph[k]); } while (0)
extern "C" int glamr_exp_blend_phases(long long* out) {    // the per-CTA sums of the blend launches since the last call, then zeroed
  void* p = nullptr;
  GLAMR_CUDA_TRY(cudaDeviceSynchronize());
  GLAMR_CUDA_TRY(cudaMemcpyFromSymbol(out, g_blend_phases, sizeof(g_blend_phases)));
  GLAMR_CUDA_TRY(cudaGetSymbolAddress(&p, g_blend_phases));
  GLAMR_CUDA_TRY(cudaMemset(p, 0, sizeof(g_blend_phases)));
  return GLAMR_OK;
}
#else
#define BLEND_CLOCK_INIT() do { } while (0)
#define BLEND_CLOCK(k) do { } while (0)
#define BLEND_CLOCK_TILE() do { } while (0)
#define BLEND_CLOCK_STORE() do { } while (0)
#endif

// bar.sync of the 128 threads of consumer warpgroup g on named barrier 1 + g (0 is __syncthreads); immediate ids, so that ptxas
// reserves 3 barriers rather than all 16
__device__ __forceinline__ void warpgroup_sync(int g) {
  if (g == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}

// mtile0 / mtiles: the 128-frame tiles [mtile0, mtile0 + mtiles) of this launch (the host launches them all, from mtile0 = 0);
// half_last: the last of them holds at most 64 frames; ntn: the 256-column tiles (the mesh's 81, plus the support columns when the
// skinning runs on the tensor cores)
__global__ void __launch_bounds__(kTcThreads, 1) lbs_blend_tc_kernel(SmplDev m, SmplWorkspace w, int mtile0, int mtiles, int half_last, int ntn) {
  extern __shared__ __align__(128) unsigned char tc_raw[];
  __half* As = reinterpret_cast<__half*>(tc_raw);                                 // [stages][hi | lo][2][128][8]
  __half* Bs = As + kTcStages * kTcAStageHalves;                                  // [stages][hi | lo][2][256][8]
  uint64_t* full = reinterpret_cast<uint64_t*>(Bs + kTcStages * kTcBStageHalves); // [stages]
  uint64_t* empty = full + kTcStages;                                             // [stages]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = ntn * mtiles;
  pdl_launch_dependents();
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kTcStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // empty: one arrival per consumer warp
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // the basis is a model constant: the first stages of the first tile are requested before this grid waits for the kernel that
      // writes the features
      {
        const __half* gB = m.tcB + (size_t)(blockIdx.x / mtiles) * kTcChunks * kTcBStageHalves;
        for (int c = 0; c < kTcStages; ++c) {
          mbar_expect_tx_only(&full[c], kTcBBytes);
          tma_bulk_g2s(Bs + c * kTcBStageHalves, gB + (size_t)c * kTcBStageHalves, kTcBBytes, &full[c]);
        }
      }
      pdl_wait();
      int q = 0;                                                                  // stage uses so far (all tiles)
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const __half* gA = w.tcA + (size_t)(mtile0 + t % mtiles) * kTcChunks * kTcAStageHalves;
        const __half* gB = m.tcB + (size_t)(t / mtiles) * kTcChunks * kTcBStageHalves;
        for (int c = 0; c < kTcChunks; ++c, ++q) {
          const int s = q % kTcStages;
          if (q >= kTcStages) {
            mbar_wait(&empty[s], ((q / kTcStages) - 1) & 1);                     // the wgmma groups that read this stage have retired
            mbar_expect_tx(&full[s], kTcABytes + kTcBBytes);
            tma_bulk_g2s(Bs + s * kTcBStageHalves, gB + (size_t)c * kTcBStageHalves, kTcBBytes, &full[s]);
          } else {
            mbar_expect_tx(&full[s], kTcABytes);
          }
          tma_bulk_g2s(As + s * kTcAStageHalves, gA + (size_t)c * kTcAStageHalves, kTcABytes, &full[s]);
        }
      }
    }
    return;
  }
  // ---- consumers: warpgroup g owns frames 64 g .. 64 g + 63 of a full tile, columns 128 g .. 128 g + 127 of a half tile
  const int g = warp >> 2;
  float acc[kTcN / 2];
  float (&acc_half)[kTcN / 4] = *reinterpret_cast<float (*)[kTcN / 4]>(acc);
  float* const vpb = vp_buffer(w);
  const size_t cstride = w.vp_tiled ? (size_t)kSkF : (size_t)w.mpad;
  int q = 0;
  BLEND_CLOCK_INIT();
#pragma unroll 1
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int ntile = t / mtiles, mt = t % mtiles, mtile = mtile0 + mt;
    const bool half = half_last && mt == mtiles - 1;
    // full tile: A rows 64 g.., all 256 columns of B; half tile: A rows 0..63, B columns 128 g..
    const int aoff = half ? 0 : g * 64 * 8, boff = half ? g * 128 * 8 : 0;
    auto mainloop = [&](auto& d, auto mma) {
#pragma unroll 1
      for (int c = 0; c < kTcChunks; ++c, ++q) {
        const int s = q % kTcStages;
        BLEND_CLOCK(3);
        mbar_wait(&full[s], (q / kTcStages) & 1);
        BLEND_CLOCK(0);
        const __half* a = As + s * kTcAStageHalves + aoff;
        const __half* b = Bs + s * kTcBStageHalves + boff;
        const uint64_t dah = wgmma_desc_kmajor_noswizzle(a, kTcM), dal = wgmma_desc_kmajor_noswizzle(a + kTcAStageHalves / 2, kTcM);
        const uint64_t dbh = wgmma_desc_kmajor_noswizzle(b, kTcN), dbl = wgmma_desc_kmajor_noswizzle(b + kTcBStageHalves / 2, kTcN);
        wgmma_fence();
        mma(d, dah, dbh, c > 0 ? 1u : 0u);
        mma(d, dal, dbh, 1u);
        mma(d, dah, dbl, 1u);
        wgmma_commit();
        wgmma_wait<1>();                                                          // the group of the previous stage use has retired
        if (c > 0 && lane == 0) mbar_arrive(&empty[(q - 1) % kTcStages]);
        BLEND_CLOCK(1);
      }
      wgmma_wait<0>();
      wgmma_fence_acc(d);
      BLEND_CLOCK(1);
    };
    if (half) mainloop(acc_half, [](float (&d)[kTcN / 4], uint64_t da, uint64_t db, uint32_t acc_in) { wgmma_m64n128k16_f16(d, da, db, acc_in); });
    else mainloop(acc, [](float (&d)[kTcN / 2], uint64_t da, uint64_t db, uint32_t acc_in) { wgmma_m64n256k16_f16(d, da, db, acc_in); });
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[(q - 1) % kTcStages]);                     // the tile's last stage: the producer moves on
    // ---- epilogue: d[4 i + 2 h + e] = D[16 (warp % 4) + lane / 4 + 8 h][8 i + 2 (lane % 4) + e], times the row's unscale factor.
    // The warpgroup stages kTcOutCols columns at a time in shared memory ([column][frame]) and stores them as 16-byte pieces of 4
    // consecutive frames: it starts at a multiple of 64 frames, so every piece lies inside one 20-frame group and is 16-byte aligned in
    // both layouts.  v_posed^T [column][mpad]: a column's 64 frames are one 256-byte run, piece p of the chunk is frame piece p % 16 of
    // column p / 16.  Frame-tiled [frame / 20][column][frame % 20] (tensor-core skinning): the chunk's pieces run group by group, and
    // inside a group column by column over the group's frames the warpgroup holds, so that a group the warpgroup holds whole goes out
    // as one contiguous run of kTcOutCols x 80 bytes.
    const int f0 = mtile * kTcM + (half ? 0 : g * 64);                            // the warpgroup's first frame
    const int col0 = ntile * kTcN + (half ? g * 128 : 0);
    const int ncols = half ? kTcN / 2 : kTcN;
    const int rl = (warp & 3) * 16 + (lane >> 2);                                 // the fragment's row for h = 0
    float unscale[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) unscale[h] = w.tcUnscale[f0 + rl + 8 * h] * m.tcB_unscale;   // 2^-(e_f + e_B): exact
    // the pieces this thread stores in every chunk: their offsets in the staging chunk and in v_posed at the chunk's first column
    constexpr int kPieces = kTcOutCols * 16 / 128;
    int soff[kPieces];
    size_t goff[kPieces];
#pragma unroll
    for (int j = 0; j < kPieces; ++j) {
      const int p = (tid & 127) + 128 * j;
      int fq, c;                                                                  // frame piece 0..15 of the warpgroup, column of the chunk
      if (w.vp_tiled) {
        const int q0 = f0 / 4, grp = (q0 + p / kTcOutCols) / 5;                   // the 20-frame group whose run holds p
        const int qa = max(5 * grp - q0, 0), qn = min(5 * grp + 5 - q0, 16) - qa; // the warpgroup's pieces qa .. qa + qn - 1 of it
        const int pg = p - kTcOutCols * qa;
        c = pg / qn;
        fq = qa + pg - c * qn;
      } else {
        fq = p & 15;
        c = p >> 4;
      }
      const int f = f0 + 4 * fq;
      soff[j] = c * kTcOutPitch + 4 * fq;
      goff[j] = w.vp_tiled ? ((size_t)(f / kSkF) * w.vp_cols + (size_t)(col0 + c)) * kSkF + f % kSkF : (size_t)(col0 + c) * w.mpad + f;
    }
    float* const stage = reinterpret_cast<float*>(tc_raw + kTcRingBytes) + g * kTcOutCols * kTcOutPitch;
#pragma unroll
    for (int k = 0; k < kTcN / kTcOutCols; ++k) {
      if (kTcOutCols * k < ncols) {
        warpgroup_sync(g);                                                    // the previous chunk has been read
#pragma unroll
        for (int i = 0; i < kTcOutCols / 8; ++i)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              stage[(8 * i + 2 * (lane & 3) + e) * kTcOutPitch + rl + 8 * h] = acc[4 * (k * kTcOutCols / 8 + i) + 2 * h + e] * unscale[h];
        warpgroup_sync(g);
        float* const out = vpb + (size_t)(k * kTcOutCols) * cstride;
#pragma unroll
        for (int j = 0; j < kPieces; ++j)
          *reinterpret_cast<float4*>(out + goff[j]) = *reinterpret_cast<const float4*>(stage + soff[j]);
      }
    }
    BLEND_CLOCK(2);
    BLEND_CLOCK_TILE();
  }
  BLEND_CLOCK_STORE();
}

// Skinning of the blended vertices (lbs.py:273-284): CTA = 128 vertices x 32 frames, warp = 32 vertices, lane = frame.
// The tile's relative joint transforms [24][32][12] arrive by one bulk TMA copy; joint indices / weights are warp-uniform
// (prefetched one vertex per lane, broadcast by shuffles); v_posed comes from the transposed blend output with one coalesced
// 128-byte load per vertex coordinate; a lane reads its frame's A_j with three conflict-free LDS.128.
constexpr size_t kSkinSmemBytes = (size_t)kATileFloats * sizeof(float) + 16;
template <int KREG>
__global__ void __launch_bounds__(kLbsThreads) lbs_skin_kernel(SmplDev m, int n_begin, int n_end, SmplWorkspace w, float* __restrict__ vertices) {
  extern __shared__ __align__(128) unsigned char skin_raw[];
  float* As = reinterpret_cast<float*>(skin_raw);
  uint64_t* abar = reinterpret_cast<uint64_t*>(As + kATileFloats);
  const int tid = threadIdx.x, lane = tid & 31;
  const int vtile = blockIdx.x;
  const int f0 = n_begin + blockIdx.y * kFramesPerCta;
  pdl_launch_dependents();
  if (tid == 0) {
    mbar_init(abar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  const int vbase = (tid >> 5) * 32;
  const int gvl = min(vtile * kVTile + vbase + lane, kVPad - 1);
  float4 my_w = make_float4(0.f, 0.f, 0.f, 0.f);
  unsigned int my_j = 0;
  if (KREG > 0) {
    my_w = *reinterpret_cast<const float4*>(m.skin_w + (size_t)gvl * 4);
    my_j = *reinterpret_cast<const unsigned int*>(m.skin_j + (size_t)gvl * 4);
  }
  const int my_ci = m.compact_of_vertex[gvl];
  pdl_wait();                                   // A (pose_prep) and vpT (blend GEMM) are written by preceding kernels
  if (tid == 0) {
    mbar_expect_tx(abar, (uint32_t)kATileFloats * sizeof(float));
    tma_bulk_g2s(As, w.A + (size_t)(f0 >> 5) * kATileFloats, (uint32_t)kATileFloats * sizeof(float), abar);
  }
  const int fr = lane;
  const int n = f0 + fr;
  const bool n_ok = n < n_end;
  const float* vp = vp_buffer(w) + (size_t)(vtile * kVTile + vbase) * 3 * w.mpad + n;      // n < mpad (frames padded to 128)
  mbar_wait(abar, 0);
  constexpr int U = 4;
#pragma unroll 1
  for (int i0 = 0; i0 < 32; i0 += U) {
    float x[U], y[U], z[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int gv = vtile * kVTile + vbase + i0 + u;
      const bool ok = gv < kV;
      const float* q = vp + (size_t)(i0 + u) * 3 * w.mpad;
      x[u] = ok ? q[0] : 0.0f;
      y[u] = ok ? q[w.mpad] : 0.0f;
      z[u] = ok ? q[2 * (size_t)w.mpad] : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u;
      const int gv = vtile * kVTile + vbase + i;
      if (gv >= kV) break;
      const int ci = __shfl_sync(0xffffffffu, my_ci, i);
      float T[12];
      if (KREG > 0) {
        const float w0 = __shfl_sync(0xffffffffu, my_w.x, i), w1 = __shfl_sync(0xffffffffu, my_w.y, i);
        const float w2 = __shfl_sync(0xffffffffu, my_w.z, i), w3 = __shfl_sync(0xffffffffu, my_w.w, i);
        const unsigned int jj = __shfl_sync(0xffffffffu, my_j, i);
        const float4* a0 = reinterpret_cast<const float4*>(As + ((jj & 0xff) * 32 + fr) * 12);
        const float4* a1 = reinterpret_cast<const float4*>(As + (((jj >> 8) & 0xff) * 32 + fr) * 12);
        const float4* a2 = reinterpret_cast<const float4*>(As + (((jj >> 16) & 0xff) * 32 + fr) * 12);
        const float4* a3 = reinterpret_cast<const float4*>(As + (((jj >> 24) & 0xff) * 32 + fr) * 12);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const float4 q0 = a0[r], q1 = a1[r], q2 = a2[r], q3 = a3[r];
          T[4 * r + 0] = fmaf(w3, q3.x, fmaf(w2, q2.x, fmaf(w1, q1.x, w0 * q0.x)));
          T[4 * r + 1] = fmaf(w3, q3.y, fmaf(w2, q2.y, fmaf(w1, q1.y, w0 * q0.y)));
          T[4 * r + 2] = fmaf(w3, q3.z, fmaf(w2, q2.z, fmaf(w1, q1.z, w0 * q0.z)));
          T[4 * r + 3] = fmaf(w3, q3.w, fmaf(w2, q2.w, fmaf(w1, q1.w, w0 * q0.w)));
        }
      } else {
#pragma unroll
        for (int k = 0; k < 12; ++k) T[k] = 0.0f;
        for (int sidx = 0; sidx < m.K; ++sidx) {
          const int jj = m.skin_j[(size_t)gv * m.K + sidx];
          const float wt = m.skin_w[(size_t)gv * m.K + sidx];
          const float* a = As + (jj * 32 + fr) * 12;
#pragma unroll
          for (int k = 0; k < 12; ++k) T[k] = fmaf(wt, a[k], T[k]);
        }
      }
      const float ox = fmaf(T[0], x[u], fmaf(T[1], y[u], fmaf(T[2], z[u], T[3])));
      const float oy = fmaf(T[4], x[u], fmaf(T[5], y[u], fmaf(T[6], z[u], T[7])));
      const float oz = fmaf(T[8], x[u], fmaf(T[9], y[u], fmaf(T[10], z[u], T[11])));
      if (n_ok) {
        if (vertices) {
          float* o = vertices + ((size_t)n * kV + gv) * 3;
          o[0] = ox; o[1] = oy; o[2] = oz;
        }
        if (ci >= 0) {
          float* o = w.vcompact + ((size_t)n * m.S + ci) * 3;
          o[0] = ox; o[1] = oy; o[2] = oz;
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------ tensor-core skinning
// lbs.py:273-284 as a GEMM with a fused epilogue.  The blended transform of vertex v in frame f is T[v][f] = sum_j W[v][j] A_j[f]
// (12 numbers), i.e. [128 vertices x 24 joints] x [24 joints x (20 frames x 12)] per CTA: two consumer warpgroups of 64 vertices,
// each m64n240k8 with the accumulator in 120 registers per thread, K = 24 in three steps, 3xTF32 (hi*hi + lo*hi + hi*lo; the
// blend's split, but in tf32).  Both operands are pre-tiled wgmma images (W: model constant built at glamr_smpl_create; A: written by pose_prep_frame), so
// the whole operand traffic of a CTA is three bulk copies: W image 24 KB, A image 45 KB, and the 128 x 20 v_posed block 30 KB (the
// blend stores v_posed frame-tiled for this).  Epilogue straight from the accumulator fragment: the quad of lanes that holds a
// vertex row owns all 24 columns of a frame pair; each lane dots its column pairs with (x, y) or (z, 1) of v_posed and one
// shuffle with the neighbouring lane completes an output coordinate -- no shared-memory traffic for the joint transforms, which
// bounded the SIMT skinning (12 LDS.128 per vertex-frame).  The epilogue has no branch before a row's stores: written with a
// lane-dependent branch and a shuffle and store check per output, every output waited on the one before and the epilogue took
// ~70 % of an item (tools/skin_phases_exp.py).  warp 8 = producer.
// A launch skins the vertex tiles [vt0, vt1): mesh tiles (< kNVTiles) store into `vertices` when it is given, support tiles (the support
// vertices again, slot by slot, with their copied weights and v_posed columns; smpl_model.cuh) into vcompact.  The optimiser skins the
// support tiles on its critical path and the mesh tiles beside it; a mesh-only or support-only launch does exactly what the same items of
// an all-tiles launch do, so a support vertex comes out bit for bit as its mesh vertex.
// Persistent: a work item is one (vertex tile, frame tile) pair, numbered vertex-tile major, and CTA b of a grid of at most one CTA per
// SM (the register file holds one) runs the contiguous item range [b items / grid, (b + 1) items / grid).  Every CTA gets within one
// item of the average, which a fixed number of frame tiles per CTA could not give for every n, and its range spans at most two vertex
// tiles (fewer items than frame tiles per CTA), so the W image is fetched at most twice.  The A image and the v_posed block are
// double-buffered: both operands of the next item land while the current one runs, so per item the CTA waits for neither; one buffered
// item alone would leave each item's copy latency exposed, which bounded the kernel.  174 KB of shared memory per CTA.
constexpr uint32_t kSkWBytes = kSkWImageFloats * sizeof(float);       // 24,576
constexpr uint32_t kSkBBytes = kSkBImageFloats * sizeof(float);       // 46,080
constexpr uint32_t kSkVBytes = kSkVpTileFloats * sizeof(float);       // 30,720
constexpr size_t kSkinTcSmemBytes = (size_t)kSkWBytes + 2 * kSkBBytes + 2 * kSkVBytes + 128;

constexpr int kSkinTcThreads = 288;     // warpgroups 0-1 consume (64 vertices each), warp 8 produces

// Phase clock of the consumer warpgroups (tools/skin_phases_exp.py), experiment build only: each consumer thread adds the clock64
// cycles since its previous stamp to a phase; lane 0 of the first warp of each warpgroup stores the sums of its CTA at the end.
#ifdef GLAMR_EXPERIMENT
constexpr int kSkinPhaseCtas = 1024;
constexpr int kSkinPhases = 6;          // wait full_b | wgmma issue + retire wait | wait full_v | epilogue | other | items
__device__ long long g_skin_phases[kSkinPhaseCtas][2][kSkinPhases];
#define SKIN_CLOCK_INIT() long long sk_ph[kSkinPhases] = {}; long long sk_t = clock64()
#define SKIN_CLOCK(k) do { const long long sk_now = clock64(); sk_ph[k] += sk_now - sk_t; sk_t = sk_now; } while (0)
#define SKIN_CLOCK_STORE(items) do { sk_ph[kSkinPhases - 1] = (items);                                                              \
    if ((warp & 3) == 0 && lane == 0 && blockIdx.x < kSkinPhaseCtas)                                                               \
      for (int k = 0; k < kSkinPhases; ++k) g_skin_phases[blockIdx.x][g][k] = sk_ph[k]; } while (0)
extern "C" int glamr_exp_skin_phases(long long* out) {     // the per-CTA sums of the skinning launches since the last call, then zeroed
  void* p = nullptr;
  GLAMR_CUDA_TRY(cudaDeviceSynchronize());
  GLAMR_CUDA_TRY(cudaMemcpyFromSymbol(out, g_skin_phases, sizeof(g_skin_phases)));
  GLAMR_CUDA_TRY(cudaGetSymbolAddress(&p, g_skin_phases));
  GLAMR_CUDA_TRY(cudaMemset(p, 0, sizeof(g_skin_phases)));
  return GLAMR_OK;
}
#else
#define SKIN_CLOCK_INIT() do { } while (0)
#define SKIN_CLOCK(k) do { } while (0)
#define SKIN_CLOCK_STORE(items) do { } while (0)
#endif

__global__ void __launch_bounds__(kSkinTcThreads, 1) lbs_skin_tc_kernel(SmplDev m, int n, SmplWorkspace w, float* __restrict__ vertices,
                                                                        int vt0, int vt1) {
  extern __shared__ __align__(128) unsigned char sk_raw[];
  float* Ws = reinterpret_cast<float*>(sk_raw);                       // [hi | lo][6][128][4]
  float* Bs = Ws + kSkWImageFloats;                                   // [2][hi | lo][6][240][4]
  float* Vs = Bs + 2 * kSkBImageFloats;                               // [2][384 rows = vertex * 3 + coordinate][20 frames]
  uint64_t* full_w = reinterpret_cast<uint64_t*>(Vs + 2 * kSkVpTileFloats);
  uint64_t* full_b = full_w + 1;          // [2] A image (and, when the vertex tile changes, the W image) of the item has landed
  uint64_t* b_empty = full_w + 3;         // [2] the 8 consumer warps' wgmmas no longer read this A image (nor Ws)
  uint64_t* full_v = full_w + 5;          // [2] v_posed block has landed
  uint64_t* v_empty = full_w + 7;         // [2] the 8 consumer warps are done with the v_posed block
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nft = (n + kSkF - 1) / kSkF;
  const int items = (vt1 - vt0) * nft;
  const int i0 = (int)((long long)blockIdx.x * items / gridDim.x), i1 = (int)((long long)(blockIdx.x + 1) * items / gridDim.x);
  pdl_launch_dependents();
  if (tid == 0) {
    mbar_init(full_w, 1);
    for (int b = 0; b < 2; ++b) {
      mbar_init(&full_b[b], 1);
      mbar_init(&b_empty[b], 8);
      mbar_init(&full_v[b], 1);
      mbar_init(&v_empty[b], 8);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(full_w, kSkWBytes);
      tma_bulk_g2s(Ws, m.skW + (size_t)(vt0 + i0 / nft) * kSkWImageFloats, kSkWBytes, full_w);   // model constant: before the dependency wait
      pdl_wait();                                                                           // skB (pose prep) and v_posed (blend) below
      const float* const vpb = vp_buffer(w);
      for (int i = i0, it = 0; i < i1; ++i, ++it) {
        const int vtile = vt0 + i / nft, ftile = i - (vtile - vt0) * nft, vb = it & 1;
        const bool new_w = it > 0 && ftile == 0;                                            // the range crossed into the next vertex tile
        if (it >= 2) mbar_wait(&b_empty[vb], ((it - 2) >> 1) & 1);
        if (new_w) mbar_wait(&b_empty[vb ^ 1], ((it - 1) >> 1) & 1);                       // Ws is read until the previous item's wgmmas retire
        mbar_expect_tx(&full_b[vb], kSkBBytes + (new_w ? kSkWBytes : 0u));
        tma_bulk_g2s(Bs + vb * kSkBImageFloats, w.skB + (size_t)ftile * kSkBImageFloats, kSkBBytes, &full_b[vb]);
        if (new_w) tma_bulk_g2s(Ws, m.skW + (size_t)vtile * kSkWImageFloats, kSkWBytes, &full_b[vb]);
        if (it >= 2) mbar_wait(&v_empty[vb], ((it - 2) >> 1) & 1);
        mbar_expect_tx(&full_v[vb], kSkVBytes);
        tma_bulk_g2s(Vs + vb * kSkVpTileFloats, vpb + ((size_t)ftile * w.vp_cols + (size_t)vtile * kTileCols) * kSkF, kSkVBytes, &full_v[vb]);
      }
    }
    return;
  }
  // ---- consumers: warpgroup g owns vertices 64 g .. 64 g + 63 of the tile
  const int g = warp >> 2, q = lane & 3;
  // column pair j of a frame pair (24 columns) this lane holds: 8 j + 2 q = 12 fr + 4 row + (0: x, y | 2: z, 1)
  int jf[3], jrow[3];
  bool jxy[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int c0 = 8 * j + 2 * q;
    jf[j] = c0 >= 12 ? 1 : 0;
    jrow[j] = (c0 - 12 * jf[j]) >> 2;
    jxy[j] = (c0 & 3) == 0;
  }
  // the outputs this lane stores after the shuffles: even lanes j = 0 and 1, odd lanes j = 2 (frame offset sf, transform row srow)
  const bool odd = (q & 1) == 1;
  const int sf[2] = {odd ? jf[2] : jf[0], jf[1]}, srow[2] = {odd ? jrow[2] : jrow[0], jrow[1]};
  SKIN_CLOCK_INIT();
  mbar_wait(full_w, 0);
  for (int i = i0, it = 0; i < i1; ++i, ++it) {
    const int vtile = vt0 + i / nft, ftile = i - (vtile - vt0) * nft, vb = it & 1;
    // the output array of the tile (nullptr: stores nothing), its stride between frames and the row of each accumulator row of this
    // thread (-1: none)
    const bool sup = vtile >= kNVTiles;
    float* const out = sup ? w.vcompact : vertices;
    const int fstride = sup ? m.S * 3 : kV * 3;
    int orow[2];
    const float* vrow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int vl = g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;   // accumulator rows of this thread
      const int v = (vtile - (sup ? kNVTiles : 0)) * kVTile + vl;      // support slot or mesh vertex
      orow[h] = out && v < (sup ? m.S : kV) ? v * 3 : -1;
      vrow[h] = Vs + vb * kSkVpTileFloats + (size_t)vl * 3 * kSkF;
    }
    SKIN_CLOCK(4);
    mbar_wait(&full_b[vb], (it >> 1) & 1);
    SKIN_CLOCK(0);
    float acc[kSkN / 2];
#pragma unroll
    for (int k = 0; k < kSkN / 2; ++k) acc[k] = 0.0f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < kNJ / 8; ++c) {
      const float* a = Ws + c * 2 * kVTile * 4 + g * 64 * 4;
      const float* b = Bs + vb * kSkBImageFloats + c * 2 * kSkN * 4;
      const uint64_t dah = wgmma_desc_kmajor_noswizzle(a, kVTile), dal = wgmma_desc_kmajor_noswizzle(a + kSkWHalf, kVTile);
      const uint64_t dbh = wgmma_desc_kmajor_noswizzle(b, kSkN), dbl = wgmma_desc_kmajor_noswizzle(b + kSkBHalf, kSkN);
      wgmma_m64n240k8_tf32(acc, dah, dbh, c > 0 ? 1u : 0u);
      wgmma_m64n240k8_tf32(acc, dal, dbh, 1u);
      wgmma_m64n240k8_tf32(acc, dah, dbl, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    SKIN_CLOCK(1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&b_empty[vb]);
    SKIN_CLOCK(4);
    mbar_wait(&full_v[vb], (it >> 1) & 1);
    SKIN_CLOCK(2);
    // Epilogue, straight-line: per frame pair x, y, z of frames 2 p and 2 p + 1 are loaded once and lane-dependent selects stand in for
    // branches, and a row is stored after all its outputs are computed, so the compiler can overlap the frame pairs; per output the same
    // arithmetic as fmaf(t0, x, t1 * y) + fmaf(t0, z, t1) (t1 * 1.0f is exact).  In the optimiser the mesh rows store nothing.
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2* const vr = reinterpret_cast<const float2*>(vrow[h]);   // [coordinate][10 frame pairs]
      float o0[kSkF / 2], o1[kSkF / 2];                                     // the outputs this lane stores: j = 0 | 2 and j = 1
#pragma unroll
      for (int p = 0; p < kSkF / 2; ++p) {
        const float2 x = vr[p], y = vr[kSkF / 2 + p], z = vr[kSkF + p];
        float part[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float t0 = acc[4 * (3 * p + j) + 2 * h], t1 = acc[4 * (3 * p + j) + 2 * h + 1];
          const float xf = jf[j] ? x.y : x.x, yf = jf[j] ? y.y : y.x, zf = jf[j] ? z.y : z.x;
          part[j] = fmaf(t0, jxy[j] ? xf : zf, t1 * (jxy[j] ? yf : 1.0f));
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) part[j] += __shfl_xor_sync(0xffffffffu, part[j], 1);   // the neighbouring lane holds the other half of the row
        o0[p] = odd ? part[2] : part[0];
        o1[p] = part[1];
      }
      if (orow[h] >= 0) {
#pragma unroll
        for (int p = 0; p < kSkF / 2; ++p)
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (k == 1 && odd) continue;                               // even lanes store j = 0, 1; odd lanes j = 2
            const int fl = ftile * kSkF + 2 * p + sf[k];               // local frame-person index
            if (fl < n) out[(size_t)fl * fstride + orow[h] + srow[k]] = k ? o1[p] : o0[p];
          }
      }
    }
    SKIN_CLOCK(3);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[vb]);
  }
  SKIN_CLOCK_STORE(i1 - i0);
}

// ------------------------------------------------------------------------------------------------ joints_finalize
// One warp per frame-person: gather the mapped joints from [24 LBS | picks | extra regressed], re-root at joint 0
// and apply scale / root translation   (lib/models/smpl.py:299-315)
__global__ void __launch_bounds__(128) joints_finalize_kernel(SmplDev m, int n, int orig_joints, const float* __restrict__ root_trans,
                                                              const float* __restrict__ root_scale, SmplWorkspace w,
                                                              float* __restrict__ joints) {
  const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (f >= n) return;
  const int n_out = orig_joints ? kNJ : m.n_map;
  float root[3];
  raw_joint(m, w, f, orig_joints ? 0 : m.joint_map[0], root);
  if (lane == 0) {
    w.root_raw[f * 3 + 0] = root[0]; w.root_raw[f * 3 + 1] = root[1]; w.root_raw[f * 3 + 2] = root[2];
  }
  const float sc = (root_trans && root_scale) ? root_scale[f] : 1.0f;
  for (int k = lane; k < n_out; k += 32) {
    float v[3];
    raw_joint(m, w, f, orig_joints ? k : m.joint_map[k], v);
    float* o = joints + ((size_t)f * n_out + k) * 3;
    if (root_trans) {
      o[0] = (v[0] - root[0]) * sc + root_trans[f * 3 + 0];
      o[1] = (v[1] - root[1]) * sc + root_trans[f * 3 + 1];
      o[2] = (v[2] - root[2]) * sc + root_trans[f * 3 + 2];
    } else {
      o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
    }
  }
}

__global__ void reroot_vertices_kernel(int n, const float* __restrict__ root_raw, const float* __restrict__ root_trans,
                                       const float* __restrict__ root_scale, float* __restrict__ vertices) {
  const size_t total = (size_t)n * kV * 3;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int f = (int)(e / (kV * 3));
    const int c = (int)(e % 3);
    const float sc = root_scale ? root_scale[f] : 1.0f;
    vertices[e] = (vertices[e] - root_raw[f * 3 + c]) * sc + root_trans[f * 3 + c];
  }
}

// fk-only joints (SMPL.get_joints): re-root the posed LBS joints
__global__ void fk24_finalize_kernel(int n, const float* __restrict__ jposed, const float* __restrict__ root_trans,
                                     const float* __restrict__ root_scale, float* __restrict__ joints) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * kNJ * 3) return;
  const int f = e / (kNJ * 3), c = e % 3;
  float v = jposed[e];
  if (root_trans) {
    const float sc = root_scale ? root_scale[f] : 1.0f;
    v = (v - jposed[(size_t)f * kNJ * 3 + c]) * sc + root_trans[f * 3 + c];
  }
  joints[e] = v;
}

// ------------------------------------------------------------------------------------------------ launches
int launch_pose_prep(const SmplDev& m, int n, const float* orient, const float* body_pose, const float* betas, int use_betas,
                     const SmplWorkspace& w, cudaStream_t s, bool pdl) {
  if (n <= 0) return GLAMR_OK;
  const int blocks = (n + 3) / 4;
  if (pdl) {
    GLAMR_CUDA_TRY(launch_pdl(2, pose_prep_kernel, dim3(blocks), dim3(128), 0, s, m, n, orient, body_pose, betas, use_betas, w));
    return GLAMR_OK;
  }
  pose_prep_kernel<<<blocks, 128, 0, s>>>(m, n, orient, body_pose, betas, use_betas, w);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

// pdl: launch with the programmatic-serialization attribute.  Only for callers whose betas are long-lived constants
// (the optimiser): the kernel reads betas / shapedirs / posedirs BEFORE it waits for the preceding grid.
// An SM runs with ONE L1 / shared-memory split at a time.  blend_features_kernel / pose_prep_kernel have no dynamic shared memory, so by
// default they run with a small shared-memory split, and the GEMM kernel that follows each of them in its stream (2 x 96-101 KB per SM)
// can only be placed on an SM after the small kernel's CTAs have drained and the SM has been re-configured.  Asking for the maximal
// shared-memory split on the small SMPL kernels too removes that hand-over: 193.0 -> 157.4 us per iteration at 4 x 300 frame-persons
// (no change at 1 x 300).  The optimiser's own small kernels lose more from the smaller L1 than they gain (+6 us at 1 x 300), so they
// keep the default split.
static int lbs_set_attrs() {
  static bool attrs = false;
  if (!attrs) {
    attrs = true;
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_blend_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_skin_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(blend_features_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(pose_prep_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_blend_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_skin_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSkinSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_skin_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSkinSmemBytes));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_skin_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSkinTcSmemBytes));
  }
  return GLAMR_OK;
}
// SMs of the device: the persistent LBS GEMM kernels launch at most one CTA per SM
int smpl_device_sms() {
  static int sms = 0;
  if (sms <= 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}
// the blend GEMM over all 128-frame tiles of n frame-persons
static int launch_blend_gemm(const SmplDev& m, int n, const SmplWorkspace& w, cudaStream_t s, bool pdl) {
  const int mtiles = (n + kTcM - 1) / kTcM;
  const int half_last = (n - (mtiles - 1) * kTcM <= kTcM / 2) ? 1 : 0;
  const int ntn = w.vp_tiled ? m.tc_ntiles : kTcNTiles;     // the support columns feed the tensor-core skinning only
  const dim3 grid(min(smpl_device_sms(), ntn * mtiles));
  if (pdl) {
    GLAMR_CUDA_TRY(launch_pdl(4, lbs_blend_tc_kernel, grid, dim3(kTcThreads), kTcSmemBytes, s, m, w, 0, mtiles, half_last, ntn));
    return GLAMR_OK;
  }
  lbs_blend_tc_kernel<<<grid, kTcThreads, kTcSmemBytes, s>>>(m, w, 0, mtiles, half_last, ntn);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
// vertex tiles [vt0, vt1) on at most max_ctas CTAs
static int launch_skin_tc(const SmplDev& m, int n, const SmplWorkspace& w, float* vertices, cudaStream_t s, bool pdl, int vt0, int vt1,
                          int max_ctas) {
  if (vt1 <= vt0) return GLAMR_OK;
  const dim3 grid(max(1, min(max_ctas, (vt1 - vt0) * ((n + kSkF - 1) / kSkF))));
  if (pdl) {
    GLAMR_CUDA_TRY(launch_pdl(4, lbs_skin_tc_kernel, grid, dim3(kSkinTcThreads), kSkinTcSmemBytes, s, m, n, w, vertices, vt0, vt1));
    return GLAMR_OK;
  }
  lbs_skin_tc_kernel<<<grid, kSkinTcThreads, kSkinTcSmemBytes, s>>>(m, n, w, vertices, vt0, vt1);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
// blend features + blend GEMM for local frame-persons [0, n): v_posed (transposed) of the workspace
// features: (re)build the A operand; gemm: run the GEMM
int launch_blend(const SmplDev& m, int n, const float* body_pose, const float* betas, const SmplWorkspace& w, cudaStream_t s, bool features,
                 bool gemm) {
  if (n <= 0) return GLAMR_OK;
  int rc;
  if ((rc = lbs_set_attrs())) return rc;
  if (features) {
    blend_features_kernel<<<(n + 3) / 4, 128, 0, s>>>(n, body_pose, betas, w);
    GLAMR_LAUNCH_CHECK();
  }
  if (gemm) return launch_blend_gemm(m, n, w, s, false);
  return GLAMR_OK;
}
// skinning of local frame-persons [0, n) from the workspace's v_posed and A
int launch_skin(const SmplDev& m, int n, const SmplWorkspace& w, float* vertices, cudaStream_t s, int vt0, int vt1, int max_ctas) {
  if (n <= 0) return GLAMR_OK;
  int rc;
  if ((rc = lbs_set_attrs())) return rc;
  if (w.vp_tiled) return launch_skin_tc(m, n, w, vertices, s, false, vt0, vt1, max_ctas);
  dim3 grid(kNVTiles, (n + kFramesPerCta - 1) / kFramesPerCta);
  if (m.K == 4) lbs_skin_kernel<4><<<grid, kLbsThreads, kSkinSmemBytes, s>>>(m, 0, n, w, vertices);
  else lbs_skin_kernel<0><<<grid, kLbsThreads, kSkinSmemBytes, s>>>(m, 0, n, w, vertices);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

static int g_lbs_path = -1;
int lbs_path() {
  if (g_lbs_path < 0) {
    const char* e = getenv("GLAMR_LBS_PATH");
    g_lbs_path = e ? (strcmp(e, "tc") == 0 ? 2 : strcmp(e, "tcblend") == 0 ? 1 : 0) : GLAMR_DEFAULT_LBS_TC;
  }
  return g_lbs_path;
}
int lbs_kernel_count(const SmplDev& m) { return (lbs_path() >= 1 && m.tcB) ? 2 : 1; }

int launch_lbs(const SmplDev& m, int n_begin, int n_end, const float* betas, const SmplWorkspace& w, float* vertices, cudaStream_t s,
               bool pdl) {
  if (n_end <= n_begin) return GLAMR_OK;
  if (n_begin % kFramesPerCta != 0) return GLAMR_EINVAL;   // the tile-major scratch is indexed by whole frame tiles
  dim3 grid(kNVTiles, (n_end - n_begin + kFramesPerCta - 1) / kFramesPerCta);
  const int path = lbs_path();             // >= 1: tensor-core blend GEMM + skinning kernel (2: tensor-core skinning), 0: the one-kernel FP32 SIMT path
  {
    const int rc = lbs_set_attrs();
    if (rc) return rc;
  }
  if (path >= 1 && m.tcB && w.tcA && n_begin == 0) {
    int rc;
    if ((rc = launch_blend_gemm(m, n_end, w, s, pdl))) return rc;
    // mesh and support tiles in one launch: the joints come from vcompact
    if (w.vp_tiled) return launch_skin_tc(m, n_end, w, vertices, s, pdl, 0, m.sk_tiles, smpl_device_sms());
    if (pdl) {
      if (m.K == 4) GLAMR_CUDA_TRY(launch_pdl(4, lbs_skin_kernel<4>, grid, dim3(kLbsThreads), kSkinSmemBytes, s, m, n_begin, n_end, w, vertices));
      else GLAMR_CUDA_TRY(launch_pdl(4, lbs_skin_kernel<0>, grid, dim3(kLbsThreads), kSkinSmemBytes, s, m, n_begin, n_end, w, vertices));
    } else {
      if (m.K == 4) lbs_skin_kernel<4><<<grid, kLbsThreads, kSkinSmemBytes, s>>>(m, n_begin, n_end, w, vertices);
      else lbs_skin_kernel<0><<<grid, kLbsThreads, kSkinSmemBytes, s>>>(m, n_begin, n_end, w, vertices);
      GLAMR_LAUNCH_CHECK();
    }
    return GLAMR_OK;
  }
  static int stages = 0, dbg = 0;
  if (!stages) {
    const char* e = getenv("GLAMR_LBS_STAGES");
    stages = (e && atoi(e) == 4) ? 4 : 3;
#ifdef GLAMR_EXPERIMENT
    const char* d = getenv("GLAMR_LBS_DEBUG");      // experiment build only: bit0 skips the FMA loop, bit1 the skinning phase
    dbg = d ? atoi(d) : 0;
#endif
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_kernel<4, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbs_smem_bytes(3)));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_kernel<0, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbs_smem_bytes(3)));
    GLAMR_CUDA_TRY(cudaFuncSetAttribute(lbs_kernel<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbs_smem_bytes(4)));
  }
  auto go = [&](auto kernel, size_t smem) -> int {
    if (pdl) {
      GLAMR_CUDA_TRY(launch_pdl(4, kernel, grid, dim3(kLbsThreads), smem, s, m, n_begin, n_end, betas, w, vertices, dbg));
    } else {
      kernel<<<grid, kLbsThreads, smem, s>>>(m, n_begin, n_end, betas, w, vertices, dbg);
      GLAMR_LAUNCH_CHECK();
    }
    return GLAMR_OK;
  };
  if (m.K == 4 && stages == 4) return go(lbs_kernel<4, 4>, lbs_smem_bytes(4));
  if (m.K == 4) return go(lbs_kernel<4, 3>, lbs_smem_bytes(3));
  return go(lbs_kernel<0, 3>, lbs_smem_bytes(3));
}

int launch_joints_finalize(const SmplDev& m, int n, int orig_joints, const float* root_trans, const float* root_scale,
                           const SmplWorkspace& w, float* joints, cudaStream_t s) {
  if (n <= 0) return GLAMR_OK;
  joints_finalize_kernel<<<(n + 3) / 4, 128, 0, s>>>(m, n, orig_joints, root_trans, root_scale, w, joints);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

int launch_reroot_vertices(int n, const float* root_raw, const float* root_trans, const float* root_scale, float* vertices,
                           cudaStream_t s) {
  if (n <= 0) return GLAMR_OK;
  const size_t total = (size_t)n * kV * 3;
  const int blocks = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
  reroot_vertices_kernel<<<blocks, 256, 0, s>>>(n, root_raw, root_trans, root_scale, vertices);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

}  // namespace glamr

// =================================================================================================== C ABI
using namespace glamr;

namespace {
template <typename T>
int upload(glamr_smpl* h, const std::vector<T>& host, const T** dev) {
  void* p = nullptr;
  GLAMR_CUDA_TRY(cudaMalloc(&p, host.size() * sizeof(T) + 256));
  GLAMR_CUDA_TRY(cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice));
  h->allocs[h->n_allocs++] = p;
  *dev = (const T*)p;
  return GLAMR_OK;
}
}  // namespace

extern "C" int glamr_version(void) { return 100; }

extern "C" int glamr_device_sm_count(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return sms;
}

extern "C" int glamr_smpl_create(glamr_smpl_t** out, const float* v_template, const float* shapedirs, const float* posedirs,
                                 const float* J_regressor, const float* lbs_weights, const int32_t* parents,
                                 const float* J_regressor_extra, int n_extra, const int32_t* pick_vertex_ids, int n_picks,
                                 const int32_t* joint_map, int n_map) {
  if (!out || !v_template || !shapedirs || !posedirs || !J_regressor || !lbs_weights || !parents || !joint_map) return GLAMR_EINVAL;
  if (n_extra < 0 || n_picks < 0 || n_map <= 0 || (n_extra > 0 && !J_regressor_extra) || (n_picks > 0 && !pick_vertex_ids)) return GLAMR_EINVAL;
  for (int k = 0; k < n_map; ++k)
    if (joint_map[k] < 0 || joint_map[k] >= kNJ + n_picks + n_extra) return GLAMR_EINVAL;
  for (int k = 0; k < n_picks; ++k)
    if (pick_vertex_ids[k] < 0 || pick_vertex_ids[k] >= kV) return GLAMR_EINVAL;
  glamr_smpl* h = (glamr_smpl*)calloc(1, sizeof(glamr_smpl));
  if (!h) return GLAMR_EINVAL;
  SmplDev& d = h->dev;
  // kinematic tree levels
  for (int j = 0; j < kNJ; ++j) d.parents[j] = parents[j];
  d.n_levels = 0;
  for (int j = 0; j < kNJ; ++j) {
    if (j > 0 && (parents[j] < 0 || parents[j] >= j)) { free(h); return GLAMR_EINVAL; }
    d.level[j] = (j == 0) ? 0 : d.level[parents[j]] + 1;
    if (d.level[j] + 1 > d.n_levels) d.n_levels = d.level[j] + 1;
  }
  d.n_extra = n_extra; d.n_picks = n_picks; d.n_map = n_map;
  int rc = GLAMR_OK;
  std::vector<int32_t> sup;                  // support vertex of each slot
  {  // support list (first, the LBS images below copy its vertices) + CSR of the extra regressor
    std::vector<int32_t> cov(kVPad, -1);
    auto touch = [&](int v) { if (cov[v] < 0) { cov[v] = (int32_t)sup.size(); sup.push_back(v); } };
    for (int k = 0; k < n_picks; ++k) touch(pick_vertex_ids[k]);
    std::vector<int32_t> ptr(n_extra + 1, 0), ci;
    std::vector<float> rw;
    for (int r = 0; r < n_extra; ++r) {
      for (int v = 0; v < kV; ++v) {
        const float wv = J_regressor_extra[(size_t)r * kV + v];
        if (wv != 0.0f) { touch(v); ci.push_back(cov[v]); rw.push_back(wv); }
      }
      ptr[r + 1] = (int32_t)ci.size();
    }
    if (ci.empty()) { ci.push_back(0); rw.push_back(0.0f); }
    if (sup.empty()) touch(0);
    d.S = (int)sup.size();
    std::vector<int32_t> pci(n_picks > 0 ? n_picks : 1, 0), jm(joint_map, joint_map + n_map);
    for (int k = 0; k < n_picks; ++k) pci[k] = cov[pick_vertex_ids[k]];
    if ((rc = upload(h, cov, &d.compact_of_vertex))) goto fail;
    if ((rc = upload(h, ptr, &d.reg_ptr))) goto fail;
    if ((rc = upload(h, ci, &d.reg_ci))) goto fail;
    if ((rc = upload(h, rw, &d.reg_w))) goto fail;
    if ((rc = upload(h, pci, &d.pick_ci))) goto fail;
    if ((rc = upload(h, jm, &d.joint_map))) goto fail;
  }
  {  // posedirs -> [tile][k][384]
    std::vector<float> t((size_t)kNVTiles * kPF * kTileCols, 0.0f);
    for (int tile = 0; tile < kNVTiles; ++tile)
      for (int k = 0; k < kPF; ++k) {
        const int c0 = tile * kTileCols;
        const int ncol = (c0 + kTileCols <= kV * 3) ? kTileCols : (kV * 3 - c0);
        memcpy(&t[((size_t)tile * kPF + k) * kTileCols], posedirs + (size_t)k * kV * 3 + c0, ncol * sizeof(float));
      }
    if ((rc = upload(h, t, &d.pd_tiles))) goto fail;
  }
  {  // blend basis [20736 cols][224 k] = posedirs^T | shapedirs | v_template scaled by 2^e_B, fp16 hi / lo, wgmma K-major core-matrix
     // image per (256-column tile, 16-wide K chunk): [hi | lo][k group (8 wide)][256 cols][8].  e_B brings max |basis| into
     // [2^14, 2^15), so every entry above 2^-18 max |basis| keeps the 22 significant bits of its hi / lo pair in FP16's normal range.
    auto tf32_rna = [](float x) {            // cvt.rna.tf32.f32: round to nearest, ties away from zero, 10-bit mantissa
      uint32_t u;
      memcpy(&u, &x, 4);
      u = (u + 0x1000u) & 0xFFFFE000u;
      float r;
      memcpy(&r, &u, 4);
      return r;
    };
    auto basis = [&](int col, int k) {
      if (k < kPF) return posedirs[(size_t)k * kV * 3 + col];
      if (k < kPF + kNB) return shapedirs[(size_t)col * kNB + (k - kPF)];       // shapedirs [v][c][l] = [col][l]
      return v_template[col];
    };
    float amax = 0.0f;
    for (int col = 0; col < kV * 3; ++col)
      for (int k = 0; k < kTcFeat; ++k) amax = std::max(amax, std::fabs(basis(col, k)));
    int ex = 0;
    if (amax > 0.0f && std::isfinite(amax)) std::frexp(amax, &ex);            // amax in [2^(ex-1), 2^ex)
    const int e_B = amax > 0.0f && std::isfinite(amax) ? 15 - ex : 0;
    d.tcB_unscale = std::ldexp(1.0f, -e_B);
    // columns past the mesh's 20736: the support vertices' columns again (slot s, coordinate c at 20736 + 3 s + c), so the GEMM blends
    // them a second time where the support tiles of the skinning read them; copies leave max |basis| and e_B as they are
    d.tc_ntiles = smpl_vp_cols(d.S) / kTcN;
    std::vector<__half> img((size_t)d.tc_ntiles * kTcChunks * kTcBStageHalves, __float2half_rn(0.0f));
    for (int col = 0; col < kTcCols + 3 * d.S; ++col) {
      if (col >= kV * 3 && col < kTcCols) continue;
      const int src = col < kTcCols ? col : sup[(col - kTcCols) / 3] * 3 + (col - kTcCols) % 3;
      const int tile = col / kTcN, r = col % kTcN;
      for (int k = 0; k < kTcFeat; ++k) {
        const float v = std::ldexp(basis(src, k), e_B);
        const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
        __half* q = &img[((size_t)tile * kTcChunks + (k >> 4)) * kTcBStageHalves + ((((k >> 3) & 1) * kTcN + r) * 8) + (k & 7)];
        q[0] = hi;
        q[kTcBStageHalves / 2] = lo;
      }
    }
    if ((rc = upload(h, img, &d.tcB))) goto fail;
    // dense skinning weights W[v][24] as the A operand of the tensor-core skinning: per 128-vertex tile [hi | lo][joint group][vertex][4];
    // row kVPad + s (support tile s / 128) holds the weights of support vertex s
    d.sk_tiles = kNVTiles + smpl_sup_tiles(d.S);
    std::vector<float> wimg((size_t)d.sk_tiles * kSkWImageFloats, 0.0f);
    for (int row = 0; row < kVPad + d.S; ++row)
      for (int j = 0; j < kNJ; ++j) {
        if (row >= kV && row < kVPad) break;
        const int v = row < kVPad ? row : sup[row - kVPad];
        const float x = lbs_weights[(size_t)v * kNJ + j];
        const float hi = tf32_rna(x), lo = tf32_rna(x - hi);
        float* q = &wimg[(size_t)(row / kVTile) * kSkWImageFloats + ((size_t)(j >> 2) * kVTile + row % kVTile) * 4 + (j & 3)];
        q[0] = hi;
        q[kSkWHalf] = lo;
      }
    if ((rc = upload(h, wimg, &d.skW))) goto fail;
  }
  {
    std::vector<float> vt((size_t)kVPad * 3, 0.0f), sd((size_t)kVPad * 30, 0.0f);
    memcpy(vt.data(), v_template, (size_t)kV * 3 * sizeof(float));
    memcpy(sd.data(), shapedirs, (size_t)kV * 30 * sizeof(float));
    if ((rc = upload(h, vt, &d.v_template))) goto fail;
    if ((rc = upload(h, sd, &d.shapedirs))) goto fail;
  }
  {  // rest joints as an affine function of beta (double accumulation on the host)
    std::vector<float> jt(kNJ * 3), js(kNJ * 3 * kNB);
    for (int j = 0; j < kNJ; ++j)
      for (int c = 0; c < 3; ++c) {
        double a = 0.0;
        double b[kNB] = {0};
        for (int v = 0; v < kV; ++v) {
          const double wv = J_regressor[(size_t)j * kV + v];
          if (wv == 0.0) continue;
          a += wv * v_template[v * 3 + c];
          for (int l = 0; l < kNB; ++l) b[l] += wv * shapedirs[((size_t)v * 3 + c) * kNB + l];
        }
        jt[j * 3 + c] = (float)a;
        for (int l = 0; l < kNB; ++l) js[(j * 3 + c) * kNB + l] = (float)b[l];
      }
    if ((rc = upload(h, jt, &d.j_template))) goto fail;
    if ((rc = upload(h, js, &d.j_shapedirs))) goto fail;
  }
  {  // K-sparse skinning weights
    int K = 1;
    for (int v = 0; v < kV; ++v) {
      int c = 0;
      for (int j = 0; j < kNJ; ++j) c += lbs_weights[(size_t)v * kNJ + j] != 0.0f;
      if (c > K) K = c;
    }
    if (K < 4) K = 4;
    d.K = K;
    std::vector<float> sw((size_t)kVPad * K, 0.0f);
    std::vector<uint8_t> sj((size_t)kVPad * K, 0);
    for (int v = 0; v < kV; ++v) {
      int c = 0;
      for (int j = 0; j < kNJ; ++j) {
        const float wv = lbs_weights[(size_t)v * kNJ + j];
        if (wv != 0.0f) { sw[(size_t)v * K + c] = wv; sj[(size_t)v * K + c] = (uint8_t)j; ++c; }
      }
    }
    if ((rc = upload(h, sw, &d.skin_w))) goto fail;
    if ((rc = upload(h, sj, &d.skin_j))) goto fail;
  }
  *out = h;
  return GLAMR_OK;
fail:
  glamr_smpl_destroy(h);
  return rc;
}

extern "C" int glamr_smpl_destroy(glamr_smpl_t* m) {
  if (!m) return GLAMR_OK;
  for (int i = 0; i < m->n_allocs; ++i) cudaFree(m->allocs[i]);
  free(m);
  return GLAMR_OK;
}

extern "C" int glamr_smpl_set_lbs_path(int path) {
  if (path < -1 || path > 2) return GLAMR_EINVAL;     // -1: back to the default (GLAMR_LBS_PATH or the compile-time choice)
  g_lbs_path = path;
  return GLAMR_OK;
}

extern "C" int glamr_smpl_info(const glamr_smpl_t* m, int what) {
  if (!m) return GLAMR_EINVAL;
  switch (what) {
    case 0: return m->dev.K;
    case 1: return m->dev.S;
    case 2: return m->dev.n_map;
    default: return GLAMR_EINVAL;
  }
}

extern "C" size_t glamr_smpl_workspace_bytes(const glamr_smpl_t* m, int n) {
  if (!m || n < 0) return 0;
  return smpl_workspace_floats(n, m->dev.S) * sizeof(float);
}

extern "C" size_t glamr_smpl_fk_workspace_bytes(const glamr_smpl_t* m, int n) {
  if (!m || n < 0) return 0;
  return smpl_workspace_floats_fk(n, m->dev.S) * sizeof(float);
}

extern "C" int glamr_smpl_forward(const glamr_smpl_t* m, int n, const float* global_orient, const float* body_pose,
                                  const float* betas, const float* root_trans, const float* root_scale, int orig_joints,
                                  float* joints, float* vertices, void* workspace, size_t workspace_bytes, void* stream) {
  if (!m || n < 0 || !body_pose || !betas || !joints || !workspace) return GLAMR_EINVAL;
  if (workspace_bytes < glamr_smpl_workspace_bytes(m, n)) return GLAMR_ENOSPACE;
  if (n == 0) return GLAMR_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const SmplWorkspace w = smpl_carve_workspace(workspace, n, m->dev.S);
  int rc;
  if ((rc = launch_pose_prep(m->dev, n, global_orient, body_pose, betas, 1, w, s))) return rc;
  if ((rc = launch_lbs(m->dev, 0, n, betas, w, vertices, s))) return rc;
  if ((rc = launch_joints_finalize(m->dev, n, orig_joints, root_trans, root_scale, w, joints, s))) return rc;
  if (vertices && root_trans)
    if ((rc = launch_reroot_vertices(n, w.root_raw, root_trans, root_scale, vertices, s))) return rc;
  return GLAMR_OK;
}

extern "C" int glamr_smpl_fk24(const glamr_smpl_t* m, int n, const float* global_orient, const float* body_pose,
                               const float* root_trans, const float* root_scale, float* joints, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (!m || n < 0 || !body_pose || !joints || !workspace) return GLAMR_EINVAL;
  if (workspace_bytes < glamr_smpl_fk_workspace_bytes(m, n)) return GLAMR_ENOSPACE;
  if (n == 0) return GLAMR_OK;
  cudaStream_t s = (cudaStream_t)stream;
  SmplWorkspace w = smpl_carve_workspace(workspace, n, m->dev.S);
  w.tcA = nullptr;                             // FK only: no blend features, no skinning operands
  w.skB = nullptr;
  w.vp_tiled = 0;
  int rc = launch_pose_prep(m->dev, n, global_orient, body_pose, nullptr, 0, w, s);
  if (rc) return rc;
  fk24_finalize_kernel<<<(n * kNJ * 3 + 255) / 256, 256, 0, s>>>(n, w.jposed, root_trans, root_scale, joints);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
