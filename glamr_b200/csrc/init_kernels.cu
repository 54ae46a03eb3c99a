// init_data on the device (glamr_b200/recon.py): rotation vectors of the HybrIK estimates, the per-person sample tables,
// the gap fill and filter_pose, every person of a sequence in one launch each.  The per-row math is init_math.cuh.
#include "common.cuh"
#include "init_math.cuh"

namespace glamr {

__global__ void init_rotvec_kernel(int n, const void* __restrict__ mats, int f64, float* __restrict__ rotvec, uint8_t* __restrict__ flags,
                                   int32_t* __restrict__ n_flagged) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double R[9];
  if (f64) {
    for (int k = 0; k < 9; ++k) R[k] = static_cast<const double*>(mats)[(size_t)i * 9 + k];
  } else {
    for (int k = 0; k < 9; ++k) R[k] = (double)static_cast<const float*>(mats)[(size_t)i * 9 + k];
  }
  float o[3] = {0.0f, 0.0f, 0.0f};
  const bool ok = rotmat_to_rotvec_f64(R, o);
  flags[i] = ok ? 0 : 1;
  if (!ok) atomicAdd(n_flagged, 1);
  for (int k = 0; k < 3; ++k) rotvec[(size_t)i * 3 + k] = o[k];
}

// one warp per person: before[t] = samples at frames < t, frames[k] = frame of sample k, info = (count, first, last)
__global__ void init_vis_tables_kernel(int P, int T, const float* __restrict__ vis, int32_t* __restrict__ before, int32_t* __restrict__ frames,
                                       int32_t* __restrict__ info, uint8_t* __restrict__ exist) {
  const int p = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (p >= P) return;
  const float* v = vis + (size_t)p * T;
  const int chunk = (T + 31) / 32, t0 = min(lane * chunk, T), t1 = min(t0 + chunk, T);
  int cnt = 0, first = T, last = -1;
  for (int t = t0; t < t1; ++t)
    if (v[t] != 0.0f) { ++cnt; first = min(first, t); last = t; }
  int incl = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  for (int o = 16; o > 0; o >>= 1) {
    first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
    last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  int k = incl - cnt;
  for (int t = t0; t < t1; ++t) {
    before[(size_t)p * T + t] = k;
    if (v[t] != 0.0f) frames[(size_t)p * T + k++] = t;
    if (exist) exist[(size_t)p * T + t] = (v[t] == 1.0f) || (t >= first && t <= last);
  }
  if (lane == 0) {
    info[3 * p] = total;
    info[3 * p + 1] = first;
    info[3 * p + 2] = last;
  }
}

template <typename W, typename Y, typename O>
__device__ __forceinline__ void fill_row(const glamr_fill_job& jb, int t, int c, int n, const int32_t* bef, const int32_t* frm) {
  const Y* src = static_cast<const Y*>(jb.src);
  O* dst = static_cast<O*>(jb.dst);
  const size_t o = (size_t)t * jb.C + c;
  if (!jb.interp) {              // scatter: sample rows at their frames, zeros elsewhere
    const int k = bef[t];
    const bool is_sample = k < n && frm[k] == t;
    dst[o] = is_sample ? (O)src[(size_t)k * jb.src_stride + jb.src_col0 + c] : (O)0;
    return;
  }
  int lo, hi;
  interp_bracket(bef[t], n, lo, hi);
  W w_hi, w_lo;
  interp_weights<W>((W)t, (W)frm[lo], (W)frm[hi], w_hi, w_lo);
  using C = decltype(W() * Y());
  const C y_lo = (C)src[(size_t)lo * jb.src_stride + jb.src_col0 + c], y_hi = (C)src[(size_t)hi * jb.src_stride + jb.src_col0 + c];
  dst[o] = (O)interp_value<C>((C)w_hi, (C)w_lo, y_hi, y_lo);
}

__global__ void init_fill_kernel(const glamr_fill_job* __restrict__ jobs, int T, const int32_t* __restrict__ before,
                                 const int32_t* __restrict__ frames, const int32_t* __restrict__ info) {
  const glamr_fill_job jb = jobs[blockIdx.y];
  const int32_t* bef = before + (size_t)jb.person * T;
  const int32_t* frm = frames + (size_t)jb.person * T;
  const int n = min(info[3 * jb.person], jb.rows);      // never past the rows the source holds
  if (jb.interp && n < 2) return;
  const int total = T * jb.C;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int t = e / jb.C, c = e - t * jb.C;
    switch (jb.kind) {
      case GLAMR_FILL_F32: fill_row<float, float, float>(jb, t, c, n, bef, frm); break;
      case GLAMR_FILL_F64: fill_row<float, double, double>(jb, t, c, n, bef, frm); break;
      case GLAMR_FILL_F32_W64: fill_row<double, float, float>(jb, t, c, n, bef, frm); break;
      default: break;
    }
  }
}

// one warp per person: jump flags in parallel, the walk on lane 0, then the keypoint rule; vis_frames = (vis == 1)
__global__ void init_filter_pose_kernel(int P, int T, int do_filter, const float* __restrict__ orient_cam, float* __restrict__ vis,
                                        uint8_t* __restrict__ jump, const double* __restrict__ kp_score, double min_score, double min_num,
                                        int32_t* __restrict__ vis_frames) {
  const int p = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (p >= P) return;
  float* v = vis + (size_t)p * T;
  uint8_t* jp = jump + (size_t)p * T;
  if (do_filter) {
    const float thr = (float)(3.14159265358979323846 / 3.0);
    for (int t = lane; t < T; t += 32)
      jp[t] = t > 0 && v[t] != 0.0f && orient_jump(orient_cam + ((size_t)p * T + t - 1) * 3, orient_cam + ((size_t)p * T + t) * 3) > thr;
    __syncwarp();
    if (lane == 0) filter_pose_walk(T, jp, v);
    __syncwarp();
    if (kp_score)
      for (int t = lane; t < T; t += 32)
        if (v[t] == 1.0f && keypoints_too_few(kp_score + ((size_t)p * T + t) * 26, min_score, min_num)) v[t] = 0.0f;
    __syncwarp();
  }
  for (int t = lane; t < T; t += 32) vis_frames[(size_t)p * T + t] = v[t] == 1.0f;
}

}  // namespace glamr

using namespace glamr;

extern "C" size_t glamr_sizeof_fill_job(void) { return sizeof(glamr_fill_job); }

extern "C" int glamr_init_rotvec(int n, const void* mats, int f64, float* rotvec, uint8_t* flags, int32_t* n_flagged, void* stream) {
  if (n < 0 || (n > 0 && (!mats || !rotvec || !flags || !n_flagged))) return GLAMR_EINVAL;
  if (n == 0) return GLAMR_OK;
  init_rotvec_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, mats, f64, rotvec, flags, n_flagged);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_init_vis_tables(int P, int T, const float* vis, int32_t* before, int32_t* frames, int32_t* info, uint8_t* exist,
                                     void* stream) {
  if (P <= 0 || T <= 0 || !vis || !before || !frames || !info) return GLAMR_EINVAL;
  init_vis_tables_kernel<<<(P + 3) / 4, 128, 0, (cudaStream_t)stream>>>(P, T, vis, before, frames, info, exist);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_init_fill(int n_jobs, const glamr_fill_job* jobs, int T, int max_cols, const int32_t* before, const int32_t* frames,
                               const int32_t* info, void* stream) {
  if (n_jobs < 0 || T <= 0 || max_cols <= 0 || (n_jobs > 0 && (!jobs || !before || !frames || !info))) return GLAMR_EINVAL;
  if (n_jobs == 0) return GLAMR_OK;
  const int blocks = min((T * max_cols + 255) / 256, 1024);
  init_fill_kernel<<<dim3(blocks, n_jobs), 256, 0, (cudaStream_t)stream>>>(jobs, T, before, frames, info);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}

extern "C" int glamr_init_filter_pose(int P, int T, int do_filter, const float* orient_cam, float* vis, uint8_t* jump, const double* kp_score,
                                      double min_score, double min_num, int32_t* vis_frames, void* stream) {
  if (P <= 0 || T <= 0 || !vis || !vis_frames || (do_filter && (!orient_cam || !jump))) return GLAMR_EINVAL;
  init_filter_pose_kernel<<<(P + 3) / 4, 128, 0, (cudaStream_t)stream>>>(P, T, do_filter, orient_cam, vis, jump, kp_score, min_score,
                                                                          min_num, vis_frames);
  GLAMR_LAUNCH_CHECK();
  return GLAMR_OK;
}
