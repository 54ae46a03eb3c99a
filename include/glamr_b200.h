/* glamr_b200 -- C ABI of the H100 (sm_90a) CUDA library behind GLAMR's global-reconstruction path.
 *
 * GLAMR (NVlabs/GLAMR) is pure Python/PyTorch: it has no FFI layer, the seams a replacement binds to are Python
 * call sites.  Each entry point below names the reference interface it stands behind (paths relative to the
 * reference tree).  The Python host code in glamr_b200/ binds these with ctypes (INTEGRATION.md shows the stub a
 * GLAMR maintainer would add).
 *
 * Conventions: plain C, no torch types.  Unless stated otherwise every pointer is a DEVICE pointer to contiguous
 * row-major float32; `stream` is a cudaStream_t passed as void*.  Functions return 0 on success, a cudaError_t
 * value (>0) for CUDA failures, or a negative GLAMR_E* code for argument errors.  They never synchronise the
 * stream and never allocate device memory, except the *_create functions whose allocations are owned by the
 * returned opaque handle and released by *_destroy.  All buffers are caller-owned.  Re-entrant across streams; no
 * global state.
 */
#ifndef GLAMR_B200_H
#define GLAMR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GLAMR_OK 0
#define GLAMR_EINVAL (-1)      /* bad argument / unsupported shape */
#define GLAMR_ENOSPACE (-2)    /* workspace too small */
#define GLAMR_EUNSUPPORTED (-3)

#define GLAMR_NUM_VERTS 6890
#define GLAMR_NUM_JOINTS 24
#define GLAMR_NUM_BETAS 10
#define GLAMR_NUM_POSE_FEAT 207

int glamr_version(void);
/* number of SMs / device ordinal the library sees for the current context (for grid sizing diagnostics) */
int glamr_device_sm_count(void);
/* Measurement aid: launches a register-resident FFMA loop (8 CTAs x 256 threads per SM, 16 independent chains, `iters`
 * rounds) on `stream`; *flops (HOST pointer) receives the flop count of the launch.  The caller times it with events: the
 * FP32 throughput this GPU sustains at its present clocks (bench.py's roofline.fp32.peak).  scratch: >= 8*256*SMs floats. */
int glamr_fp32_probe(int iters, float* scratch, size_t scratch_floats, double* flops, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * SMPL body model  --  stands behind lib/models/smpl.py:274-343 (class SMPL: forward, get_joints) and the
 * third-party smplx.lbs it calls (in-tree statement: HybrIK/hybrik/models/layers/smpl/lbs.py:195-288,402-548).
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct glamr_smpl glamr_smpl_t;

/* All constant arrays are HOST pointers (one-off upload; the library re-tiles them for its kernels).
 *   v_template [6890,3]  shapedirs [6890,3,10]  posedirs [207,20670]  J_regressor [24,6890]
 *   lbs_weights [6890,24]  parents [24]  J_regressor_extra [n_extra,6890]
 *   pick_vertex_ids [n_picks]  (smplx VertexJointSelector)     joint_map [n_map] indexes [24 | n_picks | n_extra]
 */
int glamr_smpl_create(glamr_smpl_t** out, const float* v_template, const float* shapedirs, const float* posedirs,
                      const float* J_regressor, const float* lbs_weights, const int32_t* parents,
                      const float* J_regressor_extra, int n_extra, const int32_t* pick_vertex_ids, int n_picks,
                      const int32_t* joint_map, int n_map);
int glamr_smpl_destroy(glamr_smpl_t* m);
/* introspection: 0 max skin weights per vertex, 1 support size (vertices feeding picks/regressors), 2 n_map */
int glamr_smpl_info(const glamr_smpl_t* m, int what);
size_t glamr_smpl_workspace_bytes(const glamr_smpl_t* m, int n);       /* glamr_smpl_forward */
size_t glamr_smpl_fk_workspace_bytes(const glamr_smpl_t* m, int n);    /* glamr_smpl_fk24 (no blend operands) */
/* Which kernels evaluate the blend + skinning of SMPL.forward: 1 (default) = tcgen05 3xTF32 blend GEMM + skinning kernel,
 * 0 = the single FP32 SIMT kernel (kept for A/B verification; env GLAMR_LBS_PATH=simt selects it at start-up).  Process-wide. */
int glamr_smpl_set_lbs_path(int path);

/* SMPL.forward (lib/models/smpl.py:289-316).  n frame-persons.
 *   global_orient [n,3] (NULL -> zeros)  body_pose [n,69]  betas [n,10]
 *   root_trans [n,3] or NULL (no re-rooting)   root_scale [n] or NULL (-> 1)
 *   orig_joints != 0: joints = the 24 LBS joints, else the n_map mapped joints
 *   joints [n, 24 or n_map, 3]   vertices [n,6890,3] or NULL
 */
int glamr_smpl_forward(const glamr_smpl_t* m, int n, const float* global_orient, const float* body_pose,
                       const float* betas, const float* root_trans, const float* root_scale, int orig_joints,
                       float* joints, float* vertices, void* workspace, size_t workspace_bytes, void* stream);

/* SMPL.get_joints (lib/models/smpl.py:318-343): FK only, rest joints from v_template (betas ignored). */
int glamr_smpl_fk24(const glamr_smpl_t* m, int n, const float* global_orient, const float* body_pose,
                    const float* root_trans, const float* root_scale, float* joints, void* workspace,
                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Row-wise rotation algebra  --  lib/utils/konia_transform.py:234-822, lib/utils/torch_transform.py:10-279.
 * op codes: see glamr_b200/csrc/rowops.cuh (RowOp).  in1 may be NULL for unary ops; gin* may be NULL.
 * ---------------------------------------------------------------------------------------------------------- */
int glamr_rowop_fwd(int op, int n, const float* in0, const float* in1, float* out, void* stream);
int glamr_rowop_vjp(int op, int n, const float* in0, const float* in1, const float* gout, float* gin0,
                    float* gin1, void* stream);

/* traj_pred/utils/traj_utils.py:65-88  traj_local2global_heading for B sequences of T frames, time-major
 * local_traj [T,B,11] -> trans [T,B,3], orient_q [T,B,4] (local_orient_type '6d', local_heading on/off);
 * scratch [B*T*3] floats */
int glamr_traj_local2global(int T, int B, const float* local_traj, int local_heading, float* trans, float* orient_q,
                            float* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * init_data on the device  --  global_recon/models/global_recon_model.py:88-137, :250-271 (glamr_b200/recon.py).
 * All P persons of a T-frame sequence in one launch per entry point.
 *
 * glamr_init_rotvec: n rotation matrices [n,9] (float64 if f64, else float32) -> float32 rotation vectors [n,3] by
 *   recon.rotmats_to_rotvec's float64 algorithm.  flags[i] = 1 (and *n_flagged += 1, int32, zeroed by the caller)
 *   where the two Newton steps do not reach a proper rotation; those rows of rotvec hold zeros and belong to SciPy.
 * glamr_init_vis_tables: per person p, from vis [P,T] (a frame is a sample where vis != 0): before [P,T] = samples
 *   at earlier frames, frames [P,T] = frame of each sample (first `count` entries), info [P,3] = (count, first
 *   sample frame, last sample frame; T and -1 without samples), exist [P,T] (uint8 0/1, may be NULL) = vis == 1 or
 *   first <= t <= last.
 * glamr_init_fill: job j of `jobs` (device array) writes jobs[j].dst [T, C] from the sample rows of person
 *   jobs[j].person: with `interp`, scipy interp1d(kind='linear', fill_value='extrapolate') over the sample frames
 *   (SciPy 1.18 operation order); without, the samples at their frames and zeros elsewhere.  max_cols >= every C.
 *   Only the first min(count, rows) samples are read; an interpolating job with fewer than two leaves dst untouched
 *   (the caller rejects that input, as interp1d does).
 * glamr_init_filter_pose: with do_filter, recon.filter_pose on vis [P,T] in place (orient_cam [P,T,3] float32; jump
 *   [P,T] uint8 scratch; kp_score [P,T,26] float64 or NULL for no keypoint rule); then vis_frames [P,T] int32 =
 *   (vis == 1).
 * ---------------------------------------------------------------------------------------------------------- */
#define GLAMR_FILL_F32 0        /* float32 abscissae and rows (interp1d of float32 samples at float32 frames) */
#define GLAMR_FILL_F64 1        /* float32 abscissae, float64 rows */
#define GLAMR_FILL_F32_W64 2    /* float64 abscissae (integer frame indices), float32 rows, computed in float64, float32 out */
typedef struct {
  const void* src;      /* sample k of the person at src + (k * src_stride + src_col0) elements */
  void* dst;            /* [T, C] */
  int32_t person, C, src_stride, src_col0, kind, interp;
  int32_t rows;         /* sample rows at src */
} glamr_fill_job;
size_t glamr_sizeof_fill_job(void);
int glamr_init_rotvec(int n, const void* mats, int f64, float* rotvec, uint8_t* flags, int32_t* n_flagged, void* stream);
int glamr_init_vis_tables(int P, int T, const float* vis, int32_t* before, int32_t* frames, int32_t* info, uint8_t* exist,
                          void* stream);
int glamr_init_fill(int n_jobs, const glamr_fill_job* jobs, int T, int max_cols, const int32_t* before, const int32_t* frames,
                    const int32_t* info, void* stream);
int glamr_init_filter_pose(int P, int T, int do_filter, const float* orient_cam, float* vis, uint8_t* jump, const double* kp_score,
                           double min_score, double min_num, int32_t* vis_frames, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Learned prior (inference only)  --  stands behind MotionTrajJointModel.inference
 * (motion_infiller/models/motion_traj_joint_model.py:141-145): MotionInfillerVAE.inference_one_step
 * (motion_infiller/models/motion_infiller_vae.py:551-562 with ContextEncoder :92-123, DataDecoder :345-421) and
 * TrajPredVAE.inference (traj_pred/models/traj_pred_vae.py:524-548 with ContextEncoder :72-92, DataDecoder :269-333).
 * Parameters are registered under their reference state-dict names ("context_encoder.in_fc.weight", ...), so a
 * Lightning checkpoint's state_dict maps 1:1.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct glamr_net glamr_net_t;
int glamr_net_create(glamr_net_t** out);
int glamr_net_destroy(glamr_net_t* n);
/* upload one named float32 parameter from a HOST pointer */
int glamr_net_set_tensor(glamr_net_t* n, const char* name, const float* host, size_t numel);
/* Y[M,N] = act(X[M,K] W[N,K]^T + bias): the GEMM behind every nn.Linear / attention projection / FFN of the prior
 * networks.  M <= 256 runs an exact FP32 kernel in both modes.  Above that, mode 1 (the infiller's transformer) runs
 * wgmma tf32 with a 3xTF32 split (FP32-accurate), its partial sums folded in FP32 at every K step of 32; mode 0 runs the
 * FP32 SIMT tile kernel that the trajectory predictor uses.  bias may be NULL. */
int glamr_linear_forward(int M, int N, int K, const float* X, const float* W, const float* bias, int relu, float* Y, int mode,
                         void* stream);
size_t glamr_infiller_workspace_floats(int B);
size_t glamr_trajpred_workspace_floats(int T, int B);
/* One 50-frame window (past 10 | current 30 | future 10), B sequences, seq-first buffers:
 *   in_pose [50,B,69]   key_pad_mask [B,50] uint8 (1 = frame invisible / padding)   eps [eps_rows,128], eps_rows in {1,B}, or NULL
 *   out_pose [40,B,69] = the 10 past input frames followed by the 30 decoded frames */
int glamr_infiller_window_forward(const glamr_net_t* n, int B, const float* in_pose, const uint8_t* key_pad_mask,
                                  const float* eps, int eps_rows, float* out_pose, float* workspace, size_t workspace_floats,
                                  void* stream);
/* The whole autoregressive sweep of motion_infiller_vae.py:618-632 (windows of 50 frames, stride 30) in one call:
 *   pose_io [T,B,69]: input body pose, overwritten with the infilled pose   key_pad_all [B,T] uint8 (1 = frame invisible)
 *   eps [ceil((T-10)/30)][eps_rows][128], eps_rows in {1,B}   workspace >= glamr_infiller_sequence_workspace_floats(B) floats */
size_t glamr_infiller_sequence_workspace_floats(int B);
int glamr_infiller_forward(const glamr_net_t* n, int T, int B, float* pose_io, const uint8_t* key_pad_all, const float* eps,
                           int eps_rows, float* workspace, size_t workspace_floats, void* stream);
/* The same sweep in reconstruction mode (inference_multi_step with recon=True, motion_infiller_vae.py:551-557,618-632): each window
 * encodes the ground truth of its 30 current frames with the posterior DataEncoder (:204-233, the data_encoder.* parameters, which
 * must be registered) and decodes z = the posterior mean.  No eps.
 *   pose_io [T,B,69]: input body pose, overwritten with the reconstructed pose   gt_body_pose [T,B,69]   key_pad_all as above
 *   workspace >= glamr_infiller_recon_workspace_floats(B) floats */
size_t glamr_infiller_recon_workspace_floats(int B);
int glamr_infiller_recon_forward(const glamr_net_t* n, int T, int B, float* pose_io, const float* gt_body_pose,
                                 const uint8_t* key_pad_all, float* workspace, size_t workspace_floats, void* stream);
/*   in_joint_pos [T,B,69] (23 joints from SMPL.get_joints)   eps as above   init_xy [B,2] / init_heading [B] or NULL
 *   out_local_traj [T,B,11]   out_trans [T,B,3]   out_orient_aa [T,B,3] */
int glamr_trajpred_forward(const glamr_net_t* n, int T, int B, const float* in_joint_pos, const float* eps, int eps_rows,
                           const float* init_xy, const float* init_heading, float* out_local_traj, float* out_trans,
                           float* out_orient_aa, float* workspace, size_t workspace_floats, void* stream);
/* Windowed prediction (traj_pred_vae.py:484-520, multi_step_trajpred): the track is cut into C = ceil(T/W) windows of W frames,
 * the last one zero-padded, and all C*B windows run as rows of one batch.  Each window draws its own z; no init_xy /
 * init_heading reaches a window.  The windows are stitched with the reference's heading hand-over at each window start.
 *   in_joint_pos [T,B,69]   eps [C,B,128] or NULL (z = mu)   outputs as glamr_trajpred_forward
 *   workspace >= glamr_trajpred_windows_workspace_floats(T, B, W) floats */
size_t glamr_trajpred_windows_workspace_floats(int T, int B, int W);
int glamr_trajpred_windows_forward(const glamr_net_t* n, int T, int B, int W, const float* in_joint_pos, const float* eps,
                                   float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                   size_t workspace_floats, void* stream);

/* Tracks of different lengths in one call.  B tracks are packed without padding: track b is rows offsets[b] .. offsets[b+1] - 1 of
 * every [rows, ...] buffer (offsets [B+1] int32 on the DEVICE, offsets[0] = 0).  lens [B] and row_batch [B] are HOST int32 arrays:
 * the tracks' lengths, and for each track the batch size of the single-track call it reproduces (1 for a lone track, P for each
 * track of a block of P equal-length tracks).  Track b's outputs are bit-identical to that call's outputs for it: every Linear
 * runs on the kernel that call's M selects.  So the tracks must come in an order in which those kernels change at most once per
 * Linear; any other order returns GLAMR_EINVAL:
 *   infiller: by non-decreasing class c(rb) = #{S in 50, 30, 2, 1 : S * rb > 256}, and by non-increasing length within a class;
 *   trajectory predictor: by non-decreasing (F * rb > 256) + (R * rb > 256), where F = T, R = 1 for the single pass and
 *   F = C W, R = C with C = ceil(T / W) for the windowed one.
 * Infiller: pose_io [rows,69] (overwritten with the infilled pose)  key_pad [rows] uint8 (1 = invisible)
 *   eps [B][eps_windows][128]: track b's window i reads eps[b][i]; eps_windows >= ceil((T_b - 10) / 30) for every b, T_b > 10. */
size_t glamr_infiller_ragged_workspace_floats(int B);
int glamr_infiller_forward_ragged(const glamr_net_t* n, int B, const int32_t* lens, const int32_t* row_batch, const int32_t* offsets,
                                  float* pose_io, const uint8_t* key_pad, const float* eps, int eps_windows, float* workspace,
                                  size_t workspace_floats, void* stream);
/* Single pass:  in_joint_pos [rows,69]   eps [B,128] or NULL   init_xy [B,2] / init_heading [B] or NULL
 *   out_local_traj [rows,11]   out_trans [rows,3]   out_orient_aa [rows,3] */
size_t glamr_trajpred_ragged_workspace_floats(int B, const int32_t* lens);
int glamr_trajpred_forward_ragged(const glamr_net_t* n, int B, const int32_t* lens, const int32_t* row_batch, const int32_t* offsets,
                                  const float* in_joint_pos, const float* eps, const float* init_xy, const float* init_heading,
                                  float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                  size_t workspace_floats, void* stream);
/* Windowed: track b contributes C_b = ceil(T_b / W) windows.  win_offsets [B+1] (DEVICE) = prefix sums of C_b.
 *   eps [sum C_b, 128] (track b's window c at row win_offsets[b] + c) or NULL   other buffers as the single pass */
size_t glamr_trajpred_windows_ragged_workspace_floats(int B, const int32_t* lens, int W);
int glamr_trajpred_windows_forward_ragged(const glamr_net_t* n, int B, int W, const int32_t* lens, const int32_t* row_batch,
                                          const int32_t* offsets, const int32_t* win_offsets, const float* in_joint_pos, const float* eps,
                                          float* out_local_traj, float* out_trans, float* out_orient_aa, float* workspace,
                                          size_t workspace_floats, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Global optimisation  --  stands behind GlobalReconOptimizer.forward / compute_loss / optimize_main
 * (global_recon/models/global_recon_model.py:428-570), the residual registry global_recon/models/loss_func.py:314-340
 * and torch.optim.Adam.step (:563,:642).
 * ---------------------------------------------------------------------------------------------------------- */
enum glamr_term {
  GLAMR_T_KP_2D = 0, GLAMR_T_KP_2D_DIST, GLAMR_T_CAM_TRAJ_ROT, GLAMR_T_CAM_TRAJ_TRANS, GLAMR_T_TRAJ_ROT_SMOOTH,
  GLAMR_T_TRAJ_TRANS_SMOOTH, GLAMR_T_REL_TRANSFORM, GLAMR_T_DXY_REG, GLAMR_T_DHEADING_REG, GLAMR_T_DHEADING_REG_NEW,
  GLAMR_T_ROT_REG, GLAMR_T_Z_REG, GLAMR_T_ROT_RES, GLAMR_T_TRANS_RES, GLAMR_T_CAM_INV_TRANS_RES_REG,
  GLAMR_T_CAM_INV_ROT_SMOOTH, GLAMR_T_CAM_ORIGIN_SMOOTH, GLAMR_T_CAM_UP_REG, GLAMR_T_CAM_ROT_SMOOTH,
  GLAMR_T_CAM_TRANS_SMOOTH, GLAMR_T_CAM_DEPTH_SMOOTH, GLAMR_NUM_TERMS
};

enum glamr_cam_mode {
  GLAMR_CAM_CONST = 0,        /* camera is data (cam_pose_const)                           (:473 not taken)      */
  GLAMR_CAM_PER_FRAME = 1,    /* variables cam_rot_6d [T,6], cam_trans [T,3]               (:478-480)            */
  GLAMR_CAM_FIXED = 2,        /* variables cam_rot_6d_fix [1,6], cam_trans_fix [1,3]       (:475-477)            */
  GLAMR_CAM_FROM_PERSONS = 3  /* mean of person_transform_world @ person2cam + residuals   (:481-508)            */
};

enum glamr_traj_source {
  GLAMR_TRAJ_PREDICTED = 0,   /* traj_local_pred + local variables through the trajectory codec on the exist range   (:448-449) */
  GLAMR_TRAJ_BASE = 1         /* every frame: orient/trans_base_init, then world_res / world_dheading (flag_infer_motion_traj or
                               * flag_pred_traj false: no codec, no prefix scans; the traj_local_* variables only see their
                               * regularisers).  flag_opt_traj false: the same with neither world variable active       */
};

typedef struct glamr_person {
  int32_t start, len;              /* exist range [start, start+len) of this person (exist_frames)              */
  int32_t group;                   /* group of this person (see glamr_group_t)                                    */
  int32_t off_xy, off_heading, off_dxy, off_dheading, off_z, off_rot;     /* offsets into theta (floats)        */
  int32_t off_world_dheading, off_orient_res, off_trans_res;              /* [T], [T,3], [T,3]                  */
  int32_t off_world_dxy;           /* [T,2] world_dxy (read only with has_world_dxy)                              */
  int32_t off_p2c_rot, off_p2c_trans; /* [T,6] person2cam_res_rot, [T,3] person2cam_res_trans (read only with
                                    * has_person2cam)                                                               */
  const float* traj_local_pred;    /* [len,11]                                                                    */
  const float* orient_base_init;   /* [T,3] smpl_orient_world_base outside the exist range                        */
  const float* trans_base_init;    /* [T,3]                                                                       */
  const float* cam_K;              /* [T,9]                                                                       */
  const float* kp_target;          /* [T,J,2] kp_2d_aligned                                                       */
  const float* orient_cam_6d;      /* [T,6]  rot6d(R(smpl_orient_cam)), target of cam_traj_rot                    */
  const float* orient_cam_q;       /* [T,4]  angle_axis_to_quaternion(smpl_orient_cam): target when rot_type 'quat' */
  const float* trans_cam;          /* [T,3]  root_trans_cam                                                       */
  const float* person2cam;         /* [T,12] 3x4, used by GLAMR_CAM_FROM_PERSONS                                  */
  const float* dheading_mask;      /* [len-1] (cam_fix_frames)                                                    */
  const float* rot_mask;           /* [len] or NULL (flag_opt_vis_local_rot)                                      */
  const float* vis;                /* [T] 1/0 vis_frames                                                          */
  /* per-stage weights, already containing score^2, min_conf, first-frame weighting, visibility               */
  const float* kp_w;               /* [T,J]                                                                       */
  const float* kp_dist_mask;       /* [T,J]                                                                       */
  const float* ctr_w;              /* [T]  cam_traj_rot                                                           */
  const float* ctt_w;              /* [T]  cam_traj_trans                                                         */
  /* [T,2] or NULL (-> trans_base_init): x / y of root_trans_world_base on the frames the codec does not produce.  The
   * reference adds world_dxy IN PLACE to root_trans_world, which aliases the base unless world_res alone composes the
   * pose (:451-468); the base then keeps every evaluation's world_dxy.  With world_dxy_alias each trajectory forward adds
   * the current world_dxy here exactly once.  Caller-owned, initialised to trans_base_init[:, :2], persists across
   * stages; every rank keeps its own copy (the trajectory forward is replicated).                                  */
  float* world_dxy_base;
} glamr_person_t;

/* Groups: G independent problems that share one configuration (stages, variables, loss settings) optimised as one problem: the
 * seeds of one sequence, or any (sequence, seed) pairs.  Group g owns persons [p0, p0+Q), frame-persons [n0, n0 + Q*T) (frame t of
 * its person p0+q is row n0 + q*T + t), camera rows [c0, c0+T) of every per-frame table and camera read-back, and the block of theta
 * that starts at theta0.  Its rel_transform pairs (only inside the group) are the [Q*Q, T] block at rel0, its term sums and loss
 * terms one row each.  Each group's camera, camera terms and term sums are reduced over the same elements in the same order as the
 * one-group problem of that group alone, so every group's results are those of its own one-group run bit for bit.  G > 1 needs the
 * whole frame-person range on one rank (n_begin 0, n_end = sum Q*T, owner).  G 0 (zero-initialised) = 1. */
typedef struct glamr_group {
  int32_t p0, Q;                   /* first person, persons                                                        */
  int32_t n0;                      /* first frame-person                                                           */
  int32_t c0, T;                   /* first camera row, frames                                                     */
  int32_t theta0;                  /* first float of the group's block of theta                                    */
  int32_t off_cam_rot, off_cam_trans; /* theta offsets of the group's camera variables (as glamr_problem_t's)       */
  int32_t rel0;                    /* first (pair, frame) entry of the group's block of rel_target / rel_w / rel_wt */
  float term_norm[GLAMR_NUM_TERMS];  /* the group's normalisers (denominators of the reference's means)             */
  float gs[GLAMR_NUM_TERMS];       /* term_weight / term_norm in float32 where the term enters the total, else 0   */
} glamr_group_t;

typedef struct glamr_problem {
  int32_t P, T, J;                 /* persons (all groups), frames (the longest group's), joints per person (n_map of the
                                    * SMPL handle)                                                                  */
  int32_t cam_mode;                /* enum glamr_cam_mode                                                         */
  int32_t off_cam_rot, off_cam_trans; /* variable offsets (modes 1,2: cam_rot_6d / cam_trans; mode 3: residuals); with
                                    * groups, those of group 0 (glamr_group_t has every group's)                       */
  int32_t use_world_res, has_world_dheading;
  int32_t trans_res_all;           /* mode 3: cam_inv_trans_residual has T rows (else one row per empty frame)    */
  int32_t cam_up_first_only;
  int32_t n_params;                /* length of theta / grad / adam state                                         */
  int32_t n_begin, n_end;          /* frame-persons n = p*T + t (n0 + q*T + t with groups) whose SMPL / per-frame residuals this rank evaluates
                                    * (multi-GPU shard; any contiguous range, a person may straddle two ranks)         */
  int32_t owner;                   /* != 0: this rank also evaluates the replicated terms (camera, regs, rel)    */
  int32_t cam_traj_rot_quat;       /* cam_traj_rot: rot_type 'quat' (loss_func.py:158-161) instead of '6d'          */
  int32_t traj_rot_smooth_quat;    /* traj_rot_smoothness: rot_type 'quat' (loss_func.py:126-128)                  */
  int32_t traj_source;             /* enum glamr_traj_source; 0 (zero-initialised) = the predicted trajectory      */
  int32_t heading_vec;             /* heading_type 'vec' (:403-405): traj_local_heading [2] / _dheading [len-1,2] are added to
                                    * the predicted heading VECTOR, whose angle enters the scan; 0 = 'scalar' (angle)   */
  int32_t has_world_dxy;           /* world_dxy [T,2] is added to root_trans_world x / y (:467-468)                */
  int32_t world_dxy_alias;         /* that add also lands in the base (see glamr_person_t.world_dxy_base)          */
  int32_t has_person2cam;          /* flag_opt_person2cam_rot / _trans (:484-488): mode 3 composes each person's person2cam with
                                    * [rot6d(person2cam_res_rot) | person2cam_res_trans] before the mean; 0 = person2cam as is */
  int32_t G;                       /* groups (see above); G > 1 needs `groups`                                     */
  int32_t group_params;            /* floats of theta per group when all groups have one layout (seed groups), else 0;
                                    * informational, the table holds every group's base                            */
  float cam_up_first_weight;
  float rel_trans_weight;
  float term_weight[GLAMR_NUM_TERMS];   /* YAML weight, 0 if the term is absent                                  */
  float term_norm[GLAMR_NUM_TERMS];     /* normaliser (denominator) of the reference's mean                      */
  int32_t term_enabled[GLAMR_NUM_TERMS];
  int32_t term_monitor[GLAMR_NUM_TERMS];
  const glamr_person_t* persons;   /* DEVICE array [P]                                                            */
  const glamr_group_t* groups;     /* DEVICE array [G] (G > 1; unused with one group).  glamr_opt_set_problem accepts
                                    * only a table with the p0, Q, n0, c0, T of the one given to glamr_opt_create
                                    * (theta0, camera offsets, rel0 and the normalisers may change)                */
  const float* smpl_pose_all;      /* [N,69] body pose (infilled) of every frame-person, constant during optimisation */
  const float* smpl_beta_all;      /* [N,10]                                                                      */
  const float* scale_all;          /* [N] or NULL                                                                 */
  const float* cam_pose_const;     /* [sum T,12] world->cam 3x4 (mode 0), one block of T rows per group           */
  const int32_t* empty_index;      /* [sum T] row of cam_inv_rot_residual for frames without any person, else -1  */
  const int32_t* fill_src;         /* [sum T] forward-fill source frame (mode 3), a frame of the same group        */
  const float* inv_num_persons;    /* [sum T] 1/num visible persons of the group (0 where none)                   */
  const float* rel_target;         /* per group [Q*Q,T,12] rel_transform_cam (pair i*Q+j inside the group), or NULL */
  const float* rel_w;              /* per group [Q*Q,T] squared frame weights for the rotation part (0 = unused)  */
  const float* rel_wt;             /* per group [Q*Q,T] same for the translation part                             */
  const uint8_t* active;           /* [n_params] 1 where Adam updates theta                                       */
} glamr_problem_t;

size_t glamr_sizeof_person(void);
size_t glamr_sizeof_problem(void);

typedef struct glamr_opt glamr_opt_t;

/* The handle owns scratch sized for N = sum Q*T frame-persons (P*T with one group), sum T camera rows and J, and the Adam moments.  `problem` is copied (host struct; its embedded
 * pointers are device pointers that must stay alive while the handle uses them). */
int glamr_opt_create(glamr_opt_t** out, const glamr_smpl_t* smpl, const glamr_problem_t* problem);
int glamr_opt_destroy(glamr_opt_t* st);
/* Re-read a modified problem description (new stage: weights, active mask, camera mode; same P, T, J, n_params and group shapes).
 * reset_adam bit 0 zeroes the Adam moments and step count: the reference builds a fresh torch.optim.Adam per stage
 * (global_recon_model.py:548,:642); bit 1 also zeroes all scratch (handle re-used for a new sequence).  A changed
 * frame-person range [n_begin, n_end) re-primes the pipelined blend: the next evaluation recomputes v_posed for it. */
int glamr_opt_set_problem(glamr_opt_t* st, const glamr_problem_t* problem, int reset_adam, void* stream);
/* length (floats) of the caller-owned reduce buffer: [grad (n_params) | un-normalised term sums (G x GLAMR_NUM_TERMS)] */
size_t glamr_opt_reduce_count(const glamr_opt_t* st);
/* kernels per optimiser iteration (glamr_opt_backward + glamr_opt_apply) for the current problem (bench.py: gpu_launches) */
int glamr_opt_launch_count(const glamr_opt_t* st);

/* forward (trajectory, camera, SMPL, projection) + residuals + analytic backward for the current theta, leaving
 * [grad | term sums] of THIS rank's share in reduce_buf.  With several GPUs the caller sums reduce_buf over ranks
 * (one NCCL allreduce) before glamr_opt_apply.  (closure of global_recon_model.py:551-557) */
int glamr_opt_backward(glamr_opt_t* st, const float* theta, float* reduce_buf, void* stream);
/* loss_terms [G][GLAMR_NUM_TERMS+1] (device): per group, un-weighted term values (sum / normaliser) then the weighted total.
 * Then one torch.optim.Adam step (betas 0.9/0.999, eps 1e-8) on the active entries of theta; the step count and
 * bias corrections live on the device so the call sequence can be captured in a CUDA graph.  With
 * loss_hist_stride > 0 the terms of optimiser step k (0-based, counted on the device since the last reset) are
 * written at loss_terms + k * loss_hist_stride, so a replayed graph fills a per-iteration history. */
int glamr_opt_apply(glamr_opt_t* st, float* theta, const float* reduce_buf, double lr, float* loss_terms,
                    int loss_hist_stride, void* stream);
/* n_iters x (glamr_opt_backward + glamr_opt_apply) for a single-rank job (no reduction between the two).  With
 * use_graph != 0 the iteration is captured once into a CUDA graph owned by the handle (re-captured when the problem
 * or any argument changes) and replayed: the loop `for _ in range(opt_niters): optimizer.step(closure)` of
 * global_recon_model.py:558-569 becomes opt_niters graph launches with no host work in between. */
int glamr_opt_iterate(glamr_opt_t* st, float* theta, float* reduce_buf, double lr, float* loss_terms, int loss_hist_stride,
                      int n_iters, int use_graph, void* stream);
/* loss_terms only, no update (GlobalReconOptimizer.compute_loss, :533-545) */
int glamr_opt_losses(glamr_opt_t* st, const float* reduce_buf, float* loss_terms, void* stream);

/* Measurement hooks (bench.py roofline): when enabled, glamr_opt_backward brackets the LBS kernel with CUDA events on
 * the launching stream (do not enable while capturing a CUDA graph); glamr_opt_last_lbs_ms waits for the last pair
 * and returns its duration.  The only entry point that synchronises. */
/* glamr_opt_backward for a caller that runs glamr_opt_apply next on the same stream, with its exchange of reduce_buf in between (the
 * multi-GPU loop of global_recon_model.py:558-569): the pipelined side-stream work is joined by that apply call, not at the end of this one */
int glamr_opt_backward_for_apply(glamr_opt_t* st, const float* theta, float* reduce_buf, void* stream);
int glamr_opt_kernel_timing(glamr_opt_t* st, int enable);
/* the last timed evaluation's LBS split into the critical-path kernel (the support vertices' skinning on the tensor-core path, the
 * whole skinning with tcblend, the whole LBS kernel on the SIMT path) and the side stream's part (mesh skinning + blend on the
 * tensor-core path, the blend with tcblend, 0 on the SIMT path) */
int glamr_opt_last_lbs_parts_ms(glamr_opt_t* st, float* critical_ms, float* blend_ms);
/* mean ms of the blend (feature kernel + tcgen05 GEMM) of this rank's frame-persons launched ALONE `reps` times (synchronises;
 * GLAMR_EUNSUPPORTED on the SIMT path or before the first evaluation) */
int glamr_opt_time_blend(glamr_opt_t* st, int reps, float* ms);
int glamr_opt_last_lbs_ms(glamr_opt_t* st, float* ms);
/* enable == 2: also record an event after every launch; durations (ms) between consecutive marks of the last
 * backward (+ apply) sequence on the caller's stream: traj_fwd, cam_fwd, pose_prep, skinning (the support vertices' on the
 * tensor-core path), residuals[, cam_bwd + scatter], traj_bwd, apply; on the tensor-core path two more follow, measured on the side
 * stream: the mesh skinning and the blend after it (features + GEMM) */
int glamr_opt_kernel_times(glamr_opt_t* st, float* ms, int* n);

/* [P,T,...] below: one row per frame-person, N = sum Q*T rows with groups */
enum glamr_read {
  GLAMR_R_ORIENT_WORLD = 0,    /* [P,T,3]   smpl_orient_world            */
  GLAMR_R_TRANS_WORLD = 1,     /* [P,T,3]   root_trans_world             */
  GLAMR_R_ORIENT_BASE = 2,     /* [P,T,3]   smpl_orient_world_base       */
  GLAMR_R_TRANS_BASE = 3,      /* [P,T,3]   root_trans_world_base        */
  GLAMR_R_KP_PRED = 4,         /* [P,T,J,2] kp_2d_pred                   */
  GLAMR_R_ORIENT_CAM_IN_WORLD = 5, /* [P,T,3]                            */
  GLAMR_R_TRANS_CAM_IN_WORLD = 6,  /* [P,T,3]                            */
  GLAMR_R_CAM_POSE = 7,        /* [sum T,12]  world->cam 3x4 of every group */
  GLAMR_R_CAM_POSE_INV = 8,    /* [sum T,12]                             */
  GLAMR_R_JOINTS_WORLD = 9,    /* [P,T,J,3]                              */
  GLAMR_R_TRAJ_LOCAL = 10,     /* [P,T,11]  traj_local (rows of the exist range, others 0) */
  GLAMR_R_ADAM_M = 11,         /* [n_params] Adam first moment                                */
  GLAMR_R_ADAM_V = 12          /* [n_params] Adam second moment                               */
};
/* ---- multi-GPU without a library collective: gradient reduction over NVLink peer memory --------------------------
 * One process per GPU.  Every rank allocates one buffer (glamr_peer_alloc; size glamr_opt_peer_bytes), ships its
 * 64-byte CUDA IPC handle to the other ranks (any host channel, e.g. torch.distributed.all_gather_object), opens theirs
 * (glamr_peer_open) and registers the table with glamr_opt_set_peers.  From then on, inside glamr_opt_iterate, the
 * backward pass pushes every element of [grad | term sums], tagged with the iteration number in the same 8-byte word,
 * into every rank's buffer, and the Adam kernel polls its own memory until the W tagged values of an element have
 * landed and sums them in rank order (identical bits on every rank): the all-reduce of global_recon's shared camera
 * gradient (SURVEY.md 8e) is fused into the Adam kernel -- no NCCL call, no fences, no host involvement, the whole
 * loop stays one replayed CUDA graph.  The stand-alone
 * glamr_opt_backward / glamr_opt_apply never touch peer memory (the caller reduces reduce_buf between them).
 * world <= 1 clears the table.  All ranks must call glamr_opt_iterate with the same iteration counts; a rank that
 * waits ~20 s for a peer traps (CUDA error) instead of hanging. */
#define GLAMR_MAX_PEERS 8
int glamr_peer_alloc(size_t bytes, void** dev_ptr, unsigned char* ipc_handle_64_bytes);
int glamr_peer_open(const unsigned char* ipc_handle_64_bytes, void** dev_ptr);
int glamr_peer_close(void* dev_ptr);      /* a pointer from glamr_peer_open */
int glamr_peer_free(void* dev_ptr);       /* a pointer from glamr_peer_alloc */
size_t glamr_opt_peer_bytes(const glamr_opt_t* st);
int glamr_opt_set_peers(glamr_opt_t* st, int rank, int world, void* const* bufs /* [world], own buffer included */);
/* buf[0..count) <- element-wise sum over all ranks, in place, over the registered peer buffers (one kernel: every thread pushes
 * its elements to every rank, then polls its own buffer; count <= glamr_opt_reduce_count).  Collective: every rank calls it at the
 * same point of its stream order.  No-op for a single rank.  (SURVEY.md 8b `allreduce_inplace`; the per-iteration reduction of
 * glamr_opt_iterate is the same protocol fused into the Adam kernel.) */
int glamr_allreduce_inplace(glamr_opt_t* st, float* buf, size_t count, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Evaluation  --  stands behind global_recon/utils/evaluator.py:202-327 (Evaluator.prepare_seq).
 * glamr_sparse_regress: out[n,rows,3] = R @ vertices[n,V,3] for a regressor given in CSR form (row_ptr [rows+1], col_idx /
 *   weights [nnz], all DEVICE pointers) -- `torch.matmul(self.J_regressor, smpl_motion.vertices)` (:263,:306); the H36M
 *   regressor holds ~6 non-zeros per row.
 * glamr_procrustes_align: per frame, the similarity transform (scale, R, t) that maps S1 [n,J,3] closest to S2 [n,J,3],
 *   applied to S1 -> out [n,J,3]  (lib/utils/torch_transform.py:282-345 batch_compute_similarity_transform_torch; 3x3 SVD
 *   by one-sided Jacobi in fp64, reflection fixed through sign(det(U V^T))).
 * ---------------------------------------------------------------------------------------------------------- */
int glamr_sparse_regress(int n, int V, int rows, const int32_t* row_ptr, const int32_t* col_idx, const float* weights,
                         const float* vertices, float* out, void* stream);
int glamr_procrustes_align(int n, int J, const float* S1, const float* S2, float* out, void* stream);

/* device pointer + element count of an internal output buffer (valid until the handle is destroyed) */
int glamr_opt_read(glamr_opt_t* st, int what, const float** ptr, size_t* count);

#ifdef __cplusplus
}
#endif
#endif /* GLAMR_B200_H */
