/*
 * dexr.h -- C ABI of libdexr.so, the H100 (sm_90a) batched hand-retargeting solver.
 *
 * The reference (dexsuite/dex-retargeting) has no FFI layer: its hot path is the Python call
 *     SeqRetargeting.retarget()            src/dex_retargeting/seq_retarget.py:112-134
 *       -> Optimizer.retarget()            src/dex_retargeting/optimizer.py:77-102
 *            -> objective(x, grad)         src/dex_retargeting/optimizer.py:146-198 | 249-304 | 510-575
 *                 -> pinocchio FK/Jacobian src/dex_retargeting/robot_wrapper.py:82-95
 *                 -> mimic adaptor         src/dex_retargeting/kinematics_adaptor.py:102-113
 * driven by nlopt SLSQP, one frame at a time on one CPU core.  The entry points below are what a
 * binding for that path would call instead: one launch solves a whole batch of hand-frames (or of
 * frame sequences) on the GPU.  Plain C, opaque handle, raw device pointers, caller-owned buffers,
 * everything enqueued on the caller's stream without hidden synchronisation.  No torch types.
 *
 * Return convention: 0 on success, negative DEXR_E_* on failure; dexr_last_error() returns a
 * thread-local human readable message for the last failure.
 */
#ifndef DEXR_H_
#define DEXR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DEXR_VERSION 1

#define DEXR_MAX_LANES 32  /* movable joints (pinocchio DoFs incl. mimic + dummy), one per lane   */
#define DEXR_MAX_LINKS 16  /* links whose position enters the objective                             */
#define DEXR_MAX_GROUPS 16 /* robot groups per mixed launch (dexr_solve_frames_multi)                     */
#define DEXR_MAX_RES 16    /* residual blocks: vectors (vector / dexpilot) or points (position)     */
#define DEXR_MAX_GROUP 4   /* joints driven by one optimisation variable (itself + mimic joints)    */
#define DEXR_MAX_LINKS_PER_LANE 4 /* objective links rigidly attached to the same movable joint        */
#define DEXR_NUM_KEYPOINTS 21
#define DEXR_NO_INDEX (-1)

#define DEXR_LOSS_POSITION 0 /* optimizer.py:116-200  SmoothL1 per coordinate, mean over 3m       */
#define DEXR_LOSS_VECTOR 1   /* optimizer.py:203-306  SmoothL1 of |v - s t|, mean over m           */
#define DEXR_LOSS_DEXPILOT 2 /* optimizer.py:309-577  weighted, projected, hysteresis state        */

#define DEXR_E_INVALID (-1)  /* bad argument / table                                                */
#define DEXR_E_CUDA (-2)     /* a CUDA runtime call failed                                          */
#define DEXR_E_NODEVICE (-3) /* no sm_90 device                                                      */

/* Status word written per frame (status_out): low 16 bits = accepted LM iterations,
 * bits 16-22 = trial solves beyond the first per iteration (rejections, saturating at 127), bit 23 = ended at the fp32
 * floor of the KKT residual (informational), bit 24 = hit max_iters, bit 25 = non-finite input or state (output =
 * last_qpos, mirroring optimizer.py:99-102).  `status >> 24` != 0 means the frame needs attention. */
#define DEXR_STATUS_ITERS(s) ((s) & 0xffff)
#define DEXR_STATUS_REJECTS(s) (((s) >> 16) & 0x7f)
#define DEXR_STATUS_MAXITER (1 << 24)
#define DEXR_STATUS_NONFINITE (1 << 25)
/* informational, not a failure: the frame ended at the fp32 floor of its KKT residual (two consecutive steps below the
 * resolution of the objective brought no smaller gradient) before an accepted step fell below `tol` */
#define DEXR_STATUS_NOISEFLOOR (1 << 23)

/* ---------------------------------------------------------------------------------------------
 * Robot table: the flattened kinematic + objective description one solver instance needs.
 * Replaces: pinocchio Model/Data (robot_wrapper.py:15-23), Optimizer index maps
 * (optimizer.py:25-52), nlopt bounds (optimizer.py:54-60), MimicJointKinematicAdaptor tables
 * (kinematics_adaptor.py:46-100), the per-optimizer link index lists (optimizer.py:132-134,
 * 226-237, 384-395).  Built on the host by dex_retargeting_b200.table.compile_table().
 * Lane c <-> pinocchio DoF c (depth-first URDF order, fixed joints folded into `R0`/`p0`).
 * All matrices row-major, float32.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_table {
  uint32_t magic;      /* 'DXR1' = 0x31525844 */
  uint32_t nbytes;     /* sizeof(dexr_table_t), checked on upload */
  int32_t dof;         /* lanes in use = robot.dof (<= 32) */
  int32_t n_var;       /* optimised joints = len(target_joint_names) = opt_dof */
  int32_t n_fixed;     /* len(idx_pin2fixed): joints supplied by the caller per frame */
  int32_t n_links;     /* computed links */
  int32_t n_res;       /* residual blocks m */
  int32_t loss;        /* DEXR_LOSS_* */
  int32_t n_rounds;    /* pointer-jumping rounds = ceil(log2(max chain depth)) */
  int32_t has_mimic;   /* any lane with group_count > 1 or mimic source */
  int32_t num_fingers; /* dexpilot only */
  int32_t len_proj;    /* dexpilot: number of finger-pair vectors (S1 + S2) */
  int32_t len_s1;      /* dexpilot: pairs involving the first finger (thumb) */
  int32_t block_width; /* 0: dense Hessian.  4 / 8: the joints split into decoupled groups occupying aligned lane
                          windows of this width (no residual and no ancestor relation crosses a window), so the
                          Newton system is block diagonal.  4 (dof <= 16): all blocks are factorised side by side.
                          8, or 4 with dof > 16: accepted and factorised densely (there is no solver instantiation
                          for those widths); the result is the same minimiser */
  int32_t arrow;       /* 0: none.  1 + t: ARROW structure -- lanes 0..t-1 (t <= 8) are a trunk (free-flying base and / or
                          wrist) shared by decoupled fingers, each a contiguous run of <= 8 lanes whose first lane is an
                          ancestor of the others; every residual touches the trunk and at most one finger.  The Newton
                          system is then H = [F B; B^T W] with F block diagonal and is factorised finger by finger
                          (side by side) + a t x t Schur complement.  Requires block_width == 0, no mimic joints,
                          n_var == dof, dof > 16 */
  int32_t reserved;

  /* ---- per lane ---- */
  float R0[DEXR_MAX_LANES][9];    /* joint placement rotation in the parent joint frame          */
  float RA[DEXR_MAX_LANES][9];    /* R0 * K          (K = cross matrix of the joint axis)         */
  float RB[DEXR_MAX_LANES][9];    /* R0 * K * K      so R_local = R0 + sin q RA + (1-cos q) RB    */
  float p0[DEXR_MAX_LANES][3];    /* joint placement translation                                   */
  float d0[DEXR_MAX_LANES][3];    /* R0 * axis (prismatic direction in the parent joint frame)     */
  float axis[DEXR_MAX_LANES][3];  /* unit axis in the joint frame                                  */
  int32_t jtype[DEXR_MAX_LANES];  /* 0 revolute, 1 prismatic                                       */
  int32_t var_index[DEXR_MAX_LANES];   /* position in target_joint_names, or -1                    */
  int32_t fixed_index[DEXR_MAX_LANES]; /* position in fixed_qpos, or -1                            */
  int32_t mimic_src[DEXR_MAX_LANES];   /* lane of the source joint for a mimic joint, or -1        */
  float mimic_mult[DEXR_MAX_LANES];
  float mimic_off[DEXR_MAX_LANES];
  float lower[DEXR_MAX_LANES];    /* solver bounds: joint limit -/+ 1e-3 (optimizer.py:59-60)      */
  float upper[DEXR_MAX_LANES];
  float clip_lo[DEXR_MAX_LANES];  /* un-widened limits used to clip the warm start                 */
  float clip_hi[DEXR_MAX_LANES];  /* (seq_retarget.py:118-120)                                     */
  uint32_t jump[DEXR_MAX_LANES];  /* 5 x 6 bit: lane of the 2^r-th movable ancestor, 63 = none     */
  uint32_t anc_mask[DEXR_MAX_LANES];  /* bit i: lane i is this lane or one of its ancestors       */
  uint32_t desc_mask[DEXR_MAX_LANES]; /* bit i: this lane is lane i or one of its ancestors       */
  /* joints driven by the variable hosted on this lane (itself first), for the mimic fold          */
  int32_t group_count[DEXR_MAX_LANES];
  int32_t group_lane[DEXR_MAX_LANES][DEXR_MAX_GROUP];
  float group_mult[DEXR_MAX_LANES][DEXR_MAX_GROUP];

  /* ---- per computed link ---- */
  int32_t link_parent[DEXR_MAX_LINKS];   /* lane the link rides on, -1 = fixed to the world        */
  float link_off[DEXR_MAX_LINKS][3];     /* link origin in that joint frame (world if parent -1)   */
  uint32_t link_anc_mask[DEXR_MAX_LINKS]; /* anc_mask of link_parent (0 if world)                   */

  /* ---- per residual block ---- */
  int32_t res_task[DEXR_MAX_RES];    /* computed-link slot of the task link (or the point link)    */
  int32_t res_origin[DEXR_MAX_RES];  /* slot of the origin link, -1 for position residuals         */
  int32_t res_human_task[DEXR_MAX_RES];   /* keypoint id (0..20) of the task / point               */
  int32_t res_human_origin[DEXR_MAX_RES]; /* keypoint id of the origin, -1 for position            */
  /* dexpilot S2 pairs: indices into the S1 flags (optimizer.py:445-449) */
  int32_t s2_origin[DEXR_MAX_RES];
  int32_t s2_task[DEXR_MAX_RES];
} dexr_table_t;

/* Loss / solver parameters (optimizer ctor arguments + solver knobs). */
typedef struct dexr_params {
  float huber_delta;  /* beta of SmoothL1Loss */
  float norm_delta;   /* weight of |x - last_qpos|^2 */
  float scaling;      /* vector / dexpilot: human -> robot scale */
  float project_dist; /* dexpilot, optimizer.py:344 */
  float escape_dist;  /* dexpilot, optimizer.py:345 */
  float eta1;         /* dexpilot, optimizer.py:346 */
  float eta2;         /* dexpilot, optimizer.py:347 */
  float lp_alpha;     /* sequences only: low-pass alpha; outside [0,1] = no filter */
  float tol;          /* stop when the accepted step is below this (rad / m); default 1e-5 */
  float lambda0;      /* initial LM damping; default 1e-2 */
  int32_t max_iters;  /* cap on accepted iterations; default 64 */
  int32_t clip_init;  /* 1: clip the warm start to clip_lo/clip_hi first (SeqRetargeting.retarget) */
  int32_t preprocess; /* keypoints mode only.  0: `keypoints` are wrist-centred MANO-convention points (what the reference's
                       * detector hands to the retargeting).  1 (right hand) / 2 (left hand): `keypoints` are RAW detector
                       * landmarks and the solver prelude applies example/vector_retargeting/single_hand_detector.py:100-103,
                       * 130-158 itself -- wrist frame from landmarks {0,5,9}, rotation into it and into the MANO convention
                       * (constants.py:7-21) -- to the few keypoints the objective reads: no separate launch, no second
                       * 252 B / frame round trip through HBM (dexr_preprocess_keypoints remains for callers that want the
                       * transformed frames themselves) */
} dexr_params_t;

/* Buffers of one batched solve.  All pointers are DEVICE pointers (or NULL where noted); rows are
 * contiguous.  Exactly one of `keypoints` / `ref_value` is non-NULL. */
typedef struct dexr_frames {
  const float* keypoints;  /* [B,21,3]  raw human keypoints; the reference's caller-side gather     */
                           /*           (example/profiling/profile_online_retargeting.py:24-30) is  */
                           /*           done in the kernel with the table's human indices           */
  const float* ref_value;  /* [B,m,3]   what Optimizer.retarget() receives                          */
  const float* fixed_qpos; /* [B,n_fixed] or NULL when n_fixed == 0                                 */
  const float* last_qpos;  /* [B,n_var] warm start AND regularisation anchor (optimizer.py:77-98)   */
  uint8_t* projected;      /* [B,len_proj] dexpilot hysteresis flags, read and updated; else NULL   */
  float* qpos_out;         /* [B,n_var] solution, target_joint_names order                          */
  float* robot_qpos_out;   /* [B,dof] or NULL: full qpos in pinocchio order, mimic applied          */
  int32_t* status_out;     /* [B] or NULL */
  float* cost_out;         /* [B] or NULL: final consistent objective value                         */
  float* damping_io;       /* [B] or NULL.  Stream state for callers that feed a stream frame by frame (the reference's
                            * teleoperation loop, one retarget() per camera frame): in = the Levenberg-Marquardt damping
                            * this frame starts with (<= 0: params.lambda0), out = what the stream's NEXT frame should
                            * start with (0.3 x the damping this frame's first accepted step needed, never below
                            * params.lambda0).  NULL: every frame starts at params.lambda0.  The minimiser found is the
                            * same; the state only saves the rejected steps a hard stretch of a trajectory would pay
                            * again at the start of every frame.                                                        */
} dexr_frames_t;

/* Buffers of one batched sequence solve: S independent streams of T frames with
 * SeqRetargeting.retarget semantics carried inside the kernel (seq_retarget.py:112-134):
 * clip(last) -> solve -> last := solution -> scatter + mimic -> low-pass filter. */
typedef struct dexr_sequences {
  const float* keypoints;  /* [S,T,21,3] */
  const float* fixed_qpos; /* [S,T,n_fixed] or NULL */
  float* last_qpos;        /* [S,n_var]  in: initial warm start; out: last solution                 */
  float* filter_state;     /* [S,dof]    in/out low-pass state y (ignored when no filter)           */
  uint8_t* filter_init;    /* [S]        in/out LPFilter.is_init                                    */
  uint8_t* projected;      /* [S,len_proj] in/out dexpilot flags, or NULL                           */
  float* robot_qpos_out;   /* [S,T,dof]  filtered full qpos, pinocchio order                        */
  int32_t* status_out;     /* [S,T] or NULL */
  float* damping_state;    /* [S] in/out or NULL: the streams' carried damping (dexr_frames_t.damping_io); inside a call
                            * it is carried in registers from frame to frame whether or not this array is given           */
} dexr_sequences_t;

typedef struct dexr_robot dexr_robot_t; /* opaque: device copy of the table + launch configuration */

typedef struct dexr_launch_info {
  int32_t grid, block, smem_bytes, frames_per_tile, lanes_per_frame, consumer_warps, kernels_launched;
} dexr_launch_info_t;

int dexr_version(void);
/* 16 hex digits: sha256 over the sources this library was compiled from (csrc/dexr.cu, csrc/dexr_kernels.cuh,
 * include/dexr.h) and the compile-time switches, stamped by dex_retargeting_b200/build.py.  Profiler captures
 * (profiles/roofline_traffic.json) record it so that a number is never attributed to another binary. */
const char* dexr_build_id(void);
const char* dexr_last_error(void);
size_t dexr_table_sizeof(void);
size_t dexr_params_sizeof(void);
size_t dexr_frames_sizeof(void);    /* sizeof(dexr_frames_t) / sizeof(dexr_sequences_t): a binding checks its mirror of the  */
size_t dexr_sequences_sizeof(void); /* buffer structs against the library it loaded (dexr_group_t embeds dexr_frames_t)  */
void dexr_default_params(dexr_params_t* p);

/* Upload a host table to `device` (cudaMemcpy, synchronous; init time only). */
int dexr_robot_create(const dexr_table_t* table_host, int device, dexr_robot_t** out);
/* Adopt a table already resident on `device` (e.g. received by an NCCL broadcast): copies it
 * device-to-device into the handle and reads the header back to size the launches. */
int dexr_robot_create_from_device(const void* table_dev, size_t nbytes, int device, dexr_robot_t** out);
const void* dexr_robot_device_table(const dexr_robot_t* robot);
void dexr_robot_destroy(dexr_robot_t* robot);

/* Independent frames: replaces B calls of Optimizer.retarget() (optimizer.py:77-102). */
int dexr_solve_frames(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_frames_t* io,
                      int64_t num_frames, void* cuda_stream);
/* Mixed robots: several (robot, batch) groups solved by ONE persistent launch -- replaces one Optimizer per robot run one
 * after the other (retargeting_config.py:167-257 builds exactly one optimizer per config).  Every group has its own table,
 * parameters and buffers (all on the same device); results are bit-identical to one dexr_solve_frames call per group.
 * The groups run as one launch each on library-owned side streams forked from / joined into `cuda_stream` with events (small
 * grids side by side, large ones overlapping their tails); DEXR_MULTI_MODE=persistent selects the single persistent kernel
 * whose CTAs walk the groups instead (measured slower on H100, see csrc/dexr.cu).  Either way the call is asynchronous and
 * ordered on `cuda_stream`. */
typedef struct dexr_group {
  const dexr_robot_t* robot;
  const dexr_params_t* params;
  dexr_frames_t io;
  int64_t num_frames;
} dexr_group_t;
int dexr_solve_frames_multi(const dexr_group_t* groups, int32_t num_groups, void* cuda_stream);
/* Streams: replaces S x T calls of SeqRetargeting.retarget() (seq_retarget.py:112-134). */
int dexr_solve_sequences(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                         int64_t num_streams, int64_t num_steps, void* cuda_stream);
/* Same as dexr_solve_frames but every pointer in `io` is a HOST pointer; returns when the results are in
 * the host buffers.  Page-locked buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory) take the
 * zero-copy path: one launch whose producer warps bulk-copy the input tiles from host memory over PCIe
 * into shared memory while the consumers solve, results stored directly to host memory.  Pageable
 * buffers (and DexPilot flag buffers) are staged in chunks through library-owned device buffers on two
 * internal streams. */
int dexr_solve_frames_host(dexr_robot_t* robot, const dexr_params_t* params, const dexr_frames_t* io_host,
                           int64_t num_frames);
/* Keypoint pre-processing, the step right before the hot path in the reference's teleoperation pipeline
 * (example/vector_retargeting/single_hand_detector.py:100-103 and :130-158): centre the 21 detector landmarks at
 * the wrist, estimate the wrist frame from landmarks {0,5,9} (plane normal + Gram-Schmidt, sign fixed by the
 * index->middle direction), rotate into it and into the MANO convention (constants.py:7-21).
 * raw [B,21,3] -> out [B,21,3]; wrist_rot_out [B,3,3] (the estimated frame, row-major) may be NULL.
 * hand_type: 0 = right, 1 = left.  Degenerate (collinear) landmarks produce NaN, which the solver then flags.
 * Independent of any robot: no handle.  HBM-bound (252 B in + 252 B out per frame). */
int dexr_preprocess_keypoints(const float* raw, float* out, float* wrist_rot_out, int hand_type, int64_t num_frames,
                              int device, void* cuda_stream);
/* Launch geometry of the last call on this handle (diagnostics / bench reporting). */
int dexr_get_launch_info(const dexr_robot_t* robot, dexr_launch_info_t* out);

#ifdef __cplusplus
}
#endif
#endif /* DEXR_H_ */
