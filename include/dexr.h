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

/* ---------------------------------------------------------------------------------------------
 * Objective evaluation: the value and gradient of the retargeting objective at GIVEN joint vectors, no solve.  Replaces B
 * calls of the closure returned by Optimizer.get_objective_function (optimizer.py:104-108, implemented at :138-200,
 * :241-306, :456-577): scoring recorded or foreign joint trajectories against human keypoints, and the objective as a
 * training loss.  Targets are prepared exactly as by dexr_solve_frames (keypoint gather, params.preprocess, scaling,
 * DexPilot flags and weights); the call reads the loss fields of `params` and `preprocess`, and ignores tol, lambda0,
 * max_iters, clip_init and lp_alpha.  Asynchronous on `cuda_stream`, allocates nothing; num_frames == 0 does nothing.
 * A frame with a non-finite input gets non-finite outputs; no other frame changes.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_eval {
  const float* keypoints;  /* [B,21,3] or NULL  } exactly one of the two; raw landmarks with params.preprocess     */
  const float* ref_value;  /* [B,m,3]  or NULL  }                                                                     */
  const float* fixed_qpos; /* [B,n_fixed] or NULL when n_fixed == 0                                                   */
  const float* qpos;       /* [B,n_var] the point of evaluation, target_joint_names order, used as given (no clipping) */
  const float* last_qpos;  /* [B,n_var] anchor of the norm_delta term, or NULL: no regulariser                        */
  uint8_t* projected;      /* [B,len_proj] DexPilot flags, read and updated as by dexr_solve_frames; NULL: start false */
  float* loss_out;         /* [B] or NULL: L(x), what the reference's closure returns                                 */
  float* cost_out;         /* [B] or NULL: L(x) + norm_delta |x - last|^2, the quantity dexr_frames_t.cost_out reports */
  float* grad_out;         /* [B,n_var] or NULL: gradient of cost_out = the reference closure's grad                   */
} dexr_eval_t;
size_t dexr_eval_sizeof(void);
int dexr_eval_objective(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_eval_t* io,
                        int64_t num_frames, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through the solve (vector-Jacobian product of the implicit function theorem).  At a point x of frame f
 * (normally what dexr_solve_frames returned for the same inputs) and a cotangent dl/dx, writes dl/dtheta for the frame's
 * inputs theta: the keypoints or ref_value, the fixed joints and the anchor last_qpos.  x is taken as a stationary point of
 * F(x) = L(x) + norm_delta |x - last_qpos|^2 on its free variables: a variable at a (widened) bound whose gradient does not
 * point inward is active and gets zero sensitivity; for the free ones v = H_ff^-1 dl/dx_f with H the exact Hessian of F
 * (exact Huber curvature, kinematic curvature, mimic fold), and every input cotangent is -(dg/dtheta)^T v.  A frame that
 * ended at max_iters gets the derivative of this linearisation at the point given.  Targets are prepared as by the solve:
 * DexPilot flags are read from `projected` (normally the flags the solve left) and never written; flags and Huber zones are
 * piecewise constant, so the derivative is the one-sided one at a switch.  params.preprocess must be 0 (raw landmarks are not
 * differentiated).  Asynchronous on `cuda_stream`, allocates nothing; num_frames == 0 does nothing.  A frame with a
 * non-finite input gets non-finite outputs and DEXR_STATUS_NONFINITE; a frame whose free Hessian is not positive definite
 * (not a strict local minimum) gets zero cotangents and DEXR_STATUS_NOT_PD.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
#define DEXR_STATUS_NOT_PD (1 << 26)
typedef struct dexr_vjp {
  const float* keypoints;   /* [B,21,3] or NULL  } exactly one of the two                                            */
  const float* ref_value;   /* [B,m,3]  or NULL  }                                                                   */
  const float* fixed_qpos;  /* [B,n_fixed] or NULL when n_fixed == 0                                                 */
  const float* qpos;        /* [B,n_var] the point x                                                                 */
  const float* last_qpos;   /* [B,n_var] the anchor of the norm_delta term, or NULL: no regulariser                  */
  const uint8_t* projected; /* [B,len_proj] DexPilot flags, read only; NULL: every flag as prepare_targets sets it from 0 */
  const float* grad_qpos;   /* [B,n_var] dl/dx                                                                       */
  float* grad_keypoints;    /* [B,21,3] or NULL: dl/dkeypoints (keypoints form only; all 63 entries written)         */
  float* grad_ref_value;    /* [B,m,3]  or NULL: dl/dref_value (ref_value form only)                                 */
  float* grad_fixed_qpos;   /* [B,n_fixed] or NULL                                                                   */
  float* grad_last_qpos;    /* [B,n_var] or NULL: dl/dlast_qpos (needs last_qpos)                                    */
  int32_t* status_out;      /* [B] or NULL: 0, DEXR_STATUS_NONFINITE or DEXR_STATUS_NOT_PD                           */
} dexr_vjp_t;
size_t dexr_vjp_sizeof(void);
int dexr_solve_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_vjp_t* io, int64_t num_frames,
                   void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through the sequence solve.  dexr_solve_sequences_tape is dexr_solve_sequences (same kernel code, same
 * results bit for bit) that also records what the backward needs: every frame's UNFILTERED solution x_t and, for DexPilot,
 * the hysteresis flags the frame left (DexPilot needs io->projected then).  dexr_solve_sequences_vjp then runs the
 * reverse-time recurrence of every stream in one launch, a group of lanes per stream walking t = T-1 .. 0:
 *   a_t = clip(x_{t-1}) (clip_lo / clip_hi), x_t = solve(kp_t, fixed_t, anchor a_t), q_t = scatter + mimic of x_t,
 *   y_t = init_t ? y_{t-1} + alpha (q_t - y_{t-1}) : q_t with init_t = t > 0 or filter_init, robot_qpos[t] = y_t (or q_t);
 * each frame is differentiated as by dexr_solve_vjp at (x_t, anchor a_t, the recorded flags), the anchor cotangent flows to
 * x_{t-1} where clip_lo <= x_{t-1} <= clip_hi, and the filter's cotangent is carried in registers.  The DexPilot flags, the
 * carried damping and the basin the warm start picks are not differentiated.  A frame with a non-finite input or cotangent
 * gets non-finite outputs and DEXR_STATUS_NONFINITE, and so does every earlier frame of its stream (other streams are
 * untouched); DEXR_STATUS_NOT_PD frames get zero cotangents and cut the chain through the anchor.  params as given to the
 * forward (lp_alpha selects the filter, clipping is implied); params.preprocess must be 0.  Both calls are asynchronous on
 * `cuda_stream`, allocate nothing and do nothing for 0 streams or 0 steps.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_sequences_tape {
  float* qpos;        /* [S,T,n_var] every frame's unfiltered solution                      */
  uint8_t* projected; /* [S,T,len_proj] DexPilot flags after every frame, or NULL           */
} dexr_sequences_tape_t;
size_t dexr_sequences_tape_sizeof(void);
int dexr_solve_sequences_tape(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                              const dexr_sequences_tape_t* tape, int64_t num_streams, int64_t num_steps, void* cuda_stream);

typedef struct dexr_sequences_vjp {
  const float* keypoints;             /* [S,T,21,3] as given to the forward (preprocess must be 0)   */
  const float* fixed_qpos;            /* [S,T,n_fixed] or NULL when n_fixed == 0                     */
  const float* last_qpos;             /* [S,n_var] the warm start BEFORE the forward call            */
  const uint8_t* filter_init;         /* [S] LPFilter.is_init before the forward call (filter only)  */
  const float* qpos;                  /* [S,T,n_var] tape                                            */
  const uint8_t* projected;           /* [S,T,len_proj] tape, DexPilot only                          */
  const float* grad_robot_qpos;       /* [S,T,dof] or NULL (= 0)                                     */
  const float* grad_last_qpos_out;    /* [S,n_var] dl/d final last_qpos, or NULL                     */
  const float* grad_filter_state_out; /* [S,dof] dl/d final filter_state, or NULL                    */
  float* grad_keypoints;              /* [S,T,21,3] or NULL                                          */
  float* grad_fixed_qpos;             /* [S,T,n_fixed] or NULL                                       */
  float* grad_last_qpos;              /* [S,n_var] or NULL: dl/d initial last_qpos                   */
  float* grad_filter_state;           /* [S,dof] or NULL: dl/d initial filter_state                  */
  int32_t* status_out;                /* [S,T] or NULL: 0, NONFINITE or NOT_PD                       */
} dexr_sequences_vjp_t;
size_t dexr_sequences_vjp_sizeof(void);
int dexr_solve_sequences_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_vjp_t* io,
                             int64_t num_streams, int64_t num_steps, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Per-frame Jacobians of the solve: J = dx/dtheta of frame f's solution x with respect to its inputs theta (the keypoints
 * or ref_value, the fixed joints and the anchor last_qpos), in one launch for all frames.  Row i of every block is exactly
 * what dexr_solve_vjp writes for the same frame with grad_qpos = e_i (the unit cotangent of variable i), so everything is
 * the VJP's: the point, the anchor, the read-only DexPilot flags, the solver's active-set rule, the exact Hessian, the
 * one-sided derivative at a Huber zone or flag switch, and the status bits.  Hence: the rows of active variables are zero;
 * the anchor block is 2 norm_delta H_ff^-1, with zero rows and columns for the active variables; a DEXR_STATUS_NOT_PD frame
 * gets all zeros and a frame with a non-finite input gets NaN and DEXR_STATUS_NONFINITE (no other frame changes).  The
 * Hessian is factorised once per frame and every free variable's row reuses the factor.  Uncertainty propagation is
 * Sigma_q = J Sigma_theta J^T.  params.preprocess must be 0 (raw landmarks are not differentiated).  Asynchronous on
 * `cuda_stream`, allocates nothing; num_frames == 0 does nothing.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_jacobian {
  const float* keypoints;   /* [B,21,3] or NULL  } exactly one of the two                                            */
  const float* ref_value;   /* [B,m,3]  or NULL  }                                                                   */
  const float* fixed_qpos;  /* [B,n_fixed] or NULL when n_fixed == 0                                                 */
  const float* qpos;        /* [B,n_var] the point x                                                                 */
  const float* last_qpos;   /* [B,n_var] anchor of the norm_delta term, or NULL: no regulariser                      */
  const uint8_t* projected; /* [B,len_proj] DexPilot flags, read only; NULL as in dexr_vjp_t                         */
  float* jac_keypoints;     /* [B,n_var,21,3] or NULL (keypoints form only; all 63 columns written)                  */
  float* jac_ref_value;     /* [B,n_var,m,3]  or NULL (ref_value form only)                                          */
  float* jac_fixed_qpos;    /* [B,n_var,n_fixed] or NULL                                                             */
  float* jac_last_qpos;     /* [B,n_var,n_var] or NULL (needs last_qpos)                                             */
  int32_t* status_out;      /* [B] or NULL: 0, DEXR_STATUS_NONFINITE or DEXR_STATUS_NOT_PD                           */
} dexr_jacobian_t;
size_t dexr_jacobian_sizeof(void);
int dexr_solve_jacobian(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_jacobian_t* io,
                        int64_t num_frames, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Packed streams: S streams of ANY lengths in one launch, their frames laid end to end (the cu_seqlens layout).  Stream s
 * owns frames offsets[s] .. offsets[s+1]-1 of every per-frame array; N = num_frames.  The buffer structs are those of the
 * rectangular calls with these shapes:
 *   dexr_sequences_t:      keypoints [N,21,3], fixed_qpos [N,n_fixed], robot_qpos_out [N,dof], status_out [N];
 *                          last_qpos [S,n_var], filter_state [S,dof], filter_init [S], projected [S,len_proj],
 *                          damping_state [S] (per stream, as before)
 *   dexr_sequences_tape_t: qpos [N,n_var], projected [N,len_proj]
 *   dexr_sequences_vjp_t:  keypoints, fixed_qpos, qpos, projected, grad_robot_qpos, grad_keypoints, grad_fixed_qpos,
 *                          status_out [N,...]; last_qpos, filter_init, grad_last_qpos_out, grad_filter_state_out,
 *                          grad_last_qpos, grad_filter_state [S,...]
 * Per stream everything is exactly what dexr_solve_sequences / _tape / _vjp do (a stream's results and final state are
 * bit-identical to a rectangular call on that stream alone).  A stream of length 0 leaves its state untouched; in the
 * backward its state cotangents pass through unchanged.  `tape` NULL: not recorded (raw landmarks, params.preprocess,
 * are accepted only then).  Streams are dealt to warps in index order.  offsets is a DEVICE array and is not checked on
 * the host: a stream whose range is malformed (offsets[s] < 0, offsets[s] > offsets[s+1] or offsets[s+1] > N) is treated
 * as an empty stream, so no layout makes the kernels read or write out of range.
 * num_frames == 0 does nothing.  Asynchronous on `cuda_stream`, allocates nothing.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
int dexr_solve_sequences_packed(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_t* io,
                                const dexr_sequences_tape_t* tape /* NULL: not recorded */,
                                const int64_t* offsets /* device [S+1] */, int64_t num_streams, int64_t num_frames, void* cuda_stream);
int dexr_solve_sequences_packed_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_sequences_vjp_t* io,
                                    const int64_t* offsets, int64_t num_streams, int64_t num_frames, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Offline trajectory smoothing of packed streams: every frame of a stream solved JOINTLY.  Per stream of T frames,
 *   F(X) = sum_t L_t(x_t) + w sum_{t>=1} |x_t - x_{t-1}|^2 + w |x_0 - clip(a)|^2,   x_t in [lower, upper] (widened bounds)
 * with L_t the per-frame loss of the solve (position / vector / DexPilot, mimic and fixed joints), a the stream's warm start
 * (last_qpos; NULL: no anchor term) clipped to clip_lo / clip_hi, and w = smooth_weight (< 0: params.norm_delta).  With
 * w = norm_delta, F is the sum of the costs the causal solve (dexr_solve_sequences_packed) minimises one frame at a time;
 * the joint minimiser has no lag.  One group of lanes per stream runs a damped projected Newton method on F: the Hessian is
 * block tridiagonal (diagonal blocks the exact per-frame Hessians + 2 w k_t I, k_t the frame's neighbours with the anchor
 * counting as one; off-diagonal blocks -2 w I), eliminated along the clip by block Thomas.
 *   Layout: packed only, with the offsets and malformed-range rules of dexr_solve_sequences_packed (an equal-length batch is
 *     the rectangular layout); keypoints, fixed_qpos, qpos_init, qpos_out, robot_qpos_out, status_out [N,...];
 *     last_qpos, projected, cost_out [S,...].  A stream of length 0 writes nothing.
 *   DexPilot: frame t uses the flags the causal packed solve leaves at frame t -- the hysteresis recurrence, which reads only
 *     the human vectors, walked along the clip from projected[s].  The flags are not optimised; projected is never written.
 *   Missing frames: a frame with a non-finite keypoint coordinate or fixed joint has no data term and gets
 *     DEXR_STATUS_MISSING; its output is what the smoothness terms give: an interior gap the linear interpolation (in
 *     variable space) of the frames on either side, a trailing gap the last observed frame, a leading gap the
 *     interpolation from the clipped anchor (the first observed frame repeated when there is no anchor).
 *   Non-finite start: a stream whose qpos_init (or anchor, when given) is non-finite gets qpos_init back, every frame of it
 *     DEXR_STATUS_NONFINITE and cost NaN; no other stream changes.
 *   Status: the low 16 bits hold the stream's accepted outer iterations and bits 16-22 its rejected trials and restarted
 *     eliminations (saturating at 127), on every frame of the stream; DEXR_STATUS_MAXITER after params.max_iters accepted
 *     outer iterations.  params.tol is the stopping step (max |delta| over the stream), params.lambda0 the initial damping
 *     (x 0.1 after an accepted step, x 10 after a rejected one).  An elimination that meets a pivot <= 0 (an indefinite
 *     exact Hessian) is restarted with the Gauss-Newton model, then with more damping; it uses up no outer iteration.
 *   The starting trajectory is clipped to the widened bounds.  Raw landmarks (params.preprocess != 0) are refused.
 *   `workspace`: device scratch of at least dexr_smooth_workspace_bytes(robot, num_frames) bytes (DEXR_E_INVALID below);
 *   the call allocates nothing and never synchronises.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
#define DEXR_STATUS_MISSING (1 << 27) /* smoother: the frame's inputs were non-finite; its output is interpolated by the
                                         smoothness terms alone (informational, not a failure) */
typedef struct dexr_smooth {
  const float* keypoints;   /* [N,21,3] wrist-centred MANO keypoints (params.preprocess must be 0)                   */
  const float* fixed_qpos;  /* [N,n_fixed] or NULL when n_fixed == 0                                                   */
  const float* last_qpos;   /* [S,n_var] warm start a of each stream (clipped to clip_lo/clip_hi), or NULL: no anchor term */
  const uint8_t* projected; /* [S,len_proj] DexPilot flags at the start of each stream, read only (NULL: all false)   */
  const float* qpos_init;   /* [N,n_var] starting trajectory, normally the tape of dexr_solve_sequences_packed           */
  float* qpos_out;          /* [N,n_var] the answer (may equal qpos_init): the minimiser unless DEXR_STATUS_MAXITER    */
  float* robot_qpos_out;    /* [N,dof] or NULL: scatter + mimic of qpos_out, NO low-pass filter                        */
  int32_t* status_out;      /* [N] or NULL                                                                              */
  float* cost_out;          /* [S] or NULL: F at the answer                                                             */
  float smooth_weight;      /* w; < 0: params.norm_delta                                                                */
  void* workspace;          /* device scratch of at least dexr_smooth_workspace_bytes(robot, num_frames) bytes          */
  size_t workspace_bytes;
} dexr_smooth_t;
size_t dexr_smooth_sizeof(void);
size_t dexr_smooth_workspace_bytes(const dexr_robot_t* robot, int64_t num_frames);
int dexr_smooth_sequences_packed(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_smooth_t* io,
                                 const int64_t* offsets /* device [S+1] */, int64_t num_streams, int64_t num_frames,
                                 void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through the offline smoother: the implicit-function VJP of dexr_smooth_sequences_packed's answer with
 * respect to the keypoints, the fixed joints and the anchor, every packed stream in one launch.  Per stream, X* = (x_0 ..
 * x_{T-1}) (`qpos`, the smoother's answer) is taken as a stationary point, on its free variables, of the smoother's
 *   F(X; theta) = sum_t L_t(x_t; kp_t, fixed_t) + w sum_{t>=1} |x_t - x_{t-1}|^2 + w |x_0 - clip(a)|^2,
 * theta = (keypoints, fixed joints, anchor a), w = smooth_weight (< 0: params.norm_delta).  Given G = dl/dX:
 *   1. G_t = grad_qpos_t + M^T grad_robot_qpos_t (mimic followers folded into their source; a fixed joint's share of
 *      grad_robot_qpos goes straight to grad_fixed_qpos);
 *   2. the active set is the smoother's rule on the TOTAL gradient (data + smoothness + anchor) at X*, at the widened bounds:
 *      active variables get zero sensitivity;
 *   3. H V = G over the free variables, H the exact block-tridiagonal Hessian of F (diagonal blocks D_t = M^T H_q M +
 *      2 w k_t I, k_t the frame's neighbours with the anchor counting as one; off-diagonal blocks -2 w I; no damping, no
 *      Gauss-Newton fallback), by block Thomas along the clip: S_t = D_t - (2w)^2 Z_{t-1}, y_t = G_t + 2w Z_{t-1} y_{t-1},
 *      then v_t = Z_t (y_t + 2w v_{t+1}), Z_t the inverse of S_t over the free variables of frame t;
 *   4. theta_bar = -(dg/dtheta)^T V, frame by frame: grad_keypoints_t is dexr_solve_vjp's target pass run with v_t,
 *      grad_fixed_qpos_t = -H_q[c, :] . M v_t plus the direct term of step 1, and the anchor's
 *      grad_last_qpos = 2 w v_0 where clip_lo <= a <= clip_hi (inclusive, as torch.clamp), 0 elsewhere.
 * Not differentiated: the DexPilot flags (the forward's hysteresis recurrence along the clip from projected[s], read only),
 * the starting trajectory (it only picks the basin) and w.  The gradient is NOT causal: a loss on frame t reaches the
 * keypoints of every frame of its stream.
 *   NOT_PD: at a strict local minimum the stacked free Hessian is positive definite, and so is every Schur complement; a
 *     pivot <= 0 anywhere in the elimination means X* is not one.  That stream gets zero cotangents and DEXR_STATUS_NOT_PD
 *     on every frame.  A stream the forward left at DEXR_STATUS_MAXITER gets the derivative of the linearisation at the
 *     point given.
 *   NONFINITE: the solve couples all frames of a stream, so a non-finite qpos, anchor or cotangent makes the whole stream's
 *     cotangents NaN (grad_last_qpos included) with DEXR_STATUS_NONFINITE; other streams are not affected.
 *   Missing frames (a non-finite keypoint or fixed joint: DEXR_STATUS_MISSING, as in the forward) have no data term but
 *     still carry the chain through their smoothness terms; their keypoint and fixed-joint cotangents are 0, not NaN.
 *   status_out: 0, DEXR_STATUS_NOT_PD or DEXR_STATUS_NONFINITE, | DEXR_STATUS_MISSING on a missing frame.
 *   Layout: the packed rules of dexr_smooth_sequences_packed; an empty or malformed range writes nothing in the per-frame
 *     arrays, and its grad_last_qpos row is 0.  Raw landmarks (params.preprocess != 0) are refused.
 *   `workspace`: the forward's, at least dexr_smooth_workspace_bytes(robot, num_frames) bytes (DEXR_E_INVALID below): Z_t,
 *     y_t and v_t fit in its per-frame block.  The call is asynchronous on `cuda_stream` and allocates nothing.  All
 *     pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_smooth_vjp {
  const float* keypoints;       /* [N,21,3] as given to the forward                                                     */
  const float* fixed_qpos;      /* [N,n_fixed] or NULL when n_fixed == 0                                                */
  const float* last_qpos;       /* [S,n_var] the anchor a as given to the forward, or NULL: no anchor term              */
  const uint8_t* projected;     /* [S,len_proj] DexPilot flags at the start of each stream, as given to the forward     */
  const float* qpos;            /* [N,n_var] the smoother's answer X*                                                   */
  const float* grad_qpos;       /* [N,n_var] dl/dqpos, or NULL (= 0)                                                    */
  const float* grad_robot_qpos; /* [N,dof] dl/drobot_qpos, or NULL (= 0)                                                */
  float smooth_weight;          /* w as given to the forward; < 0: params.norm_delta                                    */
  void* workspace;              /* device scratch of at least dexr_smooth_workspace_bytes(robot, num_frames) bytes      */
  size_t workspace_bytes;
  float* grad_keypoints;        /* [N,21,3] (all 63 entries of every frame of a non-empty stream written)               */
  float* grad_fixed_qpos;       /* [N,n_fixed] or NULL                                                                  */
  float* grad_last_qpos;        /* [S,n_var] or NULL (needs last_qpos)                                                  */
  int32_t* status_out;          /* [N] or NULL                                                                          */
} dexr_smooth_vjp_t;
size_t dexr_smooth_vjp_sizeof(void);
int dexr_smooth_sequences_packed_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_smooth_vjp_t* io,
                                     const int64_t* offsets /* device [S+1] */, int64_t num_streams, int64_t num_frames,
                                     void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Offline smoothing with an acceleration penalty: dexr_smooth_sequences_packed on
 *   F_c(X) = F(X) + c sum_{triples (t-1, t, t+1) of the stream} |x_{t+1} - 2 x_t + x_{t-1}|^2,
 * F the smoother's objective above and c = accel_weight (finite, >= 0).  With an anchor the clipped anchor is frame -1, so the
 * sum includes |x_1 - 2 x_0 + clip(a)|^2; a stream of fewer than two frames (three without an anchor) has no triple.  A
 * constant-velocity trajectory costs nothing under the new term, so it damps jitter without pulling motion to a standstill
 * the way raising w does; w = 0 with c > 0 is allowed.
 *   The Hessian is block pentadiagonal: diagonal blocks gain 2 c m_t I (m_t the sum of the squared coefficients (1, -2, 1)
 *   of frame t over its triples), the blocks beside them -4 c I per triple holding both frames, the blocks two away 2 c I.
 *   It is eliminated by a banded block LDL^T along the clip: Z_t, the inverse of the Schur complement over frame t's free
 *   variables, and the dense coupling block E_t between t and t+1 per frame; the back substitution's d_t reads d_{t+1} and
 *   d_{t+2}.  Everything else -- the active set on the total gradient, the damping (x 0.1 / x 10), the acceptance rule, the
 *   Gauss-Newton then more-damping restarts on a pivot <= 0, params.max_iters on accepted iterations, the DexPilot flag
 *   walk, NONFINITE isolation per stream, status and layout -- is dexr_smooth_sequences_packed's.  A missing frame has no
 *   data term; its value is what the smoothness terms give (with c > 0 no longer the linear interpolation).  cost_out
 *   holds F_c at the answer.
 *   accel_weight == 0 runs dexr_smooth_sequences_packed itself (the same bits, and its workspace size suffices).  A
 *   non-finite or negative accel_weight returns DEXR_E_INVALID, and so does a workspace below
 *   dexr_smooth_accel_workspace_bytes(robot, num_frames) when accel_weight > 0 (the io's workspace fields).  The call is
 *   asynchronous on `cuda_stream`, allocates nothing and never synchronises.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
size_t dexr_smooth_accel_workspace_bytes(const dexr_robot_t* robot, int64_t num_frames); /* >= dexr_smooth_workspace_bytes */
int dexr_smooth_sequences_packed_accel(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_smooth_t* io,
                                       float accel_weight, const int64_t* offsets /* device [S+1] */, int64_t num_streams,
                                       int64_t num_frames, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through the acceleration-penalised smoother: dexr_smooth_sequences_packed_vjp for F_c (c = accel_weight,
 * as given to the forward; c is not differentiated).  Step 3 solves H V = G with the exact block-pentadiagonal Hessian of
 * F_c over the free variables, by the forward's banded elimination with no damping and no fallback; step 4 is unchanged
 * except for the anchor: grad_last_qpos = 2 w v_0 + 4 c v_0 - 2 c v_1 where clip_lo <= a <= clip_hi (0 elsewhere), the c
 * terms only when the stream has a second frame (the triple (a, x_0, x_1)).  NOT_PD, NONFINITE, MISSING, status and layout
 * keep their meanings.  accel_weight == 0 runs dexr_smooth_sequences_packed_vjp itself; a non-finite or negative one, or a
 * workspace below dexr_smooth_accel_workspace_bytes(robot, num_frames) when accel_weight > 0, returns DEXR_E_INVALID.
 * Asynchronous on `cuda_stream`, allocates nothing; all pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
int dexr_smooth_sequences_packed_accel_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_smooth_vjp_t* io,
                                           float accel_weight, const int64_t* offsets /* device [S+1] */,
                                           int64_t num_streams, int64_t num_frames, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Fixed-lag smoothing of live streams: every new frame re-solves the last L+1 frames of its stream jointly with the offline
 * smoother and emits the frame L ticks back.  A stream trades a fixed delay of L frames for the smoother's answer on its
 * window: no jitter from the one-sided anchor of the causal solve, dropped detections filled in from both sides.
 * State per stream s (caller-owned, in/out; the lag L is fixed for the life of the state):
 *   last_qpos[s]            the anchor a: the last committed frame's solution (a fresh stream: the warm start, as
 *                           dexr_sequences_t.last_qpos);
 *   projected[s]            the DexPilot flags after the last committed frame (a fresh stream: all false);
 *   window_len[s]           h in 0..L, the frames held but not yet committed, in time order at slots 0..h-1 of
 *                           window_keypoints / window_fixed_qpos / window_qpos (slot L takes the incoming frame).
 * A tick (num_ticks of them per call, stream s reading keypoints[s,k] at tick k):
 *   1. append the frame at slot h; window_qpos[h] starts at window_qpos[h-1] (h = 0: last_qpos);
 *   2. solve: exactly dexr_smooth_sequences_packed on the h+1 window frames (keypoints = window_keypoints, fixed_qpos =
 *      window_fixed_qpos, qpos_init = qpos_out = window_qpos, last_qpos = the anchor, projected = the committed flags,
 *      w = smooth_weight (< 0: params.norm_delta); params.tol, lambda0 and max_iters per tick);
 *   3. if h + 1 = L + 1: emit slot 0 (qpos_out, robot_qpos_out = its scatter + mimic, status_out = the window solve's status
 *      word of that frame, DEXR_STATUS_MAXITER and DEXR_STATUS_MISSING included), commit it (last_qpos = window_qpos[0],
 *      projected advanced by one step of the hysteresis recurrence with its keypoints: the smoother's own walk) and shift
 *      the window down by one.  Otherwise window_len = h + 1 and the tick emits NaN with status DEXR_STATUS_PENDING.
 * Flush (flush_count_out non-NULL, after the ticks): the held frames are emitted in order as the last tick's joint solve left
 *   them (rows 0..h-1 of flush_*_out, NaN after; flush_count_out[s] = h), the last one becomes the anchor, the flags advance
 *   through them and window_len = 0.  No new solve: (x_1..x_L) of the window's minimiser minimises it with x_0 fixed.  After
 *   a flush a stream fed T frames has emitted exactly T non-pending frames.
 * So L = 0 is the causal problem (each tick minimises L_t(x) + w |x - clip(x_{t-1})|^2), and L >= T - 1 followed by a flush
 *   is the offline smoother on the whole clip from the same anchor.  A dropped detection (a NaN keypoint or fixed joint) is
 *   the smoother's missing frame: interpolated inside the window once later frames arrive, emitted with
 *   DEXR_STATUS_MISSING.  A stream whose state is non-finite emits DEXR_STATUS_NONFINITE (the smoother's rule for a
 *   non-finite start) until the caller resets it.  No low-pass filter (params.lp_alpha is ignored), no carried damping.
 *   A window_len outside 0..L reads as the nearest bound.  Raw landmarks (params.preprocess != 0) are refused.
 *   `workspace`: at least dexr_fixed_lag_workspace_bytes(robot, num_streams, lag) bytes (DEXR_E_INVALID below): the
 *   smoother's workspace for S (L+1) frames followed by S (L+1) int32 status words.  num_ticks == 0 without a flush does
 *   nothing.  Asynchronous on `cuda_stream`, allocates nothing.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
#define DEXR_STATUS_PENDING (1 << 28) /* fixed lag: the tick filled the window and emitted nothing (qpos NaN) */
#define DEXR_FIXED_LAG_MAX 4095       /* the largest lag */
typedef struct dexr_fixed_lag {
  const float* keypoints;      /* [S,K,21,3] new frames, wrist-centred (params.preprocess must be 0)                   */
  const float* fixed_qpos;     /* [S,K,n_fixed] or NULL when n_fixed == 0                                             */
  float* last_qpos;            /* [S,n_var] in/out anchor: the last committed frame / the warm start                  */
  uint8_t* projected;          /* [S,len_proj] in/out flags after the last committed frame, or NULL                   */
  float* window_keypoints;     /* [S,L+1,21,3] in/out                                                                  */
  float* window_fixed_qpos;    /* [S,L+1,n_fixed] in/out or NULL                                                       */
  float* window_qpos;          /* [S,L+1,n_var] in/out                                                                 */
  int32_t* window_len;         /* [S] in/out, 0..L                                                                     */
  float* qpos_out;             /* [S,K,n_var] frame emitted at each tick (NaN while PENDING)                           */
  float* robot_qpos_out;       /* [S,K,dof] or NULL                                                                    */
  int32_t* status_out;         /* [S,K] or NULL                                                                        */
  float* flush_qpos_out;       /* [S,L,n_var] or NULL                                                                  */
  float* flush_robot_qpos_out; /* [S,L,dof] or NULL                                                                    */
  int32_t* flush_count_out;    /* [S] or NULL: non-NULL = flush after the K ticks                                      */
  int32_t lag;
  float smooth_weight;         /* < 0: params.norm_delta                                                               */
  void* workspace;             /* >= dexr_fixed_lag_workspace_bytes(robot, S, lag) bytes                               */
  size_t workspace_bytes;
} dexr_fixed_lag_t;
size_t dexr_fixed_lag_sizeof(void);
size_t dexr_fixed_lag_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag);
int dexr_fixed_lag_step(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                        int64_t num_streams, int64_t num_ticks, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Fixed-lag smoothing with an acceleration penalty: dexr_fixed_lag_step whose window solve is
 * dexr_smooth_sequences_packed_accel (c = acc->accel_weight) and whose state also carries the frame committed before the
 * anchor, so that the triple at the window's start is not lost.  State per stream s, in addition to dexr_fixed_lag_t's:
 *   prev_qpos[s]  p, the frame committed before last_qpos[s], stored raw (unclipped);
 *   has_prev[s]   0 for a fresh stream, 1 once a frame has been committed (any non-zero value reads as 1).
 * A tick's solve is exactly smooth_packed_stream<G, ACC = true> on the h+1 window frames anchored at clip(last_qpos), plus,
 * when has_prev[s] is 1, the triple (clip(p), clip(a), x_0): F gains c |x_0 - 2 clip(a) + clip(p)|^2, which changes only
 * x_0's gradient, its diagonal block (+2c I) and F_0; p and a are constants.  p is clipped at use, as the anchor is: a
 * fresh stream's warm start may lie outside clip_lo / clip_hi, and the offline smoother uses clip(a) as frame -1.
 * On every committed frame (a tick's or a flush's): prev_qpos = last_qpos (the old anchor, raw), has_prev = 1, then
 * last_qpos = the committed frame.  So a flush of h frames leaves prev_qpos at the second-to-last committed frame.
 * Consequences: a fresh stream with L >= T-1 plus a flush is dexr_smooth_sequences_packed_accel on the whole clip from the
 * same anchor, bit for bit (no solve sees a pre-anchor); L = 0 is the causal minimiser of
 * L_t(x) + w |x - clip(a)|^2 + c |x - 2 clip(a) + clip(p)|^2 (a constant-velocity prior; the first frame of a fresh stream
 * has no c term); splitting a run into calls, or batching streams, changes no bit.
 * c is fixed for the life of a state, like the lag; a c = 0 stream uses dexr_fixed_lag_step and has no prev_qpos / has_prev.
 * A non-finite prev_qpos with has_prev = 1 is a non-finite start of the window solve (DEXR_STATUS_NONFINITE, the warm start
 * emitted as given; other streams untouched); a commit moves the pre-anchor on.  Missing frames, DexPilot flags, PENDING, MAXITER, window_len clamping, the raw-landmark refusal and asynchrony
 * are dexr_fixed_lag_step's.  DEXR_E_INVALID for any of dexr_fixed_lag_step's checks, a c that is <= 0 or non-finite,
 * prev_qpos or has_prev NULL while num_streams > 0, or io->workspace_bytes below
 * dexr_fixed_lag_accel_workspace_bytes(robot, num_streams, lag): the accel smoother's workspace for S (L+1) frames followed
 * by S (L+1) int32 status words.  The backward is dexr_fixed_lag_step_accel_tape and dexr_fixed_lag_step_accel_vjp, after
 * dexr_fixed_lag_step_vjp below.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_fixed_lag_accel {
  float accel_weight; /* c: finite, > 0 (c = 0 streams use dexr_fixed_lag_step)                                         */
  float* prev_qpos;   /* [S,n_var] in/out: the frame committed before last_qpos (raw)                                   */
  int32_t* has_prev;  /* [S] in/out: 0 fresh, 1 after the first commit                                                  */
} dexr_fixed_lag_accel_t;
size_t dexr_fixed_lag_accel_sizeof(void);
size_t dexr_fixed_lag_accel_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag);
int dexr_fixed_lag_step_accel(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                              const dexr_fixed_lag_accel_t* acc, int64_t num_streams, int64_t num_ticks, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Recording a fixed-lag call for its backward: dexr_fixed_lag_step_tape is dexr_fixed_lag_step that also stores, for tick k
 * of stream s, the window minimiser X^k the tick's solve left (tape.qpos[s,k,0..m-1], m the window's length; rows m..L are
 * not written) and the committed DexPilot flags that solve started from (tape.projected[s,k], DexPilot only; NULL
 * otherwise).  Outputs and state are bit-identical with and without recording.  The tape holds S K (L+1) n_var floats:
 * 84 MB at S = 256, K = 300, L = 16, n_var = 16.  Checks, workspace and asynchrony as dexr_fixed_lag_step.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_fixed_lag_tape {
  float* qpos;        /* [S,K,L+1,n_var] each tick's window minimiser                                                  */
  uint8_t* projected; /* [S,K,len_proj] the committed flags each tick's solve started from (DexPilot), or NULL          */
} dexr_fixed_lag_tape_t;
size_t dexr_fixed_lag_tape_sizeof(void);
int dexr_fixed_lag_step_tape(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                             const dexr_fixed_lag_tape_t* tape, int64_t num_streams, int64_t num_ticks, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through fixed-lag smoothing: the VJP of one recorded dexr_fixed_lag_step_tape call (K ticks of lag L,
 * optionally followed by a flush) with respect to its new frames and the state it started from, every stream in one launch.
 * Per stream, with h0 = clamp(window_len, 0, L) held frames, the inputs are u_0 .. u_{h0+K-1} (the held frames, then the
 * K new ones); c_k = max(0, h0 + k - L) frames are committed before tick k, which solves the window W_k = u_{c_k} ..
 * u_{h0+k} for its minimiser X^k (tape.qpos[s,k]), anchored at A_k = last_qpos when c_k = 0 and at X^{k-1}[0] (the frame
 * tick k-1 committed) otherwise.  A loss on the emitted rows, the flushed rows and the final state reaches the inputs only
 * through the emitting windows' minimisers and the last tick's; every other solve only picks a basin and is not
 * differentiated (as qpos_init is not in dexr_smooth_sequences_packed_vjp).  The backward walks k = K-1 .. 0 carrying abar,
 * the cotangent of the current anchor:
 *   1. the window cotangent: on an emitting tick slot 0 gets grad_qpos[k] + M^T grad_robot_qpos[k] + abar; the last tick
 *      also takes the flushed rows' and the final state's cotangents (grad_last_qpos_out, the held slots of
 *      grad_window_qpos_out), each at the slot it came from (shifted by one when the last tick emitted).  grad_last_qpos_out
 *      goes to the last flushed frame when the call flushed held frames, else to X^{K-1}[0] when the last tick emitted,
 *      else to last_qpos.  Cotangents on PENDING rows, and on flush rows past flush_count, are ignored;
 *   2. W_k is differentiated exactly as dexr_smooth_sequences_packed_vjp differentiates a clip (same active set, block
 *      Thomas, target pass), at X^k, anchor A_k, the flags of tape.projected[s,k] and w = smooth_weight;
 *   3. each window frame's keypoint and fixed-joint cotangent is added to the frame of the call it came from
 *      (grad_keypoints[s,k'] for a new frame, grad_window_keypoints[s,j] for one held when the call started); the anchor
 *      cotangent 2 w v_0 (where the clip passes) becomes abar, which feeds X^{k-1}[0] when c_k >= 1 and grad_last_qpos
 *      when c_k = 0.
 * Cotangents on the final state's window_keypoints / window_fixed_qpos (held slots only) go straight back to the input
 * frames those slots hold, and start those frames' sums; the window contributions follow in decreasing tick order.  So a
 * call split into chunks chained through the state cotangents gives the same bits as one call.  The incoming window_qpos is
 * a warm start: its cotangent is 0 when K > 0.  With K = 0 a flush's rows ARE the incoming held slots of window_qpos (with
 * the mimic fold; a fixed joint's share goes to grad_window_fixed_qpos), and K = 0 without a flush passes the state's
 * cotangents through.
 *   Per window, as in dexr_smooth_sequences_packed_vjp: a window whose stacked free Hessian is not positive definite
 *     contributes zero and cuts the anchor chain (its emitting tick gets DEXR_STATUS_NOT_PD); a non-finite point, anchor or
 *     cotangent makes everything the window writes NaN (DEXR_STATUS_NONFINITE), which reaches earlier ticks through abar;
 *     a missing frame gets zero cotangents but carries the chain.  One difference: a flushed row's robot_qpos cotangent on
 *     a fixed joint is that joint's direct term, added to the frame's sum before the windows (so that chunks stay
 *     bit-identical), and it is kept where dexr_smooth_sequences_packed_vjp zeroes its direct term: on a NOT_PD window and
 *     on a missing frame.  Without those, L >= K - 1 with a flush gives the smoother VJP's bits on the whole clip.
 *   status_out[s,k]: the emitted frame's window status (0, NOT_PD or NONFINITE, | MISSING) on emitting ticks,
 *     DEXR_STATUS_PENDING on the others.
 * Not differentiated: the DexPilot flags, w, the starting trajectories.  Raw landmarks (params.preprocess != 0) are refused.
 * last_qpos and window_len must be the state before the call; keypoints, fixed_qpos and the tape the call's own;
 * `projected` and `window_qpos` are not read (the flags come from the tape, the warm start gets no derivative).
 * Every output is written in full (zeros where nothing reaches): grad_keypoints / grad_fixed_qpos [S,K,...], the
 * grad_window_* [S,L+1,...], grad_last_qpos [S,n_var].  Every cotangent input and every output but grad_keypoints (when
 * K > 0) may be NULL.  `workspace`: at least dexr_fixed_lag_vjp_workspace_bytes(robot, num_streams, lag) bytes
 * (DEXR_E_INVALID below): one rebuilt window per stream.  Asynchronous on `cuda_stream`, allocates nothing, does nothing for
 * num_streams == 0.  All pointers are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_fixed_lag_vjp {
  /* the forward's inputs and the state before the call */
  const float* keypoints;             /* [S,K,21,3] as given to the forward                                           */
  const float* fixed_qpos;            /* [S,K,n_fixed] or NULL when n_fixed == 0                                      */
  const float* last_qpos;             /* [S,n_var] the anchor before the call                                         */
  const uint8_t* projected;           /* [S,len_proj] the flags before the call (not read: the tape holds each tick's) */
  const float* window_keypoints;      /* [S,L+1,21,3] before the call                                                 */
  const float* window_fixed_qpos;     /* [S,L+1,n_fixed] before the call, or NULL                                     */
  const float* window_qpos;           /* [S,L+1,n_var] before the call (not read: a warm start)                       */
  const int32_t* window_len;          /* [S] before the call                                                          */
  dexr_fixed_lag_tape_t tape;         /* the call's recording                                                         */
  /* cotangents (NULL = 0) */
  const float* grad_qpos;             /* [S,K,n_var] of qpos_out                                                      */
  const float* grad_robot_qpos;       /* [S,K,dof] of robot_qpos_out                                                  */
  const float* grad_flush_qpos;       /* [S,L,n_var] of flush_qpos_out                                                */
  const float* grad_flush_robot_qpos; /* [S,L,dof] of flush_robot_qpos_out                                            */
  const float* grad_last_qpos_out;    /* [S,n_var] of the final last_qpos                                             */
  const float* grad_window_qpos_out;  /* [S,L+1,n_var] of the final window_qpos (held slots read)                     */
  const float* grad_window_keypoints_out;  /* [S,L+1,21,3] of the final window_keypoints (held slots read)            */
  const float* grad_window_fixed_qpos_out; /* [S,L+1,n_fixed] of the final window_fixed_qpos (held slots read)        */
  /* outputs (NULL: not written; grad_keypoints is required when K > 0) */
  float* grad_keypoints;              /* [S,K,21,3]                                                                   */
  float* grad_fixed_qpos;             /* [S,K,n_fixed]                                                                */
  float* grad_last_qpos;              /* [S,n_var] of the incoming anchor                                             */
  float* grad_window_keypoints;       /* [S,L+1,21,3] of the incoming held frames                                     */
  float* grad_window_fixed_qpos;      /* [S,L+1,n_fixed]                                                              */
  float* grad_window_qpos;            /* [S,L+1,n_var] (0 when K > 0)                                                 */
  int32_t* status_out;                /* [S,K]                                                                        */
  int32_t lag;
  int32_t flushed;                    /* non-zero: the forward flushed after its ticks (flush_count_out non-NULL)     */
  float smooth_weight;                /* as given to the forward; < 0: params.norm_delta                              */
  void* workspace;                    /* >= dexr_fixed_lag_vjp_workspace_bytes(robot, S, lag) bytes                   */
  size_t workspace_bytes;
} dexr_fixed_lag_vjp_t;
size_t dexr_fixed_lag_vjp_sizeof(void);
size_t dexr_fixed_lag_vjp_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag);
int dexr_fixed_lag_step_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_vjp_t* io,
                            int64_t num_streams, int64_t num_ticks, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Backpropagation through fixed-lag smoothing with an acceleration penalty.
 * dexr_fixed_lag_step_accel_tape is dexr_fixed_lag_step_accel that also records into `tape` as dexr_fixed_lag_step_tape
 * does (same layout); its outputs and state, prev_qpos and has_prev included, are bit-identical to dexr_fixed_lag_step_accel's.
 * Checks as dexr_fixed_lag_step_accel's plus dexr_fixed_lag_step_tape's tape check.
 * dexr_fixed_lag_step_accel_vjp is dexr_fixed_lag_step_vjp for such a recorded call, `io` as there (io->smooth_weight w)
 * and `acc` the acceleration weight c, the pre-anchor state before the call and the pre-anchor's cotangents.  With
 * a_in = last_qpos, p_in = prev_qpos and hp_in = has_prev before the call, tick k's window has the anchor A_k, the
 * pre-anchor P_k and the flag H_k:
 *   c_k = 0: A_k = a_in, P_k = p_in, H_k = hp_in;   c_k = 1: X^{k-1}[0], a_in, 1;   c_k >= 2: X^{k-1}[0], X^{k-2}[0], 1.
 * Window k is differentiated as dexr_smooth_sequences_packed_accel_vjp differentiates a clip anchored at clip(A_k), plus,
 * when H_k = 1, the triple c |x_0 - 2 clip(A_k) + clip(P_k)|^2: 2c I more on block 0 of the Hessian, the anchor's cotangent
 * (2w v_0) + (4c v_0 - 2c v_1 when the window has a second frame) + (4c v_0 when H_k = 1), summed in that order and all of
 * it only where the clip passes A_k, and the pre-anchor's cotangent -2c v_0 where the clip passes P_k (0 when H_k = 0).
 * The reverse walk carries two rows per stream: C1, the cotangent of X^k[0], and C2, that of X^{k-1}[0].  At the start C1
 * is grad_last_qpos_out where the final last_qpos is X^{K-1}[0], and C2 is grad_prev_qpos_out where the final prev_qpos is
 * X^{K-2}[0].  Slot 0 of an emitting window k gets its emitted row's cotangent + C1 (on the last tick, grad_last_qpos_out
 * or grad_prev_qpos_out, whichever lands there).  After window k's VJP, with ga its anchor cotangent and gp its pre-anchor's:
 *   c_k >= 2: C1 = C2 + ga, C2 = gp;   c_k = 1: C1 = C2 + ga, grad_last_qpos += gp;
 *   c_k = 0:  grad_last_qpos += ga, grad_prev_qpos += gp.
 * The final prev_qpos is the second-to-last committed frame, the incoming p_in and a_in counting as the two commits before
 * the call; grad_prev_qpos_out goes to it: a flushed slot (summed after grad_last_qpos_out's place in the slot's order),
 * X^{K-1}[0] (a flush of one frame), X^{K-2}[0] (C2), grad_last_qpos (written with it) or grad_prev_qpos (written with it).
 * So the cotangent of a committed frame X^j[0] is its emitted row's + ((the pre-anchor cotangent of window j + 2) + (the
 * anchor cotangent of window j + 1)), in that order, and a call split into chunks chained through grad_last_qpos /
 * grad_prev_qpos gives the bits of one call.
 * A NOT_PD window contributes zero and drops the slot cotangents that land on it, but no longer cuts the chain completely:
 * the pre-anchor cotangent of the window after it (in C2) skips over it to X^{k-1}[0] -- correctly, as P_{k+1} does not
 * pass through window k.  A non-finite point, anchor, pre-anchor (a non-finite prev_qpos with has_prev = 1 included) or
 * cotangent makes the window's outputs NaN, which reaches earlier ticks through C1 and C2; other streams are untouched.
 * Missing frames carry the chain; a flushed row's fixed-joint share starts its frame's sum.  Not differentiated: the
 * DexPilot flags, w, c, has_prev and the warm start.  Everything else -- the outputs (grad_prev_qpos [S,n_var] too, written
 * in full when non-NULL), status, layout, asynchrony -- is dexr_fixed_lag_step_vjp's.  DEXR_E_INVALID for any of
 * dexr_fixed_lag_step_vjp's checks, a c that is <= 0 or non-finite, prev_qpos or has_prev NULL while num_streams > 0, or
 * io->workspace_bytes below dexr_fixed_lag_accel_vjp_workspace_bytes(robot, num_streams, lag).
 * ------------------------------------------------------------------------------------------- */
typedef struct dexr_fixed_lag_accel_vjp {
  float accel_weight;              /* c as given to the forward: finite, > 0                                             */
  const float* prev_qpos;          /* [S,n_var] the pre-anchor before the call (raw)                                     */
  const int32_t* has_prev;         /* [S] before the call                                                                */
  const float* grad_prev_qpos_out; /* [S,n_var] cotangent of the final prev_qpos, or NULL (= 0)                          */
  float* grad_prev_qpos;           /* [S,n_var] output: cotangent of the incoming prev_qpos, or NULL                     */
} dexr_fixed_lag_accel_vjp_t;
size_t dexr_fixed_lag_accel_vjp_sizeof(void);
size_t dexr_fixed_lag_accel_vjp_workspace_bytes(const dexr_robot_t* robot, int64_t num_streams, int32_t lag);
int dexr_fixed_lag_step_accel_tape(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_t* io,
                                   const dexr_fixed_lag_accel_t* acc, const dexr_fixed_lag_tape_t* tape, int64_t num_streams,
                                   int64_t num_ticks, void* cuda_stream);
int dexr_fixed_lag_step_accel_vjp(const dexr_robot_t* robot, const dexr_params_t* params, const dexr_fixed_lag_vjp_t* io,
                                  const dexr_fixed_lag_accel_vjp_t* acc, int64_t num_streams, int64_t num_ticks,
                                  void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* DEXR_H_ */
