"""ctypes binding of libdexr.so (the C ABI declared in include/dexr.h).

The library is built in-tree by `__graft_entry__.build()` / `python -m dex_retargeting_b200.build`
(nvcc, sm_90a).  There is NO fallback: if the shared object is missing or a call fails, this module
raises -- the product path never silently runs on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

MAX_LANES, MAX_LINKS, MAX_RES, MAX_GROUP, NUM_KEYPOINTS = 32, 16, 16, 4, 21
MAX_LINKS_PER_LANE = 4
LOSS_POSITION, LOSS_VECTOR, LOSS_DEXPILOT = 0, 1, 2
TABLE_MAGIC = 0x31525844

STATUS_MAXITER = 1 << 24
STATUS_NONFINITE = 1 << 25
STATUS_NOT_PD = 1 << 26
STATUS_MISSING = 1 << 27
STATUS_PENDING = 1 << 28
FIXED_LAG_MAX = 4095

_f, _i, _u = C.c_float, C.c_int32, C.c_uint32


class DexrTable(C.Structure):
    """Mirror of `dexr_table_t` (include/dexr.h) -- keep field order identical."""

    _fields_ = [
        ("magic", _u), ("nbytes", _u), ("dof", _i), ("n_var", _i), ("n_fixed", _i), ("n_links", _i),
        ("n_res", _i), ("loss", _i), ("n_rounds", _i), ("has_mimic", _i), ("num_fingers", _i),
        ("len_proj", _i), ("len_s1", _i), ("block_width", _i), ("arrow", _i), ("reserved", _i),
        ("R0", (_f * 9) * MAX_LANES), ("RA", (_f * 9) * MAX_LANES), ("RB", (_f * 9) * MAX_LANES),
        ("p0", (_f * 3) * MAX_LANES), ("d0", (_f * 3) * MAX_LANES), ("axis", (_f * 3) * MAX_LANES),
        ("jtype", _i * MAX_LANES), ("var_index", _i * MAX_LANES), ("fixed_index", _i * MAX_LANES),
        ("mimic_src", _i * MAX_LANES), ("mimic_mult", _f * MAX_LANES), ("mimic_off", _f * MAX_LANES),
        ("lower", _f * MAX_LANES), ("upper", _f * MAX_LANES), ("clip_lo", _f * MAX_LANES), ("clip_hi", _f * MAX_LANES),
        ("jump", _u * MAX_LANES), ("anc_mask", _u * MAX_LANES), ("desc_mask", _u * MAX_LANES),
        ("group_count", _i * MAX_LANES), ("group_lane", (_i * MAX_GROUP) * MAX_LANES),
        ("group_mult", (_f * MAX_GROUP) * MAX_LANES),
        ("link_parent", _i * MAX_LINKS), ("link_off", (_f * 3) * MAX_LINKS), ("link_anc_mask", _u * MAX_LINKS),
        ("res_task", _i * MAX_RES), ("res_origin", _i * MAX_RES), ("res_human_task", _i * MAX_RES),
        ("res_human_origin", _i * MAX_RES), ("s2_origin", _i * MAX_RES), ("s2_task", _i * MAX_RES),
    ]


class DexrParams(C.Structure):
    _fields_ = [
        ("huber_delta", _f), ("norm_delta", _f), ("scaling", _f), ("project_dist", _f), ("escape_dist", _f),
        ("eta1", _f), ("eta2", _f), ("lp_alpha", _f), ("tol", _f), ("lambda0", _f),
        ("max_iters", _i), ("clip_init", _i), ("preprocess", _i),
    ]


class DexrFrames(C.Structure):
    _fields_ = [
        ("keypoints", C.c_void_p), ("ref_value", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p),
        ("projected", C.c_void_p), ("qpos_out", C.c_void_p), ("robot_qpos_out", C.c_void_p),
        ("status_out", C.c_void_p), ("cost_out", C.c_void_p), ("damping_io", C.c_void_p),
    ]


class DexrSequences(C.Structure):
    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("filter_state", C.c_void_p),
        ("filter_init", C.c_void_p), ("projected", C.c_void_p), ("robot_qpos_out", C.c_void_p), ("status_out", C.c_void_p),
        ("damping_state", C.c_void_p),
    ]


class DexrEval(C.Structure):
    """Mirror of `dexr_eval_t`: buffers of one objective evaluation (`dexr_eval_objective`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("ref_value", C.c_void_p), ("fixed_qpos", C.c_void_p), ("qpos", C.c_void_p),
        ("last_qpos", C.c_void_p), ("projected", C.c_void_p), ("loss_out", C.c_void_p), ("cost_out", C.c_void_p),
        ("grad_out", C.c_void_p),
    ]


class DexrVjp(C.Structure):
    """Mirror of `dexr_vjp_t`: buffers of one backpropagation through the solve (`dexr_solve_vjp`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("ref_value", C.c_void_p), ("fixed_qpos", C.c_void_p), ("qpos", C.c_void_p),
        ("last_qpos", C.c_void_p), ("projected", C.c_void_p), ("grad_qpos", C.c_void_p), ("grad_keypoints", C.c_void_p),
        ("grad_ref_value", C.c_void_p), ("grad_fixed_qpos", C.c_void_p), ("grad_last_qpos", C.c_void_p),
        ("status_out", C.c_void_p),
    ]


class DexrSequencesTape(C.Structure):
    """Mirror of `dexr_sequences_tape_t`: what `dexr_solve_sequences_tape` records for the backward."""

    _fields_ = [("qpos", C.c_void_p), ("projected", C.c_void_p)]


class DexrSequencesVjp(C.Structure):
    """Mirror of `dexr_sequences_vjp_t`: buffers of one backpropagation through the sequence solve."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("filter_init", C.c_void_p),
        ("qpos", C.c_void_p), ("projected", C.c_void_p), ("grad_robot_qpos", C.c_void_p),
        ("grad_last_qpos_out", C.c_void_p), ("grad_filter_state_out", C.c_void_p), ("grad_keypoints", C.c_void_p),
        ("grad_fixed_qpos", C.c_void_p), ("grad_last_qpos", C.c_void_p), ("grad_filter_state", C.c_void_p),
        ("status_out", C.c_void_p),
    ]


class DexrJacobian(C.Structure):
    """Mirror of `dexr_jacobian_t`: buffers of one per-frame Jacobian launch (`dexr_solve_jacobian`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("ref_value", C.c_void_p), ("fixed_qpos", C.c_void_p), ("qpos", C.c_void_p),
        ("last_qpos", C.c_void_p), ("projected", C.c_void_p), ("jac_keypoints", C.c_void_p), ("jac_ref_value", C.c_void_p),
        ("jac_fixed_qpos", C.c_void_p), ("jac_last_qpos", C.c_void_p), ("status_out", C.c_void_p),
    ]


class DexrSmooth(C.Structure):
    """Mirror of `dexr_smooth_t`: buffers of one offline smoothing launch (`dexr_smooth_sequences_packed`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("projected", C.c_void_p),
        ("qpos_init", C.c_void_p), ("qpos_out", C.c_void_p), ("robot_qpos_out", C.c_void_p), ("status_out", C.c_void_p),
        ("cost_out", C.c_void_p), ("smooth_weight", _f), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class DexrSmoothVjp(C.Structure):
    """Mirror of `dexr_smooth_vjp_t`: buffers of one backpropagation through the smoother
    (`dexr_smooth_sequences_packed_vjp`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("projected", C.c_void_p),
        ("qpos", C.c_void_p), ("grad_qpos", C.c_void_p), ("grad_robot_qpos", C.c_void_p), ("smooth_weight", _f),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("grad_keypoints", C.c_void_p),
        ("grad_fixed_qpos", C.c_void_p), ("grad_last_qpos", C.c_void_p), ("status_out", C.c_void_p),
    ]


class DexrFixedLag(C.Structure):
    """Mirror of `dexr_fixed_lag_t`: inputs, caller-owned state and outputs of one fixed-lag smoothing call
    (`dexr_fixed_lag_step`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("projected", C.c_void_p),
        ("window_keypoints", C.c_void_p), ("window_fixed_qpos", C.c_void_p), ("window_qpos", C.c_void_p),
        ("window_len", C.c_void_p), ("qpos_out", C.c_void_p), ("robot_qpos_out", C.c_void_p), ("status_out", C.c_void_p),
        ("flush_qpos_out", C.c_void_p), ("flush_robot_qpos_out", C.c_void_p), ("flush_count_out", C.c_void_p),
        ("lag", _i), ("smooth_weight", _f), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class DexrFixedLagAccel(C.Structure):
    """Mirror of `dexr_fixed_lag_accel_t`: the acceleration weight and the pre-anchor state of accelerated fixed-lag
    streams (`dexr_fixed_lag_step_accel`)."""

    _fields_ = [("accel_weight", _f), ("prev_qpos", C.c_void_p), ("has_prev", C.c_void_p)]


class DexrFixedLagTape(C.Structure):
    """Mirror of `dexr_fixed_lag_tape_t`: what `dexr_fixed_lag_step_tape` records for the backward."""

    _fields_ = [("qpos", C.c_void_p), ("projected", C.c_void_p)]


class DexrFixedLagVjp(C.Structure):
    """Mirror of `dexr_fixed_lag_vjp_t`: buffers of one backpropagation through a fixed-lag call
    (`dexr_fixed_lag_step_vjp`)."""

    _fields_ = [
        ("keypoints", C.c_void_p), ("fixed_qpos", C.c_void_p), ("last_qpos", C.c_void_p), ("projected", C.c_void_p),
        ("window_keypoints", C.c_void_p), ("window_fixed_qpos", C.c_void_p), ("window_qpos", C.c_void_p),
        ("window_len", C.c_void_p), ("tape", DexrFixedLagTape), ("grad_qpos", C.c_void_p),
        ("grad_robot_qpos", C.c_void_p), ("grad_flush_qpos", C.c_void_p), ("grad_flush_robot_qpos", C.c_void_p),
        ("grad_last_qpos_out", C.c_void_p), ("grad_window_qpos_out", C.c_void_p),
        ("grad_window_keypoints_out", C.c_void_p), ("grad_window_fixed_qpos_out", C.c_void_p),
        ("grad_keypoints", C.c_void_p), ("grad_fixed_qpos", C.c_void_p), ("grad_last_qpos", C.c_void_p),
        ("grad_window_keypoints", C.c_void_p), ("grad_window_fixed_qpos", C.c_void_p), ("grad_window_qpos", C.c_void_p),
        ("status_out", C.c_void_p), ("lag", _i), ("flushed", _i), ("smooth_weight", _f), ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_size_t),
    ]


class DexrFixedLagAccelVjp(C.Structure):
    """Mirror of `dexr_fixed_lag_accel_vjp_t`: the acceleration weight, the pre-anchor state before the call and the
    pre-anchor's cotangents of `dexr_fixed_lag_step_accel_vjp`."""

    _fields_ = [("accel_weight", _f), ("prev_qpos", C.c_void_p), ("has_prev", C.c_void_p), ("grad_prev_qpos_out", C.c_void_p),
                ("grad_prev_qpos", C.c_void_p)]


class DexrGroup(C.Structure):
    """Mirror of `dexr_group_t`: one (robot, batch) group of a mixed-robot launch."""

    _fields_ = [("robot", C.c_void_p), ("params", C.POINTER(DexrParams)), ("io", DexrFrames), ("num_frames", C.c_int64)]


MAX_GROUPS = 16


class DexrLaunchInfo(C.Structure):
    _fields_ = [("grid", _i), ("block", _i), ("smem_bytes", _i), ("frames_per_tile", _i), ("lanes_per_frame", _i),
                ("consumer_warps", _i), ("kernels_launched", _i)]


EXPORTS = [
    "dexr_version", "dexr_build_id", "dexr_last_error", "dexr_table_sizeof", "dexr_params_sizeof", "dexr_frames_sizeof",
    "dexr_sequences_sizeof", "dexr_default_params",
    "dexr_robot_create", "dexr_robot_create_from_device", "dexr_robot_device_table", "dexr_robot_destroy",
    "dexr_solve_frames", "dexr_solve_frames_multi", "dexr_solve_sequences", "dexr_solve_frames_host", "dexr_get_launch_info",
    "dexr_preprocess_keypoints", "dexr_eval_sizeof", "dexr_eval_objective", "dexr_vjp_sizeof", "dexr_solve_vjp",
    "dexr_sequences_tape_sizeof", "dexr_solve_sequences_tape", "dexr_sequences_vjp_sizeof", "dexr_solve_sequences_vjp",
    "dexr_jacobian_sizeof", "dexr_solve_jacobian", "dexr_solve_sequences_packed", "dexr_solve_sequences_packed_vjp",
    "dexr_smooth_sizeof", "dexr_smooth_workspace_bytes", "dexr_smooth_sequences_packed", "dexr_smooth_vjp_sizeof",
    "dexr_smooth_sequences_packed_vjp", "dexr_fixed_lag_sizeof", "dexr_fixed_lag_workspace_bytes", "dexr_fixed_lag_step",
    "dexr_fixed_lag_tape_sizeof", "dexr_fixed_lag_step_tape", "dexr_fixed_lag_vjp_sizeof",
    "dexr_fixed_lag_vjp_workspace_bytes", "dexr_fixed_lag_step_vjp", "dexr_smooth_accel_workspace_bytes",
    "dexr_smooth_sequences_packed_accel", "dexr_smooth_sequences_packed_accel_vjp", "dexr_fixed_lag_accel_sizeof",
    "dexr_fixed_lag_accel_workspace_bytes", "dexr_fixed_lag_step_accel", "dexr_fixed_lag_accel_vjp_sizeof",
    "dexr_fixed_lag_accel_vjp_workspace_bytes", "dexr_fixed_lag_step_accel_tape", "dexr_fixed_lag_step_accel_vjp",
]

_LIB = None


def library_path() -> Path:
    env = os.environ.get("DEXR_LIBRARY")
    return Path(env) if env else Path(__file__).resolve().parent / "libdexr.so"


class DexrError(RuntimeError):
    pass


def load():
    """Load libdexr.so once; raise if it is missing or its struct layouts disagree with this file."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not path.exists():
        raise DexrError(
            f"{path} not found: build the CUDA library first (python -c 'import __graft_entry__ as g; g.build()' "
            f"or python -m dex_retargeting_b200.build).  There is no CPU fallback."
        )
    lib = C.CDLL(str(path))
    lib.dexr_version.restype = C.c_int
    lib.dexr_last_error.restype = C.c_char_p
    lib.dexr_build_id.restype = C.c_char_p
    lib.dexr_table_sizeof.restype = C.c_size_t
    lib.dexr_params_sizeof.restype = C.c_size_t
    lib.dexr_default_params.argtypes = [C.POINTER(DexrParams)]
    lib.dexr_default_params.restype = None
    lib.dexr_robot_create.argtypes = [C.POINTER(DexrTable), C.c_int, C.POINTER(C.c_void_p)]
    lib.dexr_robot_create_from_device.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]
    lib.dexr_robot_device_table.argtypes = [C.c_void_p]
    lib.dexr_robot_device_table.restype = C.c_void_p
    lib.dexr_robot_destroy.argtypes = [C.c_void_p]
    lib.dexr_robot_destroy.restype = None
    lib.dexr_solve_frames.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFrames), C.c_int64, C.c_void_p]
    lib.dexr_solve_frames_multi.argtypes = [C.POINTER(DexrGroup), C.c_int32, C.c_void_p]
    lib.dexr_solve_sequences.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSequences), C.c_int64,
                                         C.c_int64, C.c_void_p]
    lib.dexr_solve_frames_host.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFrames), C.c_int64]
    lib.dexr_get_launch_info.argtypes = [C.c_void_p, C.POINTER(DexrLaunchInfo)]
    lib.dexr_preprocess_keypoints.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p]
    if lib.dexr_table_sizeof() != C.sizeof(DexrTable):
        raise DexrError(f"dexr_table_t layout mismatch: library {lib.dexr_table_sizeof()} vs binding {C.sizeof(DexrTable)}")
    if lib.dexr_params_sizeof() != C.sizeof(DexrParams):
        raise DexrError("dexr_params_t layout mismatch between library and binding")
    if hasattr(lib, "dexr_frames_sizeof"):
        lib.dexr_frames_sizeof.restype = C.c_size_t
        lib.dexr_sequences_sizeof.restype = C.c_size_t
        if lib.dexr_frames_sizeof() != C.sizeof(DexrFrames) or lib.dexr_sequences_sizeof() != C.sizeof(DexrSequences):
            raise DexrError("dexr_frames_t / dexr_sequences_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_frames_sizeof: rebuild it (python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_eval_sizeof"):
        lib.dexr_eval_sizeof.restype = C.c_size_t
        if lib.dexr_eval_sizeof() != C.sizeof(DexrEval):
            raise DexrError("dexr_eval_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_eval_objective.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrEval), C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_eval_sizeof: rebuild it (python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_vjp_sizeof"):
        lib.dexr_vjp_sizeof.restype = C.c_size_t
        if lib.dexr_vjp_sizeof() != C.sizeof(DexrVjp):
            raise DexrError("dexr_vjp_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_solve_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrVjp), C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_vjp_sizeof: rebuild it (python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_sequences_vjp_sizeof"):
        lib.dexr_sequences_tape_sizeof.restype = C.c_size_t
        lib.dexr_sequences_vjp_sizeof.restype = C.c_size_t
        if (lib.dexr_sequences_tape_sizeof() != C.sizeof(DexrSequencesTape)
                or lib.dexr_sequences_vjp_sizeof() != C.sizeof(DexrSequencesVjp)):
            raise DexrError("dexr_sequences_tape_t / dexr_sequences_vjp_t layout mismatch between library and binding "
                            "(stale DEXR_LIBRARY?)")
        lib.dexr_solve_sequences_tape.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSequences),
                                                  C.POINTER(DexrSequencesTape), C.c_int64, C.c_int64, C.c_void_p]
        lib.dexr_solve_sequences_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSequencesVjp), C.c_int64,
                                                 C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_sequences_vjp_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_jacobian_sizeof"):
        lib.dexr_jacobian_sizeof.restype = C.c_size_t
        if lib.dexr_jacobian_sizeof() != C.sizeof(DexrJacobian):
            raise DexrError("dexr_jacobian_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_solve_jacobian.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrJacobian), C.c_int64,
                                            C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_jacobian_sizeof: rebuild it (python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_solve_sequences_packed"):
        lib.dexr_solve_sequences_packed.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSequences),
                                                    C.POINTER(DexrSequencesTape), C.c_void_p, C.c_int64, C.c_int64,
                                                    C.c_void_p]
        lib.dexr_solve_sequences_packed_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSequencesVjp),
                                                        C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_solve_sequences_packed: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_smooth_sizeof"):
        lib.dexr_smooth_sizeof.restype = C.c_size_t
        if lib.dexr_smooth_sizeof() != C.sizeof(DexrSmooth):
            raise DexrError("dexr_smooth_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_smooth_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
        lib.dexr_smooth_workspace_bytes.restype = C.c_size_t
        lib.dexr_smooth_sequences_packed.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSmooth), C.c_void_p,
                                                     C.c_int64, C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_smooth_sizeof: rebuild it (python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_smooth_vjp_sizeof"):
        lib.dexr_smooth_vjp_sizeof.restype = C.c_size_t
        if lib.dexr_smooth_vjp_sizeof() != C.sizeof(DexrSmoothVjp):
            raise DexrError("dexr_smooth_vjp_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_smooth_sequences_packed_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSmoothVjp),
                                                         C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    if hasattr(lib, "dexr_smooth_sequences_packed_accel"):
        lib.dexr_smooth_accel_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
        lib.dexr_smooth_accel_workspace_bytes.restype = C.c_size_t
        lib.dexr_smooth_sequences_packed_accel.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrSmooth), _f,
                                                           C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
        lib.dexr_smooth_sequences_packed_accel_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams),
                                                               C.POINTER(DexrSmoothVjp), _f, C.c_void_p, C.c_int64,
                                                               C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_smooth_sequences_packed_accel: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_smooth_vjp_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_fixed_lag_sizeof"):
        lib.dexr_fixed_lag_sizeof.restype = C.c_size_t
        if lib.dexr_fixed_lag_sizeof() != C.sizeof(DexrFixedLag):
            raise DexrError("dexr_fixed_lag_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_fixed_lag_workspace_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        lib.dexr_fixed_lag_workspace_bytes.restype = C.c_size_t
        lib.dexr_fixed_lag_step.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLag), C.c_int64,
                                            C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_fixed_lag_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_fixed_lag_vjp_sizeof"):
        lib.dexr_fixed_lag_tape_sizeof.restype = C.c_size_t
        lib.dexr_fixed_lag_vjp_sizeof.restype = C.c_size_t
        if (lib.dexr_fixed_lag_tape_sizeof() != C.sizeof(DexrFixedLagTape)
                or lib.dexr_fixed_lag_vjp_sizeof() != C.sizeof(DexrFixedLagVjp)):
            raise DexrError("dexr_fixed_lag_tape_t / dexr_fixed_lag_vjp_t layout mismatch between library and binding "
                            "(stale DEXR_LIBRARY?)")
        lib.dexr_fixed_lag_step_tape.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLag),
                                                 C.POINTER(DexrFixedLagTape), C.c_int64, C.c_int64, C.c_void_p]
        lib.dexr_fixed_lag_vjp_workspace_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        lib.dexr_fixed_lag_vjp_workspace_bytes.restype = C.c_size_t
        lib.dexr_fixed_lag_step_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLagVjp), C.c_int64,
                                                C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_fixed_lag_vjp_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_fixed_lag_accel_sizeof"):
        lib.dexr_fixed_lag_accel_sizeof.restype = C.c_size_t
        if lib.dexr_fixed_lag_accel_sizeof() != C.sizeof(DexrFixedLagAccel):
            raise DexrError("dexr_fixed_lag_accel_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_fixed_lag_accel_workspace_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        lib.dexr_fixed_lag_accel_workspace_bytes.restype = C.c_size_t
        lib.dexr_fixed_lag_step_accel.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLag),
                                                  C.POINTER(DexrFixedLagAccel), C.c_int64, C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_fixed_lag_accel_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    if hasattr(lib, "dexr_fixed_lag_accel_vjp_sizeof"):
        lib.dexr_fixed_lag_accel_vjp_sizeof.restype = C.c_size_t
        if lib.dexr_fixed_lag_accel_vjp_sizeof() != C.sizeof(DexrFixedLagAccelVjp):
            raise DexrError("dexr_fixed_lag_accel_vjp_t layout mismatch between library and binding (stale DEXR_LIBRARY?)")
        lib.dexr_fixed_lag_accel_vjp_workspace_bytes.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        lib.dexr_fixed_lag_accel_vjp_workspace_bytes.restype = C.c_size_t
        lib.dexr_fixed_lag_step_accel_tape.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLag),
                                                       C.POINTER(DexrFixedLagAccel), C.POINTER(DexrFixedLagTape), C.c_int64,
                                                       C.c_int64, C.c_void_p]
        lib.dexr_fixed_lag_step_accel_vjp.argtypes = [C.c_void_p, C.POINTER(DexrParams), C.POINTER(DexrFixedLagVjp),
                                                      C.POINTER(DexrFixedLagAccelVjp), C.c_int64, C.c_int64, C.c_void_p]
    elif not os.environ.get("DEXR_LIBRARY"):
        raise DexrError(f"{path} does not export dexr_fixed_lag_accel_vjp_sizeof: rebuild it "
                        "(python -m dex_retargeting_b200.build --force)")
    # (an older A/B library named by DEXR_LIBRARY reads a prefix of the buffer structs -- fields are only ever appended -- so
    # the single-robot entry points still work with it; dexr_solve_frames_multi, whose groups embed the struct, does not)
    _LIB = lib
    return lib


def build_id() -> str:
    """The loaded library's source stamp (`dexr_build_id`)."""
    return load().dexr_build_id().decode()


def check(code: int, what: str):
    if code != 0:
        msg = load().dexr_last_error().decode("utf-8", "replace")
        raise DexrError(f"{what} failed ({code}): {msg}")


def default_params() -> DexrParams:
    p = DexrParams()
    load().dexr_default_params(C.byref(p))
    return p
