"""Sequence wrapper: temporal state around the optimizer.

Drop-in for `dex_retargeting.seq_retarget.SeqRetargeting` (reference:
src/dex_retargeting/seq_retarget.py:12-161): `retarget()` clips the previous solution to the joint
limits, solves, keeps the UNFILTERED solution as the next warm start, scatters it into the full
pinocchio-ordered qpos, applies mimic joints and the low-pass filter, returns float64 (robot.dof,).

New, batched: `retarget_sequences()` runs S independent streams x T frames with exactly that recurrence
inside ONE kernel launch (`dexr_solve_sequences`): a group of lanes owns a stream and walks its frames,
`last_qpos`, the DexPilot hysteresis flags and the filter state never leave the SM between frames.
With a `SequenceTape` the same launch also records every frame's unfiltered solution (and DexPilot flags), and
`retarget_sequences_vjp()` backpropagates through all T frames of every stream in one launch
(`dexr_solve_sequences_vjp`; `objective.differentiable_retarget_sequences` wraps both for autograd).
`retarget_packed_sequences()` / `retarget_packed_sequences_vjp()` do the same for streams of different lengths laid end to
end (`PackedStreams`, the cu_seqlens layout): recorded clips of any length in one launch, no padding.
`smooth_packed_sequences()` solves every frame of each packed clip jointly (`dexr_smooth_sequences_packed`): the offline
trajectory, with no lag and with dropped frames filled in.  `retarget_fixed_lag()` brings it to live streams
(`dexr_fixed_lag_step`, `FixedLagState`): each new frame re-solves the last L+1 frames jointly and emits the frame L ticks
back; a state made with `accel_weight` also penalises acceleration there (`dexr_fixed_lag_step_accel`), and
`retarget_fixed_lag_accel_vjp` backpropagates through it.
"""
from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _native as N
from .constants import OPERATOR2MANO, HandType
from .optimizer import Optimizer
from .optimizer_utils import LPFilter
from .urdf import DUMMY_JOINT_NAMES


@dataclass
class StreamState:
    """Device-resident state of S streams (torch tensors); resumable / checkpointable."""

    last_qpos: "torch.Tensor"     # [S, opt_dof] float32, unfiltered previous solution
    filter_state: "torch.Tensor"  # [S, dof] float32
    filter_init: "torch.Tensor"   # [S] uint8
    projected: Optional["torch.Tensor"]  # [S, len_proj] uint8 (DexPilot) or None
    damping: Optional["torch.Tensor"] = None  # [S] float32: the solver's carried damping (dexr_sequences_t.damping_state)

    _FIELDS = ("last_qpos", "filter_state", "filter_init", "projected", "damping")

    def state_dict(self) -> dict:
        """Host copies of every tensor (None stays None): what a checkpoint of S running streams has to hold.  A run resumed
        from it continues bit-identically (the state is complete: tests/test_gpu_parity.py splits a call in two)."""
        return {k: (None if getattr(self, k) is None else getattr(self, k).detach().cpu().clone()) for k in self._FIELDS}

    @classmethod
    def from_state_dict(cls, state: dict, device=None) -> "StreamState":
        """Inverse of `state_dict` (tensors moved to `device`); a checkpoint written before `damping` existed resumes with the
        solver's default damping."""
        import torch

        missing = [k for k in cls._FIELDS[:3] if state.get(k) is None]
        if missing:
            raise ValueError(f"stream state checkpoint lacks {missing}")
        S = int(state["last_qpos"].shape[0])
        for k in cls._FIELDS[1:]:
            t = state.get(k)
            if t is not None and int(t.shape[0]) != S:
                raise ValueError(f"stream state checkpoint: {k} holds {int(t.shape[0])} streams, last_qpos {S}")

        def put(t):
            return None if t is None else torch.as_tensor(t).to(device if device is not None else t.device).contiguous()

        st = cls(**{k: put(state.get(k)) for k in cls._FIELDS})
        if st.damping is None:
            st.damping = torch.zeros((S,), dtype=torch.float32, device=st.last_qpos.device)
        return st


@dataclass
class FixedLagState:
    """Device-resident state of S live streams smoothed with a fixed lag L (`SeqRetargeting.retarget_fixed_lag`, the
    `dexr_fixed_lag_t` state): the anchor and DexPilot flags after the last committed frame and a window of up to L frames
    received but not yet committed.  Resumable / checkpointable as `StreamState`."""

    lag: int
    last_qpos: "torch.Tensor"          # [S, opt_dof] float32, the last committed frame (a fresh stream: the warm start)
    projected: Optional["torch.Tensor"]  # [S, len_proj] uint8 (DexPilot) or None
    window_keypoints: "torch.Tensor"   # [S, L+1, 21, 3] float32
    window_fixed_qpos: Optional["torch.Tensor"]  # [S, L+1, n_fixed] float32, or None without fixed joints
    window_qpos: "torch.Tensor"        # [S, L+1, opt_dof] float32
    window_len: "torch.Tensor"         # [S] int32, frames held (0..L)
    # the acceleration penalty c (`dexr_fixed_lag_step_accel`), fixed for the life of the state like the lag; 0: none, and
    # the two fields after it are None
    accel_weight: float = 0.0
    prev_qpos: Optional["torch.Tensor"] = None  # [S, opt_dof] float32, the frame committed before last_qpos (raw)
    has_prev: Optional["torch.Tensor"] = None   # [S] int32, 0 fresh, 1 after the first commit

    _FIELDS = ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len", "prev_qpos",
               "has_prev")

    def state_dict(self) -> dict:
        """Host copies of every tensor (None stays None) and the lag: a run resumed from it continues bit-identically.  An
        accelerated state also holds accel_weight, prev_qpos and has_prev; a c = 0 state has none of these keys."""
        keys = self._FIELDS if self.accel_weight else self._FIELDS[:-2]
        d = {k: (None if getattr(self, k) is None else getattr(self, k).detach().cpu().clone()) for k in keys}
        d["lag"] = int(self.lag)
        if self.accel_weight:
            d["accel_weight"] = float(self.accel_weight)
        return d

    @classmethod
    def from_state_dict(cls, state: dict, device=None) -> "FixedLagState":
        """Inverse of `state_dict`: copies of its tensors on `device`.  A checkpoint without accel_weight is a c = 0 state."""
        import torch

        accel = float(state.get("accel_weight") or 0.0)
        required = ("lag", "last_qpos", "window_keypoints", "window_qpos", "window_len")
        missing = [k for k in required + (("prev_qpos", "has_prev") if accel else ()) if state.get(k) is None]
        if missing:
            raise ValueError(f"fixed-lag state checkpoint lacks {missing}")
        if not accel and (state.get("prev_qpos") is not None or state.get("has_prev") is not None):
            raise ValueError("fixed-lag state checkpoint: prev_qpos / has_prev without accel_weight")
        S, lag = int(state["last_qpos"].shape[0]), int(state["lag"])
        for k in cls._FIELDS[1:]:
            t = state.get(k)
            if t is not None and int(t.shape[0]) != S:
                raise ValueError(f"fixed-lag state checkpoint: {k} holds {int(t.shape[0])} streams, last_qpos {S}")
        for k in ("window_keypoints", "window_fixed_qpos", "window_qpos"):
            t = state.get(k)
            if t is not None and int(t.shape[1]) != lag + 1:
                raise ValueError(f"fixed-lag state checkpoint: {k} holds {int(t.shape[1])} frames, lag {lag} needs {lag + 1}")

        def put(t):  # (a copy: the restored state never aliases the checkpoint)
            return None if t is None else torch.as_tensor(t).to(device if device is not None else t.device, copy=True).contiguous()

        return cls(lag=lag, accel_weight=accel, **{k: put(state.get(k)) for k in cls._FIELDS})


def _refuse_accel_backward(state: FixedLagState, what: str, taped: bool = True):
    """The velocity-only backward entry points have no slot for the pre-anchor's cotangent: refuse an accelerated state
    there rather than differentiate the velocity-only problem (its backward is the *_accel_vjp family)."""
    if taped and state.accel_weight:
        raise ValueError(f"{what}: this backward is the velocity-only one; fixed-lag streams with an acceleration penalty "
                         f"(accel_weight = {state.accel_weight}) backpropagate through retarget_fixed_lag_accel_vjp, "
                         "flush_fixed_lag_accel_vjp and the differentiable_*_fixed_lag_accel functions, with a tape from "
                         "make_fixed_lag_tape(..., accel_weight=c)")


def _check_tape_accel(state: FixedLagState, tape: Optional["FixedLagTape"]):
    """`retarget_fixed_lag(tape=...)` records through the kernel of the state's c, so the tape must have been made for that
    c: a velocity-only tape on an accelerated state is `_refuse_accel_backward`'s refusal, any other mismatch a ValueError."""
    if tape is None or float(getattr(tape, "accel_weight", 0.0) or 0.0) == float(state.accel_weight):
        return
    if not getattr(tape, "accel_weight", 0.0):
        _refuse_accel_backward(state, "retarget_fixed_lag(tape=...)")
    raise ValueError(f"retarget_fixed_lag(tape=...): the tape was made for accel_weight = {tape.accel_weight}, the state "
                     f"has {state.accel_weight}: record with make_fixed_lag_tape(..., accel_weight={state.accel_weight})")


@dataclass
class FixedLagTape:
    """What a recorded `retarget_fixed_lag` call leaves for its backward (`dexr_fixed_lag_tape_t`): torch tensors on the
    optimizer's device.  S K (L+1) opt_dof floats: 84 MB at S = 256, K = 300, L = 16, opt_dof = 16."""

    qpos: "torch.Tensor"                 # [S, K, L+1, opt_dof] float32: each tick's window minimiser
    projected: Optional["torch.Tensor"]  # [S, K, len_proj] uint8: the committed flags each tick's solve started from, or None
    # the acceleration penalty c of the state it records (`dexr_fixed_lag_step_accel_tape`); 0: a velocity-only state
    accel_weight: float = 0.0


@dataclass
class SequenceTape:
    """What a recorded `retarget_sequences` call leaves for its backward (`dexr_sequences_tape_t`): torch tensors on the
    optimizer's device."""

    qpos: "torch.Tensor"                 # [S, T, opt_dof] float32: every frame's unfiltered solution
    projected: Optional["torch.Tensor"]  # [S, T, len_proj] uint8: the DexPilot flags after every frame, or None


@dataclass
class PackedStreams:
    """Layout of S streams of any lengths packed end to end (`SeqRetargeting.pack_streams`): stream s owns frames
    offsets[s] .. offsets[s+1]-1 of every per-frame tensor [N,...]; per-stream tensors (`StreamState`) stay [S,...]."""

    lengths: tuple                # S host ints
    offsets: "torch.Tensor"       # [S+1] int64 on the device

    @property
    def num_streams(self) -> int:
        return len(self.lengths)

    @property
    def num_frames(self) -> int:
        return int(sum(self.lengths))

    def split(self, t):
        """Per-stream views of a packed tensor [N,...]: a list of S tensors [len_s,...]."""
        if int(t.shape[0]) != self.num_frames:
            raise ValueError(f"packed tensor has {int(t.shape[0])} frames, the layout {self.num_frames}")
        return list(t.split(list(self.lengths), dim=0))


def _checker(dev):
    """The shape / dtype / device check of the stream calls' tensor arguments; returns the data pointer."""

    def chk(t, shape, dtype, name):
        if t.device != dev or t.dtype != dtype or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
            raise ValueError(f"{name}: expected contiguous {dtype} tensor of shape {tuple(shape)} on {dev}, "
                             f"got {t.dtype} {tuple(t.shape)} on {t.device}")
        return t.data_ptr()

    return chk


def _quat_to_matrix(q):
    w, x, y, z = (float(v) for v in q)
    n = (w * w + x * x + y * y + z * z) ** 0.5
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
    ])


def _intrinsic_xyz_from_matrix(R):
    """Angles (a, b, c) with R = Rx(a) Ry(b) Rz(c) (intrinsic x-y'-z'')."""
    sb = float(np.clip(R[0, 2], -1.0, 1.0))
    b = np.arcsin(sb)
    if abs(sb) < 1 - 1e-10:
        a = np.arctan2(-R[1, 2], R[2, 2])
        c = np.arctan2(-R[0, 1], R[0, 0])
    else:  # gimbal lock: put everything into the first angle
        a = np.arctan2(R[2, 1], R[1, 1])
        c = 0.0
    return np.array([a, b, c])


class SeqRetargeting:
    def __init__(self, optimizer: Optimizer, has_joint_limits=True, lp_filter: Optional[LPFilter] = None):
        self.optimizer = optimizer
        robot = optimizer.robot

        self.has_joint_limits = has_joint_limits
        joint_limits = np.ones_like(robot.joint_limits)
        joint_limits[:, 0] = -1e4  # a large value is equivalent to no limit
        joint_limits[:, 1] = 1e4
        if has_joint_limits:
            joint_limits[:] = robot.joint_limits[:]
            optimizer.set_joint_limit(joint_limits[optimizer.idx_pin2target])
        self.joint_limits = joint_limits[optimizer.idx_pin2target]

        self.last_qpos = joint_limits.mean(1)[optimizer.idx_pin2target].astype(np.float32)
        self._damping = np.zeros(1, dtype=np.float32)  # the stream's carried solver damping (Optimizer.retarget, `damping`)
        self.accumulated_time = 0
        self.num_retargeting = 0
        self.filter = lp_filter
        self.is_warm_started = False

    # ------------------------------------------------------------------------------ single stream
    def warm_start(self, wrist_pos: np.ndarray, wrist_quat: np.ndarray, hand_type: HandType = HandType.right,
                   is_mano_convention: bool = False):
        """Analytic initialisation of the 6 dummy free joints from a wrist pose (position retargeting
        with a flying hand; seq_retarget.py:45-110).  wrist_quat is (w, x, y, z)."""
        if len(wrist_pos) != 3:
            raise ValueError(f"Wrist pos: {wrist_pos} is not a 3-dim vector.")
        if len(wrist_quat) != 4:
            raise ValueError(f"Wrist quat: {wrist_quat} is not a 4-dim vector.")
        operator2mano = OPERATOR2MANO[hand_type] if is_mano_convention else np.eye(3)
        robot = self.optimizer.robot
        target_wrist_pose = np.eye(4)
        target_wrist_pose[:3, :3] = _quat_to_matrix(wrist_quat) @ operator2mano.T
        target_wrist_pose[:3, 3] = wrist_pos

        wrist_link_id = robot.get_joint_parent_child_frames(DUMMY_JOINT_NAMES[5])[1]
        qpos = robot.q0.copy()
        for num, name in enumerate(self.optimizer.target_joint_names):
            if name in DUMMY_JOINT_NAMES:
                qpos[num] = 0
        robot.compute_forward_kinematics(qpos)
        root2wrist = robot.get_link_pose_inv(wrist_link_id)
        target_root_pose = target_wrist_pose @ root2wrist
        pose_vec = np.concatenate([target_root_pose[:3, 3], _intrinsic_xyz_from_matrix(target_root_pose[:3, :3])])
        for num, name in enumerate(self.optimizer.target_joint_names):
            if name in DUMMY_JOINT_NAMES:
                self.last_qpos[num] = pose_vec[DUMMY_JOINT_NAMES.index(name)]
        self.is_warm_started = True

    def warm_start_batch(self, last_qpos, wrist_pos, wrist_quat, hand_type: HandType = HandType.right,
                         is_mano_convention: bool = False):
        """Batched `warm_start` (seq_retarget.py:45-110) for S streams: writes the analytic 6-D dummy-joint
        pose into `last_qpos` [S, opt_dof] (a torch tensor on any device, e.g. `StreamState.last_qpos`) from
        wrist positions [S,3] and quaternions [S,4] (w, x, y, z).  Pure tensor algebra, no host round trip."""
        import torch

        if wrist_pos.shape[-1] != 3 or wrist_quat.shape[-1] != 4:
            raise ValueError("wrist_pos must be [S,3] and wrist_quat [S,4]")
        robot = self.optimizer.robot
        names = self.optimizer.target_joint_names
        cols = [names.index(n) if n in names else -1 for n in DUMMY_JOINT_NAMES]
        if min(cols) < 0:
            raise ValueError("warm_start needs the 6 dummy free joints among the optimised joints")
        dt, dev = last_qpos.dtype, last_qpos.device
        # constant of the robot: root -> wrist transform with the dummy joints at zero
        qpos = robot.q0.copy()
        for num, name in enumerate(names):
            if name in DUMMY_JOINT_NAMES:
                qpos[num] = 0
        robot.compute_forward_kinematics(qpos)
        wrist_link_id = robot.get_joint_parent_child_frames(DUMMY_JOINT_NAMES[5])[1]
        root2wrist = torch.as_tensor(robot.get_link_pose_inv(wrist_link_id), dtype=torch.float64, device=dev)
        o2m = torch.as_tensor(OPERATOR2MANO[hand_type] if is_mano_convention else np.eye(3), dtype=torch.float64, device=dev)
        q = wrist_quat.to(torch.float64)
        q = q / q.norm(dim=-1, keepdim=True)
        w, x, y, z = q.unbind(-1)
        Rw = torch.stack([
            torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
            torch.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
            torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2) @ o2m.T
        R = Rw @ root2wrist[:3, :3]
        t = (Rw @ root2wrist[:3, 3]) + wrist_pos.to(torch.float64)
        sb = R[..., 0, 2].clamp(-1.0, 1.0)
        b = torch.asin(sb)
        regular = sb.abs() < 1 - 1e-10
        a = torch.where(regular, torch.atan2(-R[..., 1, 2], R[..., 2, 2]), torch.atan2(R[..., 2, 1], R[..., 1, 1]))
        c = torch.where(regular, torch.atan2(-R[..., 0, 1], R[..., 0, 0]), torch.zeros_like(b))
        pose = torch.cat([t, torch.stack([a, b, c], -1)], dim=-1).to(dt)
        last_qpos[:, cols] = pose
        self.is_warm_started = True
        return last_qpos

    def retarget(self, ref_value, fixed_qpos=np.array([])):
        tic = time.perf_counter()
        qpos = self.optimizer.retarget(
            ref_value=np.asarray(ref_value).astype(np.float32),
            fixed_qpos=np.asarray(fixed_qpos).astype(np.float32),
            last_qpos=np.clip(self.last_qpos, self.joint_limits[:, 0], self.joint_limits[:, 1]),
            damping=self._damping,
        )
        self.accumulated_time += time.perf_counter() - tic
        self.num_retargeting += 1
        self.last_qpos = qpos
        robot_qpos = np.zeros(self.optimizer.robot.dof)
        robot_qpos[self.optimizer.idx_pin2fixed] = fixed_qpos
        robot_qpos[self.optimizer.idx_pin2target] = qpos
        if self.optimizer.adaptor is not None:
            robot_qpos = self.optimizer.adaptor.forward_qpos(robot_qpos)
        if self.filter is not None:
            robot_qpos = self.filter.next(robot_qpos)
        return robot_qpos

    def set_qpos(self, robot_qpos: np.ndarray):
        self.last_qpos = np.asarray(robot_qpos)[self.optimizer.idx_pin2target]
        self._damping[:] = 0  # a new warm start: the solver's default damping again

    def get_qpos(self, fixed_qpos: Optional[np.ndarray] = None):
        robot_qpos = np.zeros(self.optimizer.robot.dof)
        robot_qpos[self.optimizer.idx_pin2target] = self.last_qpos
        if fixed_qpos is not None:
            robot_qpos[self.optimizer.idx_pin2fixed] = fixed_qpos
        return robot_qpos

    def verbose(self):
        print(f"Retargeting {self.num_retargeting} times takes: {self.accumulated_time}s")
        print(f"Last distance: {self.optimizer.opt.last_optimum_value()}")

    def reset(self):
        self.last_qpos = self.joint_limits.mean(1).astype(np.float32)
        self._damping[:] = 0
        self.num_retargeting = 0
        self.accumulated_time = 0

    @property
    def joint_names(self):
        return self.optimizer.robot.dof_joint_names

    # ------------------------------------------------------------------------------ batched streams
    @property
    def low_pass_alpha(self) -> float:
        return float(self.filter.alpha) if self.filter is not None else -1.0

    def make_stream_state(self, num_streams: int) -> StreamState:
        """Initial state of S fresh streams: mid-range warm start (seq_retarget.py:33-35), filter not
        initialised, no DexPilot projection."""
        import torch

        opt = self.optimizer
        dev = torch.device("cuda", opt.device_index)
        last = torch.from_numpy(np.ascontiguousarray(self.joint_limits.mean(1), dtype=np.float32)).to(dev)
        len_proj = opt._objective_spec().len_proj
        return StreamState(
            last_qpos=last[None].repeat(num_streams, 1).contiguous(),
            filter_state=torch.zeros((num_streams, opt.robot.dof), dtype=torch.float32, device=dev),
            filter_init=torch.zeros((num_streams,), dtype=torch.uint8, device=dev),
            projected=torch.zeros((num_streams, len_proj), dtype=torch.uint8, device=dev) if len_proj else None,
            damping=torch.zeros((num_streams,), dtype=torch.float32, device=dev),
        )

    def make_sequence_tape(self, num_streams: int, num_steps: int) -> SequenceTape:
        """Empty tape buffers for a recorded `retarget_sequences` call of S streams x T frames."""
        import torch

        opt = self.optimizer
        dev = torch.device("cuda", opt.device_index)
        len_proj = opt._objective_spec().len_proj
        return SequenceTape(
            qpos=torch.empty((num_streams, num_steps, opt.opt_dof), dtype=torch.float32, device=dev),
            projected=(torch.empty((num_streams, num_steps, len_proj), dtype=torch.uint8, device=dev)
                       if opt.retargeting_type == "DEXPILOT" else None))

    def retarget_sequences(self, keypoints, state: Optional[StreamState] = None, fixed_qpos=None, out=None,
                           status_out=None, stream=None, raw_hand=None, tape: Optional[SequenceTape] = None):
        """keypoints: float32 CUDA tensor [S,T,21,3] (raw 21-point hand frames).  Runs every stream
        through T SeqRetargeting.retarget() steps in one launch.  Returns (robot_qpos [S,T,dof] float32
        in pinocchio joint order, filtered; state) -- `state` is updated in place and can be passed
        to the next call to continue the streams.  `raw_hand` (HandType): the keypoints are raw detector landmarks of that
        hand, pre-processed inside the kernel (Optimizer.params).
        `tape` (`make_sequence_tape(S, T)`): the same launch also records what `retarget_sequences_vjp` needs
        (`dexr_solve_sequences_tape`); the results are bit-identical to an unrecorded call."""
        if tape is not None and raw_hand is not None:
            raise ValueError("raw_hand with a tape: raw-landmark pre-processing is not differentiated; pre-process the "
                             "keypoints (dexr_preprocess_keypoints) and record the call without raw_hand")
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        if keypoints.dim() != 4 or tuple(keypoints.shape[2:]) != (N.NUM_KEYPOINTS, 3):
            raise ValueError(f"keypoints must have shape [S,T,21,3], got {tuple(keypoints.shape)}")
        S, T = int(keypoints.shape[0]), int(keypoints.shape[1])
        if state is None:
            state = self.make_stream_state(S)

        def chk(t, shape, dtype, name):
            if t.device != dev or t.dtype != dtype or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
                raise ValueError(f"{name}: expected contiguous {dtype} tensor of shape {tuple(shape)} on {dev}, "
                                 f"got {t.dtype} {tuple(t.shape)} on {t.device}")
            return t.data_ptr()

        io = N.DexrSequences()
        io.keypoints = chk(keypoints, (S, T, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        nf = len(opt.idx_pin2fixed)
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (S, T, nf), torch.float32, "fixed_qpos")
        io.last_qpos = chk(state.last_qpos, (S, opt.opt_dof), torch.float32, "state.last_qpos")
        io.filter_state = chk(state.filter_state, (S, opt.robot.dof), torch.float32, "state.filter_state")
        io.filter_init = chk(state.filter_init, (S,), torch.uint8, "state.filter_init")
        if state.projected is not None:
            io.projected = chk(state.projected, (S, state.projected.shape[1]), torch.uint8, "state.projected")
        if state.damping is not None:
            io.damping_state = chk(state.damping, (S,), torch.float32, "state.damping")
        if out is None:
            out = torch.empty((S, T, opt.robot.dof), dtype=torch.float32, device=dev)
        io.robot_qpos_out = chk(out, (S, T, opt.robot.dof), torch.float32, "out")
        if status_out is not None:
            io.status_out = chk(status_out, (S, T), torch.int32, "status_out")
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha, raw_hand=raw_hand)
        if tape is None:
            N.check(eng.lib.dexr_solve_sequences(eng.handle, C.byref(p), C.byref(io), S, T, C.c_void_p(s.cuda_stream)),
                    "dexr_solve_sequences")
            return out, state
        tp = N.DexrSequencesTape()
        tp.qpos = chk(tape.qpos, (S, T, opt.opt_dof), torch.float32, "tape.qpos")
        if tape.projected is not None:
            tp.projected = chk(tape.projected, (S, T, opt._objective_spec().len_proj), torch.uint8, "tape.projected")
        N.check(eng.lib.dexr_solve_sequences_tape(eng.handle, C.byref(p), C.byref(io), C.byref(tp), S, T,
                                                  C.c_void_p(s.cuda_stream)), "dexr_solve_sequences_tape")
        return out, state

    def retarget_sequences_vjp(self, keypoints, tape: SequenceTape, last_qpos0, filter_init0, grad_robot_qpos=None,
                               grad_last_qpos=None, grad_filter_state=None, fixed_qpos=None, grad_keypoints_out=None,
                               grad_fixed_qpos_out=None, grad_last_qpos_out=None, grad_filter_state_out=None,
                               status_out=None, stream=None):
        """Backpropagate through a recorded `retarget_sequences(keypoints, state, fixed_qpos, tape=tape)` call, one launch
        (`dexr_solve_sequences_vjp`).  `last_qpos0` [S,opt_dof] and `filter_init0` [S] uint8 are the state's `last_qpos` and
        `filter_init` as they were BEFORE that call; the cotangents are dl/drobot_qpos [S,T,dof] (`grad_robot_qpos`) and
        dl/d the final `state.last_qpos` / `state.filter_state` (`grad_last_qpos`, `grad_filter_state`), each None for 0.
        Returns (grad_keypoints [S,T,21,3], grad_fixed_qpos [S,T,n_fixed] or None, grad_last_qpos0 [S,opt_dof],
        grad_filter_state0 [S,dof]): the gradients with respect to the call's keypoints, fixed joints and initial state.
        Every frame is differentiated as by `Optimizer.retarget_batch_vjp` at its recorded solution and clipped anchor;
        the DexPilot flags, the carried damping and the basin the warm start picks are not differentiated.  `status_out`
        [S,T] int32 receives 0, STATUS_NONFINITE (this frame or a later one of the stream is non-finite: NaN outputs) or
        STATUS_NOT_PD (zero cotangents through the solve).  Keypoints must not be raw landmarks.  Nothing is synchronised."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        if keypoints.dim() != 4 or tuple(keypoints.shape[2:]) != (N.NUM_KEYPOINTS, 3):
            raise ValueError(f"keypoints must have shape [S,T,21,3], got {tuple(keypoints.shape)}")
        S, T = int(keypoints.shape[0]), int(keypoints.shape[1])
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)

        def chk(t, shape, dtype, name):
            if t.device != dev or t.dtype != dtype or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
                raise ValueError(f"{name}: expected contiguous {dtype} tensor of shape {tuple(shape)} on {dev}, "
                                 f"got {t.dtype} {tuple(t.shape)} on {t.device}")
            return t.data_ptr()

        def out(t, shape, name):
            t = torch.empty(shape, dtype=torch.float32, device=dev) if t is None else t
            return t, chk(t, shape, torch.float32, name)

        io = N.DexrSequencesVjp()
        io.keypoints = chk(keypoints, (S, T, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (S, T, nf), torch.float32, "fixed_qpos")
        io.last_qpos = chk(last_qpos0, (S, n), torch.float32, "last_qpos0")
        io.filter_init = chk(filter_init0, (S,), torch.uint8, "filter_init0")
        io.qpos = chk(tape.qpos, (S, T, n), torch.float32, "tape.qpos")
        if tape.projected is not None:
            io.projected = chk(tape.projected, (S, T, opt._objective_spec().len_proj), torch.uint8, "tape.projected")
        if grad_robot_qpos is not None:
            io.grad_robot_qpos = chk(grad_robot_qpos, (S, T, dof), torch.float32, "grad_robot_qpos")
        if grad_last_qpos is not None:
            io.grad_last_qpos_out = chk(grad_last_qpos, (S, n), torch.float32, "grad_last_qpos")
        if grad_filter_state is not None:
            io.grad_filter_state_out = chk(grad_filter_state, (S, dof), torch.float32, "grad_filter_state")
        g_kp, io.grad_keypoints = out(grad_keypoints_out, (S, T, N.NUM_KEYPOINTS, 3), "grad_keypoints_out")
        g_fixed = None
        if nf:
            g_fixed, io.grad_fixed_qpos = out(grad_fixed_qpos_out, (S, T, nf), "grad_fixed_qpos_out")
        g_last, io.grad_last_qpos = out(grad_last_qpos_out, (S, n), "grad_last_qpos_out")
        g_filter, io.grad_filter_state = out(grad_filter_state_out, (S, dof), "grad_filter_state_out")
        if status_out is not None:
            io.status_out = chk(status_out, (S, T), torch.int32, "status_out")
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        N.check(eng.lib.dexr_solve_sequences_vjp(eng.handle, C.byref(p), C.byref(io), S, T, C.c_void_p(s.cuda_stream)),
                "dexr_solve_sequences_vjp")
        return g_kp, g_fixed, g_last, g_filter

    # ------------------------------------------------------------------------------ packed streams (any lengths)
    def pack_streams(self, lengths) -> PackedStreams:
        """The layout of S streams of the given frame counts (0 allowed), packed end to end in that order.  Validated on
        the host; the offsets are uploaded without synchronising (a pinned host copy).  Build it once per batch of clips
        and pass it to every packed call on them.  The streams are dealt to warps in this order; dealing them longest first
        measured no faster on an H100 (DESIGN.md section 3.11)."""
        import torch

        lens = np.asarray(lengths)
        if lens.ndim != 1 or (lens.size and not np.issubdtype(lens.dtype, np.integer)):
            raise ValueError(f"lengths must be a 1-D sequence of ints, got {lens.dtype} of shape {lens.shape}")
        lens = lens.astype(np.int64)
        if (lens < 0).any():
            raise ValueError("stream lengths must be >= 0")
        if int(lens.sum()) > np.iinfo(np.int32).max:
            raise ValueError("at most 2**31 - 1 frames in one packed batch")
        offsets = np.zeros(lens.size + 1, np.int64)
        np.cumsum(lens, out=offsets[1:])
        dev = torch.device("cuda", self.optimizer.device_index)
        return PackedStreams(lengths=tuple(int(v) for v in lens),
                             offsets=torch.from_numpy(offsets).pin_memory().to(dev, non_blocking=True))

    def make_packed_sequence_tape(self, layout: PackedStreams) -> SequenceTape:
        """Empty tape buffers for a recorded `retarget_packed_sequences` call: qpos [N,opt_dof], projected [N,len_proj]."""
        import torch

        opt = self.optimizer
        dev = torch.device("cuda", opt.device_index)
        N_ = layout.num_frames
        len_proj = opt._objective_spec().len_proj
        return SequenceTape(
            qpos=torch.empty((N_, opt.opt_dof), dtype=torch.float32, device=dev),
            projected=(torch.empty((N_, len_proj), dtype=torch.uint8, device=dev)
                       if opt.retargeting_type == "DEXPILOT" else None))

    def retarget_packed_sequences(self, keypoints, layout: PackedStreams, state: Optional[StreamState] = None,
                                  fixed_qpos=None, out=None, status_out=None, stream=None, raw_hand=None,
                                  tape: Optional[SequenceTape] = None):
        """`retarget_sequences` for S streams of any lengths in one launch (`dexr_solve_sequences_packed`): keypoints
        [N,21,3] float32 CUDA tensor with stream s at frames layout.offsets[s] .. offsets[s+1]-1 (`pack_streams`),
        fixed_qpos [N,n_fixed].  Returns (robot_qpos [N,dof], state); `state` ([S,...], `make_stream_state(S)`) is updated
        in place, each stream ending at its own last frame (a stream of length 0 keeps its state), so chunks of the same
        clips chain exactly.  Every stream's results are bit-identical to a `retarget_sequences` call on it alone.
        `tape` (`make_packed_sequence_tape(layout)`) records the call for `retarget_packed_sequences_vjp`."""
        if tape is not None and raw_hand is not None:
            raise ValueError("raw_hand with a tape: raw-landmark pre-processing is not differentiated; pre-process the "
                             "keypoints (dexr_preprocess_keypoints) and record the call without raw_hand")
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        S, N_ = layout.num_streams, layout.num_frames
        chk = _checker(dev)
        if state is None:
            state = self.make_stream_state(S)
        io = N.DexrSequences()
        io.keypoints = chk(keypoints, (N_, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        nf = len(opt.idx_pin2fixed)
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (N_, nf), torch.float32, "fixed_qpos")
        io.last_qpos = chk(state.last_qpos, (S, opt.opt_dof), torch.float32, "state.last_qpos")
        io.filter_state = chk(state.filter_state, (S, opt.robot.dof), torch.float32, "state.filter_state")
        io.filter_init = chk(state.filter_init, (S,), torch.uint8, "state.filter_init")
        if state.projected is not None:
            io.projected = chk(state.projected, (S, state.projected.shape[1]), torch.uint8, "state.projected")
        if state.damping is not None:
            io.damping_state = chk(state.damping, (S,), torch.float32, "state.damping")
        if out is None:
            out = torch.empty((N_, opt.robot.dof), dtype=torch.float32, device=dev)
        io.robot_qpos_out = chk(out, (N_, opt.robot.dof), torch.float32, "out")
        if status_out is not None:
            io.status_out = chk(status_out, (N_,), torch.int32, "status_out")
        tp = None
        if tape is not None:
            tp = N.DexrSequencesTape()
            tp.qpos = chk(tape.qpos, (N_, opt.opt_dof), torch.float32, "tape.qpos")
            if tape.projected is not None:
                tp.projected = chk(tape.projected, (N_, opt._objective_spec().len_proj), torch.uint8, "tape.projected")
        offsets = chk(layout.offsets, (S + 1,), torch.int64, "layout.offsets")
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha, raw_hand=raw_hand)
        N.check(eng.lib.dexr_solve_sequences_packed(eng.handle, C.byref(p), C.byref(io), None if tp is None else C.byref(tp),
                                                    C.c_void_p(offsets), S, N_,
                                                    C.c_void_p(s.cuda_stream)), "dexr_solve_sequences_packed")
        return out, state

    def retarget_packed_sequences_vjp(self, keypoints, layout: PackedStreams, tape: SequenceTape, last_qpos0, filter_init0,
                                      grad_robot_qpos=None, grad_last_qpos=None, grad_filter_state=None, fixed_qpos=None,
                                      grad_keypoints_out=None, grad_fixed_qpos_out=None, grad_last_qpos_out=None,
                                      grad_filter_state_out=None, status_out=None, stream=None):
        """`retarget_sequences_vjp` for a recorded `retarget_packed_sequences` call, one launch
        (`dexr_solve_sequences_packed_vjp`): per-frame tensors [N,...] (keypoints, fixed_qpos, tape, grad_robot_qpos,
        status_out and the returned grad_keypoints / grad_fixed_qpos), per-stream ones [S,...] (last_qpos0, filter_init0,
        grad_last_qpos, grad_filter_state and the returned initial-state gradients).  A stream of length 0 passes its
        state cotangents through.  Nothing is synchronised."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        S, N_ = layout.num_streams, layout.num_frames
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)
        chk = _checker(dev)

        def out(t, shape, name):
            t = torch.empty(shape, dtype=torch.float32, device=dev) if t is None else t
            return t, chk(t, shape, torch.float32, name)

        io = N.DexrSequencesVjp()
        io.keypoints = chk(keypoints, (N_, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (N_, nf), torch.float32, "fixed_qpos")
        io.last_qpos = chk(last_qpos0, (S, n), torch.float32, "last_qpos0")
        io.filter_init = chk(filter_init0, (S,), torch.uint8, "filter_init0")
        io.qpos = chk(tape.qpos, (N_, n), torch.float32, "tape.qpos")
        if tape.projected is not None:
            io.projected = chk(tape.projected, (N_, opt._objective_spec().len_proj), torch.uint8, "tape.projected")
        if grad_robot_qpos is not None:
            io.grad_robot_qpos = chk(grad_robot_qpos, (N_, dof), torch.float32, "grad_robot_qpos")
        if grad_last_qpos is not None:
            io.grad_last_qpos_out = chk(grad_last_qpos, (S, n), torch.float32, "grad_last_qpos")
        if grad_filter_state is not None:
            io.grad_filter_state_out = chk(grad_filter_state, (S, dof), torch.float32, "grad_filter_state")
        g_kp, io.grad_keypoints = out(grad_keypoints_out, (N_, N.NUM_KEYPOINTS, 3), "grad_keypoints_out")
        g_fixed = None
        if nf:
            g_fixed, io.grad_fixed_qpos = out(grad_fixed_qpos_out, (N_, nf), "grad_fixed_qpos_out")
        g_last, io.grad_last_qpos = out(grad_last_qpos_out, (S, n), "grad_last_qpos_out")
        g_filter, io.grad_filter_state = out(grad_filter_state_out, (S, dof), "grad_filter_state_out")
        if status_out is not None:
            io.status_out = chk(status_out, (N_,), torch.int32, "status_out")
        offsets = chk(layout.offsets, (S + 1,), torch.int64, "layout.offsets")
        if N_ == 0:  # (the library does nothing for 0 frames: every stream is empty and passes its cotangents through)
            g_last.copy_(grad_last_qpos) if grad_last_qpos is not None else g_last.zero_()
            g_filter.copy_(grad_filter_state) if grad_filter_state is not None else g_filter.zero_()
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        N.check(eng.lib.dexr_solve_sequences_packed_vjp(eng.handle, C.byref(p), C.byref(io), C.c_void_p(offsets), S, N_,
                                                        C.c_void_p(s.cuda_stream)),
                "dexr_solve_sequences_packed_vjp")
        return g_kp, g_fixed, g_last, g_filter

    def smooth_packed_sequences(self, keypoints, layout: PackedStreams, state: Optional[StreamState] = None, *,
                                fixed_qpos=None, qpos_init=None, smooth_weight=None, accel_weight=None, out=None,
                                status_out=None, stream=None):
        """Offline smoothing of recorded clips (`dexr_smooth_sequences_packed`, one launch): every frame of each packed
        stream solved jointly, minimising sum_t L_t(x_t) + w sum_t |x_t - x_{t-1}|^2 + w |x_0 - clip(a)|^2 over the
        clip.  With w = norm_delta (`smooth_weight` None) this is the sum of the costs `retarget_packed_sequences` minimises
        one frame at a time, without its lag.  keypoints [N,21,3] (wrist-centred, not raw landmarks) and fixed_qpos
        [N,n_fixed] as for `retarget_packed_sequences`; `state` is read only: the anchor a is `state.last_qpos` and the
        DexPilot flags start at `state.projected` (None: a fresh `make_stream_state`).  `qpos_init` [N,opt_dof] is the
        starting trajectory; None runs the taped `retarget_packed_sequences` on a copy of the state and starts from its
        tape.  A frame with a non-finite keypoint or fixed joint is filled in by the smoothness terms (STATUS_MISSING).
        Returns (robot_qpos [N,dof] (scatter + mimic, no low-pass filter), qpos [N,opt_dof], status [N] int32); a stream
        whose status has STATUS_MAXITER returns its last accepted iterate (lower F than its start), not the minimiser.
        `accel_weight` c > 0 adds c sum_t |x_{t+1} - 2 x_t + x_{t-1}|^2, the anchor counting as frame -1
        (`dexr_smooth_sequences_packed_accel`): an acceleration penalty, which leaves constant-velocity motion alone; None
        or 0 is the call above.  Allocates its workspace on the device; nothing is synchronised."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        S, N_ = layout.num_streams, layout.num_frames
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)
        chk = _checker(dev)
        if state is None:
            state = self.make_stream_state(S)
        io = N.DexrSmooth()
        io.keypoints = chk(keypoints, (N_, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (N_, nf), torch.float32, "fixed_qpos")
        io.last_qpos = chk(state.last_qpos, (S, n), torch.float32, "state.last_qpos")
        if state.projected is not None:
            io.projected = chk(state.projected, (S, state.projected.shape[1]), torch.uint8, "state.projected")
        offsets = chk(layout.offsets, (S + 1,), torch.int64, "layout.offsets")
        if qpos_init is None:
            tape = self.make_packed_sequence_tape(layout)
            copy = StreamState(**{k: (None if getattr(state, k) is None else getattr(state, k).clone())
                                  for k in StreamState._FIELDS})
            self.retarget_packed_sequences(keypoints, layout, copy, fixed_qpos=fixed_qpos, stream=stream, tape=tape)
            qpos_init = tape.qpos
        io.qpos_init = chk(qpos_init, (N_, n), torch.float32, "qpos_init")
        qpos = torch.empty((N_, n), dtype=torch.float32, device=dev)
        io.qpos_out = qpos.data_ptr()
        if out is None:
            out = torch.empty((N_, dof), dtype=torch.float32, device=dev)
        io.robot_qpos_out = chk(out, (N_, dof), torch.float32, "out")
        if status_out is None:
            status_out = torch.empty((N_,), dtype=torch.int32, device=dev)
        io.status_out = chk(status_out, (N_,), torch.int32, "status_out")
        io.smooth_weight = -1.0 if smooth_weight is None else float(smooth_weight)
        accel = 0.0 if accel_weight is None else float(accel_weight)
        nbytes = int(eng.lib.dexr_smooth_accel_workspace_bytes(eng.handle, N_) if accel != 0.0
                     else eng.lib.dexr_smooth_workspace_bytes(eng.handle, N_))
        ws = torch.empty((max(nbytes, 4),), dtype=torch.uint8, device=dev)
        io.workspace, io.workspace_bytes = ws.data_ptr(), nbytes
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        if accel != 0.0:
            N.check(eng.lib.dexr_smooth_sequences_packed_accel(eng.handle, C.byref(p), C.byref(io), accel, C.c_void_p(offsets),
                                                               S, N_, C.c_void_p(s.cuda_stream)),
                    "dexr_smooth_sequences_packed_accel")
        else:
            N.check(eng.lib.dexr_smooth_sequences_packed(eng.handle, C.byref(p), C.byref(io), C.c_void_p(offsets), S, N_,
                                                         C.c_void_p(s.cuda_stream)), "dexr_smooth_sequences_packed")
        ws.record_stream(s)
        return out, qpos, status_out

    def smooth_packed_sequences_vjp(self, keypoints, layout: PackedStreams, qpos, last_qpos0=None, projected0=None,
                                    grad_qpos=None, grad_robot_qpos=None, *, fixed_qpos=None, smooth_weight=None,
                                    accel_weight=None, grad_keypoints_out=None, grad_fixed_qpos_out=None,
                                    grad_last_qpos_out=None, status_out=None, stream=None):
        """Backpropagation through `smooth_packed_sequences` (`dexr_smooth_sequences_packed_vjp`, one launch): the
        implicit-function VJP of the smoothed clips `qpos` [N,opt_dof] (the forward's answer) with respect to the keypoints,
        the fixed joints and the anchor.  Per-frame tensors [N,...] (keypoints, fixed_qpos, qpos, grad_qpos,
        grad_robot_qpos, status_out and the returned grad_keypoints / grad_fixed_qpos), per-stream ones [S,...]
        (last_qpos0 and projected0: the forward's `state.last_qpos` and `state.projected`; the returned grad_last_qpos).
        `smooth_weight` as given to the forward.  Returns (grad_keypoints [N,21,3], grad_fixed_qpos [N,n_fixed] or None,
        grad_last_qpos [S,opt_dof] or None when last_qpos0 is None).  The gradient is not causal: a loss on one frame
        reaches the keypoints of every frame of its stream.  A stream whose stacked Hessian is not positive definite gets
        zero gradients (STATUS_NOT_PD), one with a non-finite qpos, anchor or cotangent NaN (STATUS_NONFINITE).
        `accel_weight` as given to the forward (`dexr_smooth_sequences_packed_accel_vjp`; None or 0: the call above).
        Allocates its workspace on the device; nothing is synchronised."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        S, N_ = layout.num_streams, layout.num_frames
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)
        chk = _checker(dev)

        def out(t, shape, name):
            t = torch.empty(shape, dtype=torch.float32, device=dev) if t is None else t
            return t, chk(t, shape, torch.float32, name)

        io = N.DexrSmoothVjp()
        io.keypoints = chk(keypoints, (N_, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
        if nf:
            if fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
            io.fixed_qpos = chk(fixed_qpos, (N_, nf), torch.float32, "fixed_qpos")
        if last_qpos0 is not None:
            io.last_qpos = chk(last_qpos0, (S, n), torch.float32, "last_qpos0")
        if projected0 is not None:
            io.projected = chk(projected0, (S, projected0.shape[1]), torch.uint8, "projected0")
        io.qpos = chk(qpos, (N_, n), torch.float32, "qpos")
        if grad_qpos is not None:
            io.grad_qpos = chk(grad_qpos, (N_, n), torch.float32, "grad_qpos")
        if grad_robot_qpos is not None:
            io.grad_robot_qpos = chk(grad_robot_qpos, (N_, dof), torch.float32, "grad_robot_qpos")
        io.smooth_weight = -1.0 if smooth_weight is None else float(smooth_weight)
        g_kp, io.grad_keypoints = out(grad_keypoints_out, (N_, N.NUM_KEYPOINTS, 3), "grad_keypoints_out")
        g_fixed = None
        if nf:
            g_fixed, io.grad_fixed_qpos = out(grad_fixed_qpos_out, (N_, nf), "grad_fixed_qpos_out")
        g_last = None
        if last_qpos0 is not None:
            g_last, io.grad_last_qpos = out(grad_last_qpos_out, (S, n), "grad_last_qpos_out")
            if N_ == 0:  # (the library does nothing for 0 frames: every stream is empty)
                g_last.zero_()
        if status_out is not None:
            io.status_out = chk(status_out, (N_,), torch.int32, "status_out")
        offsets = chk(layout.offsets, (S + 1,), torch.int64, "layout.offsets")
        accel = 0.0 if accel_weight is None else float(accel_weight)
        nbytes = int(eng.lib.dexr_smooth_accel_workspace_bytes(eng.handle, N_) if accel != 0.0
                     else eng.lib.dexr_smooth_workspace_bytes(eng.handle, N_))
        ws = torch.empty((max(nbytes, 4),), dtype=torch.uint8, device=dev)
        io.workspace, io.workspace_bytes = ws.data_ptr(), nbytes
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        if accel != 0.0:
            N.check(eng.lib.dexr_smooth_sequences_packed_accel_vjp(eng.handle, C.byref(p), C.byref(io), accel,
                                                                   C.c_void_p(offsets), S, N_, C.c_void_p(s.cuda_stream)),
                    "dexr_smooth_sequences_packed_accel_vjp")
        else:
            N.check(eng.lib.dexr_smooth_sequences_packed_vjp(eng.handle, C.byref(p), C.byref(io), C.c_void_p(offsets), S,
                                                             N_, C.c_void_p(s.cuda_stream)), "dexr_smooth_sequences_packed_vjp")
        ws.record_stream(s)
        return g_kp, g_fixed, g_last

    def make_fixed_lag_state(self, num_streams: int, lag: int, accel_weight: Optional[float] = None) -> FixedLagState:
        """Initial state of S fresh live streams smoothed with lag L (`retarget_fixed_lag`): the anchor at the mid-range warm
        start (as `make_stream_state`; `warm_start_batch` applies to `last_qpos`), no DexPilot projection, an empty window.
        `accel_weight` c > 0: each window solve also penalises c |x_{t+1} - 2 x_t + x_{t-1}|^2, the frame committed before
        the anchor counting as frame -2 (`dexr_fixed_lag_step_accel`); the state then carries prev_qpos and has_prev.  c
        is fixed for the life of the state; None or 0: no acceleration penalty."""
        import torch

        lag = int(lag)
        if not 0 <= lag <= N.FIXED_LAG_MAX:
            raise ValueError(f"lag must be in 0..{N.FIXED_LAG_MAX}, got {lag}")
        accel = 0.0 if accel_weight is None else float(accel_weight)
        if not (accel == 0.0 or 0.0 < accel <= 3.0e38):
            raise ValueError(f"accel_weight must be finite and >= 0, got {accel_weight}")
        opt = self.optimizer
        base = self.make_stream_state(num_streams)
        dev = base.last_qpos.device
        nf = len(opt.idx_pin2fixed)
        return FixedLagState(
            lag=lag, last_qpos=base.last_qpos, projected=base.projected,
            window_keypoints=torch.zeros((num_streams, lag + 1, N.NUM_KEYPOINTS, 3), dtype=torch.float32, device=dev),
            window_fixed_qpos=(torch.zeros((num_streams, lag + 1, nf), dtype=torch.float32, device=dev) if nf else None),
            window_qpos=torch.zeros((num_streams, lag + 1, opt.opt_dof), dtype=torch.float32, device=dev),
            window_len=torch.zeros((num_streams,), dtype=torch.int32, device=dev), accel_weight=accel,
            prev_qpos=torch.zeros((num_streams, opt.opt_dof), dtype=torch.float32, device=dev) if accel else None,
            has_prev=torch.zeros((num_streams,), dtype=torch.int32, device=dev) if accel else None)

    def make_fixed_lag_tape(self, num_streams: int, num_ticks: int, lag: int,
                            accel_weight: Optional[float] = None) -> FixedLagTape:
        """Buffers for recording a `retarget_fixed_lag` call of K ticks on S streams of lag L (`tape=`), the input of
        `retarget_fixed_lag_vjp`.  `accel_weight` c: a tape for a state made with the same c (the layout is the same; the
        recording runs `dexr_fixed_lag_step_accel_tape`), the input of `retarget_fixed_lag_accel_vjp`."""
        import torch

        accel = 0.0 if accel_weight is None else float(accel_weight)
        if not (accel == 0.0 or 0.0 < accel <= 3.0e38):
            raise ValueError(f"accel_weight must be finite and >= 0, got {accel_weight}")

        opt = self.optimizer
        dev = torch.device("cuda", opt.engine().device)
        len_proj = opt._objective_spec().len_proj
        S, K, L = int(num_streams), int(num_ticks), int(lag)
        return FixedLagTape(
            qpos=torch.empty((S, K, L + 1, opt.opt_dof), dtype=torch.float32, device=dev),
            projected=torch.empty((S, K, len_proj), dtype=torch.uint8, device=dev) if len_proj else None,
            accel_weight=accel)

    def _fixed_lag_call(self, state: FixedLagState, K: int, fill, smooth_weight, stream, tape: Optional[FixedLagTape] = None):
        """One `dexr_fixed_lag_step` call on `state` with K ticks (`dexr_fixed_lag_step_tape` into `tape` when given,
        `dexr_fixed_lag_step_accel` for an accelerated state, `dexr_fixed_lag_step_accel_tape` for both); `fill(io, chk)`
        sets the per-call buffers."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        chk = _checker(dev)
        S, L = int(state.last_qpos.shape[0]), int(state.lag)
        n, nf = opt.opt_dof, len(opt.idx_pin2fixed)
        io = N.DexrFixedLag()
        io.lag = L
        io.last_qpos = chk(state.last_qpos, (S, n), torch.float32, "state.last_qpos")
        len_proj = opt._objective_spec().len_proj
        if len_proj:
            if state.projected is None:
                raise ValueError("DexPilot streams need state.projected")
            io.projected = chk(state.projected, (S, len_proj), torch.uint8, "state.projected")
        io.window_keypoints = chk(state.window_keypoints, (S, L + 1, N.NUM_KEYPOINTS, 3), torch.float32,
                                  "state.window_keypoints")
        if nf:
            if state.window_fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but state.window_fixed_qpos is None")
            io.window_fixed_qpos = chk(state.window_fixed_qpos, (S, L + 1, nf), torch.float32, "state.window_fixed_qpos")
        io.window_qpos = chk(state.window_qpos, (S, L + 1, n), torch.float32, "state.window_qpos")
        io.window_len = chk(state.window_len, (S,), torch.int32, "state.window_len")
        io.smooth_weight = -1.0 if smooth_weight is None else float(smooth_weight)
        fill(io, chk)
        accel = float(state.accel_weight)
        nbytes = int(eng.lib.dexr_fixed_lag_accel_workspace_bytes(eng.handle, S, L) if accel
                     else eng.lib.dexr_fixed_lag_workspace_bytes(eng.handle, S, L))
        ws = torch.empty((max(nbytes, 4),), dtype=torch.uint8, device=dev)
        io.workspace, io.workspace_bytes = ws.data_ptr(), nbytes
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        tp = None
        if tape is not None:
            tp = N.DexrFixedLagTape()
            tp.qpos = chk(tape.qpos, (S, K, L + 1, n), torch.float32, "tape.qpos")
            if len_proj:
                if tape.projected is None:
                    raise ValueError("DexPilot streams need tape.projected")
                tp.projected = chk(tape.projected, (S, K, len_proj), torch.uint8, "tape.projected")
        if accel:
            acc = N.DexrFixedLagAccel()
            acc.accel_weight = accel
            if state.prev_qpos is None or state.has_prev is None:
                raise ValueError("an accelerated fixed-lag state needs prev_qpos and has_prev")
            acc.prev_qpos = chk(state.prev_qpos, (S, n), torch.float32, "state.prev_qpos")
            acc.has_prev = chk(state.has_prev, (S,), torch.int32, "state.has_prev")
            if tp is None:
                N.check(eng.lib.dexr_fixed_lag_step_accel(eng.handle, C.byref(p), C.byref(io), C.byref(acc), S, K,
                                                          C.c_void_p(s.cuda_stream)), "dexr_fixed_lag_step_accel")
            else:
                N.check(eng.lib.dexr_fixed_lag_step_accel_tape(eng.handle, C.byref(p), C.byref(io), C.byref(acc),
                                                               C.byref(tp), S, K, C.c_void_p(s.cuda_stream)),
                        "dexr_fixed_lag_step_accel_tape")
        elif tape is None:
            N.check(eng.lib.dexr_fixed_lag_step(eng.handle, C.byref(p), C.byref(io), S, K, C.c_void_p(s.cuda_stream)),
                    "dexr_fixed_lag_step")
        else:
            N.check(eng.lib.dexr_fixed_lag_step_tape(eng.handle, C.byref(p), C.byref(io), C.byref(tp), S, K,
                                                     C.c_void_p(s.cuda_stream)), "dexr_fixed_lag_step_tape")
        ws.record_stream(s)

    def retarget_fixed_lag(self, keypoints, state: FixedLagState, *, fixed_qpos=None, smooth_weight=None, out=None,
                           qpos_out=None, status_out=None, stream=None, tape: Optional[FixedLagTape] = None):
        """Fixed-lag smoothing of S live streams (`dexr_fixed_lag_step`, one launch): each of the K new frames per stream
        (keypoints [S,K,21,3], wrist-centred; fixed_qpos [S,K,n_fixed]) re-solves the last L+1 frames of its stream jointly
        with the offline smoother (`smooth_packed_sequences`, anchored at the last committed frame, w = smooth_weight or
        norm_delta) and emits the frame L ticks back.  Until a stream's window holds L+1 frames its ticks emit NaN with
        STATUS_PENDING.  L = 0 is the causal problem; a dropped detection (NaN keypoints) is interpolated from both sides
        (STATUS_MISSING).  `state` (`make_fixed_lag_state`) is updated in place.  Returns (robot_qpos [S,K,dof] (scatter +
        mimic, no low-pass filter), qpos [S,K,opt_dof], status [S,K] int32), into `out` / `qpos_out` / `status_out` when
        given.  `tape` (`make_fixed_lag_tape(S, K, L)`): also record what `retarget_fixed_lag_vjp` needs; the outputs and
        the state are the same bits either way.  An accelerated state records into a tape made with its own accel_weight
        (for `retarget_fixed_lag_accel_vjp`); a tape whose c differs from the state's is refused (ValueError).  Allocates
        its workspace on the device; nothing is synchronised."""
        import torch

        _check_tape_accel(state, tape)
        opt = self.optimizer
        if keypoints.dim() != 4 or tuple(keypoints.shape[2:]) != (N.NUM_KEYPOINTS, 3):
            raise ValueError(f"keypoints must have shape [S,K,21,3], got {tuple(keypoints.shape)}")
        S, K = int(keypoints.shape[0]), int(keypoints.shape[1])
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)
        dev = state.last_qpos.device
        qpos = torch.empty((S, K, n), dtype=torch.float32, device=dev) if qpos_out is None else qpos_out
        if out is None:
            out = torch.empty((S, K, dof), dtype=torch.float32, device=dev)
        if status_out is None:
            status_out = torch.empty((S, K), dtype=torch.int32, device=dev)

        def fill(io, chk):
            io.keypoints = chk(keypoints, (S, K, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
            if nf:
                if fixed_qpos is None:
                    raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
                io.fixed_qpos = chk(fixed_qpos, (S, K, nf), torch.float32, "fixed_qpos")
            io.qpos_out = chk(qpos, (S, K, n), torch.float32, "qpos_out")
            io.robot_qpos_out = chk(out, (S, K, dof), torch.float32, "out")
            io.status_out = chk(status_out, (S, K), torch.int32, "status_out")

        self._fixed_lag_call(state, K, fill, smooth_weight, stream, tape)
        return out, qpos, status_out

    def flush_fixed_lag(self, state: FixedLagState, *, out=None, qpos_out=None, count_out=None, stream=None):
        """End S fixed-lag streams: emit the frames each still holds, in order, as the last tick's joint solve left them (no
        new solve), commit the last of them as the anchor and empty the windows.  Returns (robot_qpos [S,L,dof], qpos
        [S,L,opt_dof], count [S] int32), into `out` / `qpos_out` / `count_out` when given: stream s's rows 0..count[s]-1 are
        its held frames, the rest NaN."""
        import torch

        opt = self.optimizer
        S, L = int(state.last_qpos.shape[0]), int(state.lag)
        dev = state.last_qpos.device
        qpos = torch.empty((S, L, opt.opt_dof), dtype=torch.float32, device=dev) if qpos_out is None else qpos_out
        rq = torch.empty((S, L, opt.robot.dof), dtype=torch.float32, device=dev) if out is None else out
        count = torch.empty((S,), dtype=torch.int32, device=dev) if count_out is None else count_out

        def fill(io, chk):
            io.flush_qpos_out = chk(qpos, (S, L, opt.opt_dof), torch.float32, "qpos_out")
            io.flush_robot_qpos_out = chk(rq, (S, L, opt.robot.dof), torch.float32, "out")
            io.flush_count_out = chk(count, (S,), torch.int32, "count_out")

        self._fixed_lag_call(state, 0, fill, None, stream)
        return rq, qpos, count

    def _fixed_lag_vjp_call(self, state0: FixedLagState, K: int, fill, flushed: bool, smooth_weight, grads: dict, stream,
                            outputs: Optional[dict] = None, accel: bool = False):
        """One `dexr_fixed_lag_step_vjp` call: `state0` the state before the forward, `fill(io, chk, new)` the per-call
        buffers, `grads` the final state's cotangents (None = 0), `outputs` tensors to write the outputs into, by their
        dexr_fixed_lag_vjp_t names (the others are allocated).  Returns (grad_last_qpos, grad_window_keypoints,
        grad_window_fixed_qpos or None, grad_window_qpos) of state0.  `accel`: `dexr_fixed_lag_step_accel_vjp` on the
        accelerated state0 (grads may hold grad_prev_qpos_out, outputs grad_prev_qpos), grad_prev_qpos appended."""
        import torch

        opt = self.optimizer
        eng = opt.engine()
        dev = torch.device("cuda", eng.device)
        chk = _checker(dev)
        S, L = int(state0.last_qpos.shape[0]), int(state0.lag)
        n, nf = opt.opt_dof, len(opt.idx_pin2fixed)
        io = N.DexrFixedLagVjp()
        io.lag, io.flushed = L, int(bool(flushed))
        io.smooth_weight = -1.0 if smooth_weight is None else float(smooth_weight)
        io.last_qpos = chk(state0.last_qpos, (S, n), torch.float32, "state0.last_qpos")
        io.window_keypoints = chk(state0.window_keypoints, (S, L + 1, N.NUM_KEYPOINTS, 3), torch.float32,
                                  "state0.window_keypoints")
        if nf:
            if state0.window_fixed_qpos is None:
                raise ValueError(f"Optimizer has {nf} fixed joints but state0.window_fixed_qpos is None")
            io.window_fixed_qpos = chk(state0.window_fixed_qpos, (S, L + 1, nf), torch.float32, "state0.window_fixed_qpos")
        io.window_len = chk(state0.window_len, (S,), torch.int32, "state0.window_len")
        shapes = dict(grad_last_qpos_out=(S, n), grad_window_qpos_out=(S, L + 1, n),
                      grad_window_keypoints_out=(S, L + 1, N.NUM_KEYPOINTS, 3), grad_window_fixed_qpos_out=(S, L + 1, nf))
        for k, shape in shapes.items():
            g = grads.get(k)
            if g is not None and (nf or k != "grad_window_fixed_qpos_out"):
                setattr(io, k, chk(g, shape, torch.float32, k))

        outputs = outputs or {}
        unknown = set(outputs) - {"grad_keypoints", "grad_fixed_qpos", "grad_last_qpos", "grad_window_keypoints",
                                  "grad_window_fixed_qpos", "grad_window_qpos", "status_out"} - (
                                      {"grad_prev_qpos"} if accel else set())
        if unknown:
            raise ValueError(f"outputs: unknown names {sorted(unknown)}")

        def new(shape, name, dtype=torch.float32):
            t = outputs.get(name)
            if t is None:
                t = torch.empty(shape, dtype=dtype, device=dev)
            setattr(io, name, chk(t, shape, dtype, f"outputs[{name!r}]"))
            return t

        g_last = new((S, n), "grad_last_qpos")
        g_wkp = new((S, L + 1, N.NUM_KEYPOINTS, 3), "grad_window_keypoints")
        g_wfix = new((S, L + 1, nf), "grad_window_fixed_qpos") if nf else None
        g_wq = new((S, L + 1, n), "grad_window_qpos")
        fill(io, chk, new)
        nbytes = int(eng.lib.dexr_fixed_lag_accel_vjp_workspace_bytes(eng.handle, S, L) if accel
                     else eng.lib.dexr_fixed_lag_vjp_workspace_bytes(eng.handle, S, L))
        ws = torch.empty((max(nbytes, 4),), dtype=torch.uint8, device=dev)
        io.workspace, io.workspace_bytes = ws.data_ptr(), nbytes
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        p = opt.params(clip_init=True, lp_alpha=self.low_pass_alpha)
        if not accel:
            N.check(eng.lib.dexr_fixed_lag_step_vjp(eng.handle, C.byref(p), C.byref(io), S, K, C.c_void_p(s.cuda_stream)),
                    "dexr_fixed_lag_step_vjp")
            ws.record_stream(s)
            return g_last, g_wkp, g_wfix, g_wq
        if state0.prev_qpos is None or state0.has_prev is None:
            raise ValueError("an accelerated fixed-lag state needs prev_qpos and has_prev")
        acc = N.DexrFixedLagAccelVjp()
        acc.accel_weight = float(state0.accel_weight)
        acc.prev_qpos = chk(state0.prev_qpos, (S, n), torch.float32, "state0.prev_qpos")
        acc.has_prev = chk(state0.has_prev, (S,), torch.int32, "state0.has_prev")
        if grads.get("grad_prev_qpos_out") is not None:
            acc.grad_prev_qpos_out = chk(grads["grad_prev_qpos_out"], (S, n), torch.float32, "grad_prev_qpos_out")
        g_prev = outputs.get("grad_prev_qpos")
        if g_prev is None:
            g_prev = torch.empty((S, n), dtype=torch.float32, device=dev)
        acc.grad_prev_qpos = chk(g_prev, (S, n), torch.float32, "outputs['grad_prev_qpos']")
        N.check(eng.lib.dexr_fixed_lag_step_accel_vjp(eng.handle, C.byref(p), C.byref(io), C.byref(acc), S, K,
                                                      C.c_void_p(s.cuda_stream)), "dexr_fixed_lag_step_accel_vjp")
        ws.record_stream(s)
        return g_last, g_wkp, g_wfix, g_wq, g_prev

    def retarget_fixed_lag_vjp(self, keypoints, tape: FixedLagTape, state0: FixedLagState, *, fixed_qpos=None,
                               grad_qpos=None, grad_robot_qpos=None, grad_last_qpos_out=None, grad_window_qpos_out=None,
                               grad_window_keypoints_out=None, grad_window_fixed_qpos_out=None, smooth_weight=None,
                               stream=None, outputs: Optional[dict] = None):
        """Backpropagation through a recorded `retarget_fixed_lag` call (`dexr_fixed_lag_step_vjp`, one launch): the
        reverse-time VJP of its emitted rows (grad_qpos [S,K,opt_dof], grad_robot_qpos [S,K,dof]) and of the state it left
        (grad_last_qpos_out [S,opt_dof], grad_window_*_out [S,L+1,...]) with respect to its frames and `state0`, the state
        before the call (a copy: the forward updates its state in place).  Each emitting tick's window, and the last
        tick's, is differentiated as `smooth_packed_sequences_vjp` differentiates a clip, at the minimiser the tape holds;
        the anchor cotangent runs back through the committed frames.  Cotangents on PENDING rows are ignored.  Returns
        (grad_keypoints [S,K,21,3], grad_fixed_qpos [S,K,n_fixed] or None, grad_last_qpos [S,opt_dof],
        grad_window_keypoints [S,L+1,21,3], grad_window_fixed_qpos [S,L+1,n_fixed] or None, grad_window_qpos [S,L+1,opt_dof]
        (zero: a warm start), status [S,K] int32 (the emitted frame's window status, STATUS_PENDING elsewhere)).
        Chunks chained through these state cotangents give the same bits as one call.  `outputs`: tensors to write into,
        by their dexr_fixed_lag_vjp_t names (grad_keypoints, ..., status_out).  Nothing is synchronised."""
        import torch

        _refuse_accel_backward(state0, "retarget_fixed_lag_vjp")
        return self._retarget_fixed_lag_vjp(keypoints, tape, state0, fixed_qpos, grad_qpos, grad_robot_qpos,
                                            grad_last_qpos_out, grad_window_qpos_out, grad_window_keypoints_out,
                                            grad_window_fixed_qpos_out, smooth_weight, stream, outputs)

    def _retarget_fixed_lag_vjp(self, keypoints, tape, state0, fixed_qpos, grad_qpos, grad_robot_qpos, grad_last_qpos_out,
                                grad_window_qpos_out, grad_window_keypoints_out, grad_window_fixed_qpos_out, smooth_weight,
                                stream, outputs, accel=False, grad_prev_qpos_out=None):
        """retarget_fixed_lag_vjp, and retarget_fixed_lag_accel_vjp when `accel` (grad_prev_qpos appended)."""
        import torch

        opt = self.optimizer
        if keypoints.dim() != 4 or tuple(keypoints.shape[2:]) != (N.NUM_KEYPOINTS, 3):
            raise ValueError(f"keypoints must have shape [S,K,21,3], got {tuple(keypoints.shape)}")
        S, K, L = int(keypoints.shape[0]), int(keypoints.shape[1]), int(state0.lag)
        n, dof, nf = opt.opt_dof, opt.robot.dof, len(opt.idx_pin2fixed)
        len_proj = opt._objective_spec().len_proj
        res = {}

        def fill(io, chk, new):
            io.keypoints = chk(keypoints, (S, K, N.NUM_KEYPOINTS, 3), torch.float32, "keypoints")
            if nf:
                if fixed_qpos is None:
                    raise ValueError(f"Optimizer has {nf} fixed joints but no fixed_qpos is given")
                io.fixed_qpos = chk(fixed_qpos, (S, K, nf), torch.float32, "fixed_qpos")
            io.tape.qpos = chk(tape.qpos, (S, K, L + 1, n), torch.float32, "tape.qpos")
            if len_proj:
                if tape.projected is None:
                    raise ValueError("DexPilot streams need tape.projected")
                io.tape.projected = chk(tape.projected, (S, K, len_proj), torch.uint8, "tape.projected")
            if grad_qpos is not None:
                io.grad_qpos = chk(grad_qpos, (S, K, n), torch.float32, "grad_qpos")
            if grad_robot_qpos is not None:
                io.grad_robot_qpos = chk(grad_robot_qpos, (S, K, dof), torch.float32, "grad_robot_qpos")
            res["kp"] = new((S, K, N.NUM_KEYPOINTS, 3), "grad_keypoints")
            res["fixed"] = new((S, K, nf), "grad_fixed_qpos") if nf else None
            res["status"] = new((S, K), "status_out", torch.int32)

        grads = dict(grad_last_qpos_out=grad_last_qpos_out, grad_window_qpos_out=grad_window_qpos_out,
                     grad_window_keypoints_out=grad_window_keypoints_out,
                     grad_window_fixed_qpos_out=grad_window_fixed_qpos_out, grad_prev_qpos_out=grad_prev_qpos_out)
        r = self._fixed_lag_vjp_call(state0, K, fill, False, smooth_weight, grads, stream, outputs, accel)
        return (res["kp"], res["fixed"], *r[:4], res["status"], *r[4:])

    def flush_fixed_lag_vjp(self, state0: FixedLagState, *, grad_qpos=None, grad_robot_qpos=None, grad_last_qpos_out=None,
                            grad_window_qpos_out=None, grad_window_keypoints_out=None, grad_window_fixed_qpos_out=None,
                            stream=None):
        """Backpropagation through `flush_fixed_lag` (the K = 0 form of `retarget_fixed_lag_vjp`): the flushed rows
        (grad_qpos [S,L,opt_dof], grad_robot_qpos [S,L,dof]; rows past the count are ignored) are state0's held slots of
        window_qpos, the last of them the new anchor.  Returns (grad_last_qpos, grad_window_keypoints,
        grad_window_fixed_qpos or None, grad_window_qpos) of `state0`, the state before the flush."""
        import torch

        _refuse_accel_backward(state0, "flush_fixed_lag_vjp")
        return self._flush_fixed_lag_vjp(state0, grad_qpos, grad_robot_qpos, grad_last_qpos_out, grad_window_qpos_out,
                                         grad_window_keypoints_out, grad_window_fixed_qpos_out, stream)

    def _flush_fixed_lag_vjp(self, state0, grad_qpos, grad_robot_qpos, grad_last_qpos_out, grad_window_qpos_out,
                             grad_window_keypoints_out, grad_window_fixed_qpos_out, stream, accel=False,
                             grad_prev_qpos_out=None):
        """flush_fixed_lag_vjp, and flush_fixed_lag_accel_vjp when `accel` (grad_prev_qpos appended)."""
        import torch

        opt = self.optimizer
        S, L = int(state0.last_qpos.shape[0]), int(state0.lag)
        n, dof = opt.opt_dof, opt.robot.dof

        def fill(io, chk, new):
            if grad_qpos is not None:
                io.grad_flush_qpos = chk(grad_qpos, (S, L, n), torch.float32, "grad_qpos")
            if grad_robot_qpos is not None:
                io.grad_flush_robot_qpos = chk(grad_robot_qpos, (S, L, dof), torch.float32, "grad_robot_qpos")

        grads = dict(grad_last_qpos_out=grad_last_qpos_out, grad_window_qpos_out=grad_window_qpos_out,
                     grad_window_keypoints_out=grad_window_keypoints_out,
                     grad_window_fixed_qpos_out=grad_window_fixed_qpos_out, grad_prev_qpos_out=grad_prev_qpos_out)
        return self._fixed_lag_vjp_call(state0, 0, fill, True, None, grads, stream, accel=accel)

    @staticmethod
    def _accel_state0(state0: FixedLagState, what: str, tape: Optional[FixedLagTape] = None):
        if not state0.accel_weight:
            raise ValueError(f"{what}: state0 has no acceleration penalty (accel_weight = 0): use "
                             f"{what.replace('_accel', '')}")
        if tape is not None and float(getattr(tape, "accel_weight", 0.0) or 0.0) != float(state0.accel_weight):
            raise ValueError(f"{what}: the tape was recorded for accel_weight = {getattr(tape, 'accel_weight', 0.0)}, "
                             f"state0 has {state0.accel_weight}")

    def retarget_fixed_lag_accel_vjp(self, keypoints, tape: FixedLagTape, state0: FixedLagState, *, fixed_qpos=None,
                                     grad_qpos=None, grad_robot_qpos=None, grad_last_qpos_out=None,
                                     grad_prev_qpos_out=None, grad_window_qpos_out=None, grad_window_keypoints_out=None,
                                     grad_window_fixed_qpos_out=None, smooth_weight=None, stream=None,
                                     outputs: Optional[dict] = None):
        """`retarget_fixed_lag_vjp` for a call on an accelerated state (`dexr_fixed_lag_step_accel_vjp`, one launch;
        DESIGN.md 3.18): `tape` from `make_fixed_lag_tape(S, K, L, accel_weight=c)` with the state's c, `state0` the
        accelerated state before the call.  Each differentiated window is the accel smoother's clip with the pre-anchor
        triple of the forward; the reverse walk carries the cotangents of the last two committed frames.  Also takes
        grad_prev_qpos_out [S,opt_dof], the cotangent of the final prev_qpos.  Returns retarget_fixed_lag_vjp's tuple with
        grad_prev_qpos [S,opt_dof] (of state0.prev_qpos) appended; `outputs` may also name grad_prev_qpos.  The acceleration
        weight and has_prev are not differentiated.  Nothing is synchronised."""
        self._accel_state0(state0, "retarget_fixed_lag_accel_vjp", tape)
        return self._retarget_fixed_lag_vjp(keypoints, tape, state0, fixed_qpos, grad_qpos, grad_robot_qpos,
                                            grad_last_qpos_out, grad_window_qpos_out, grad_window_keypoints_out,
                                            grad_window_fixed_qpos_out, smooth_weight, stream, outputs, True,
                                            grad_prev_qpos_out)

    def flush_fixed_lag_accel_vjp(self, state0: FixedLagState, *, grad_qpos=None, grad_robot_qpos=None,
                                  grad_last_qpos_out=None, grad_prev_qpos_out=None, grad_window_qpos_out=None,
                                  grad_window_keypoints_out=None, grad_window_fixed_qpos_out=None, stream=None):
        """`flush_fixed_lag_vjp` for an accelerated state: also takes grad_prev_qpos_out and returns its tuple with
        grad_prev_qpos (of state0.prev_qpos) appended."""
        self._accel_state0(state0, "flush_fixed_lag_accel_vjp")
        return self._flush_fixed_lag_vjp(state0, grad_qpos, grad_robot_qpos, grad_last_qpos_out, grad_window_qpos_out,
                                         grad_window_keypoints_out, grad_window_fixed_qpos_out, stream, True,
                                         grad_prev_qpos_out)
