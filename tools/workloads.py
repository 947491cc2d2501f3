"""Synthetic workloads of the BASELINE.json configurations (SURVEY.md section 8d), generated on the HOST with seeded numpy so
that bench.py, the parity fixtures (tests/tools/gen_bench_parity.py) and the GPU tests see bit-identical frames on any box.

Everything here is input generation: float64 FK of the packaged kinematic model (dex_retargeting_b200.urdf.KinematicModel) to
place reachable targets, then float32 keypoint frames and warm starts.  No solver, no oracle.

  metric / config 2   Vector Allegro right (teleop YAML): q* ~ U(limits), wrist + tips written at the human keypoint ids divided
                      by the scaling, warm start q* + sigma N(0,1) clipped (sigma 0.05 warm / 0.5 cold, tests/test_optimizer.py:28-42)
  real trajectory     the 621 recorded frames (example/profiling/human_joint_right.pkl) tiled with 2 mm per-copy offsets, started
                      from the mid-range pose (SeqRetargeting's initial last_qpos, seq_retarget.py:33-35)
  config 3            Position Shadow right, offline YAML (24 + 6 dummy joints = 30), targets at the 10 position links; dummy joint
                      range as shipped (+-5 m, +-2 pi) or narrowed (+-0.5 m, +-pi)
  config 4            DexPilot LEAP right streams: the first T recorded frames with a 2 mm per-stream offset (keeps the thumb-finger
                      distances crossing the 0.03 / 0.05 m hysteresis band as the recording does)
  config 5            {Allegro, Shadow, LEAP, Ability, SVH, Inspire} right, teleop vector YAMLs, frames as in config 2
"""
from __future__ import annotations

import hashlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
TRAJECTORY = ROOT / "tests" / "golden" / "human_joint_right.npy"

METRIC_KEY = "teleop/allegro_hand_right"
SHADOW_POS_KEY = "offline/shadow_hand_right"
LEAP_DEXPILOT_KEY = "teleop/leap_hand_right_dexpilot"
MIXED_KEYS = ["teleop/allegro_hand_right", "teleop/shadow_hand_right", "teleop/leap_hand_right", "teleop/ability_hand_right",
              "teleop/schunk_svh_hand_right", "teleop/inspire_hand_right"]
METRIC_SEED = 1234          # + rank (weak scaling: every rank its own frames)
SHADOW_SEED = 100
STREAM_SEED = 7
MIXED_SEED = 300


def build(key, device=None, override=None):
    """SeqRetargeting from the packaged YAML + packaged URDF (the product's own loader; no test helpers)."""
    from dex_retargeting_b200.constants import config_root
    from dex_retargeting_b200.retargeting_config import RetargetingConfig

    RetargetingConfig.set_default_urdf_dir(str(RetargetingConfig.packaged_urdf_dir()))
    return RetargetingConfig.load_from_file(config_root() / (key + ".yml"), override).build(device=device)


def keypoint_spec(opt):
    """(link names, human keypoint ids, scale, centre) that turn link positions into a keypoint frame for this optimizer."""
    hi = np.asarray(opt.target_link_human_indices)
    if opt.retargeting_type == "POSITION":
        return list(opt.body_names), [int(v) for v in hi.reshape(-1)], 1.0, False
    names = list(opt.origin_link_names[:1]) + list(opt.task_link_names)
    human = [int(hi[0, 0])] + [int(v) for v in hi[1]]
    return names, human, float(opt.scaling), True


def batched_fk(kin, q):
    """World rotation / origin of every movable joint frame, float64, batched over the leading axis of q [n, dof]."""
    n, dof = q.shape
    Rw = np.zeros((n, dof, 3, 3))
    pw = np.zeros((n, dof, 3))
    for i in range(dof):
        a = kin.joint_axis[i]
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        Rq = np.eye(3)[None] + np.sin(q[:, i])[:, None, None] * K[None] + (1 - np.cos(q[:, i]))[:, None, None] * (K @ K)[None]
        par = kin.joint_parent[i]
        if par >= 0:
            Rb = Rw[:, par] @ kin.joint_R[i]
            pb = np.einsum("bij,j->bi", Rw[:, par], kin.joint_p[i]) + pw[:, par]
        else:
            Rb = np.broadcast_to(kin.joint_R[i], (n, 3, 3))
            pb = np.broadcast_to(kin.joint_p[i], (n, 3))
        if kin.joint_type[i] == 0:
            Rw[:, i] = Rb @ Rq
            pw[:, i] = pb
        else:  # prismatic
            Rw[:, i] = Rb
            pw[:, i] = pb + np.einsum("bij,j->bi", Rb, a) * q[:, i:i + 1]
    return Rw, pw


def link_positions(kin, Rw, pw, name):
    li = kin.link_index(name)
    par = kin.link_parent[li]
    if par >= 0:
        return np.einsum("bij,j->bi", Rw[:, par], kin.link_p[li]) + pw[:, par]
    return np.broadcast_to(kin.link_p[li], (Rw.shape[0], 3))


def make_batch(kin, spec, n, seed, centre=True, sigma=0.05, limits=None):
    """n reachable keypoint frames [n,21,3] f32 and warm starts [n,dof] f32 (pinocchio order, all DoFs)."""
    rng = np.random.RandomState(seed)
    lim = kin.joint_limits if limits is None else limits
    dof = kin.dof
    q = rng.uniform(lim[:, 0], lim[:, 1], size=(n, dof))
    init = np.clip(q + sigma * rng.randn(n, dof), lim[:, 0], lim[:, 1]).astype(np.float32)
    Rw, pw = batched_fk(kin, q)
    kp = np.zeros((n, 21, 3), dtype=np.float32)
    names, human, scale = spec[:3]
    for name, h in zip(names, human):
        kp[:, h] = (link_positions(kin, Rw, pw, name) / scale).astype(np.float32)
    if centre:  # the wrist is the origin of the keypoint frame, like a wrist-centred detector output
        kp -= kp[:, 0:1].copy()
    return kp, init


def frames(seq, n, seed, sigma=0.05, narrow_dummy=False):
    """(keypoints [n,21,3], last_qpos [n,opt_dof], fixed_qpos [n,k] or None, info) for an independent-frames launch."""
    opt = seq.optimizer
    kin = opt.robot.kin
    names, human, scale, centre = keypoint_spec(opt)
    lim = kin.joint_limits.copy()
    has_dummy = False
    for i, nm in enumerate(kin.dof_joint_names):
        if "dummy" in nm:
            has_dummy = True
            if narrow_dummy:  # +-0.5 m / +-pi instead of the shipped +-5 m / +-2 pi (yourdfpy.py:1945-1946)
                lim[i] = [-0.5, 0.5] if "translation" in nm else [-np.pi, np.pi]
    if opt.adaptor is not None:  # mimic joints follow their sources in the generating pose as well
        pass
    kp, init = make_batch(kin, (names, human, scale), n, seed, centre=centre, sigma=sigma, limits=lim)
    x0 = np.ascontiguousarray(init[:, opt.idx_pin2target])
    fixed = np.ascontiguousarray(init[:, opt.idx_pin2fixed]) if len(opt.idx_pin2fixed) else None
    return kp, x0, fixed, dict(dummy_joints=has_dummy, dummy_range="narrowed +-0.5 m / +-pi" if (has_dummy and narrow_dummy) else
                               ("shipped +-5 m / +-2 pi" if has_dummy else None))


def real_frames(seq, n, seed=11):
    """The recorded trajectory tiled to n frames with 2 mm per-copy offsets; warm start = mid-range pose for every frame."""
    traj = np.load(TRAJECTORY).astype(np.float32)
    rng = np.random.RandomState(seed)
    reps = (n + len(traj) - 1) // len(traj)
    kp = np.concatenate([traj + (rng.randn(1, 21, 3) * 0.002).astype(np.float32) for _ in range(reps)])[:n].copy()
    kp[:, 0] = 0
    x0 = np.tile(seq.joint_limits.mean(1).astype(np.float32), (n, 1))
    return np.ascontiguousarray(kp), x0


def streams(S, T, seed=STREAM_SEED):
    """[S,T,21,3] f32: the first T recorded frames, every stream with its own 2 mm keypoint offsets (wrist kept at 0)."""
    base = np.load(TRAJECTORY)[:T].astype(np.float32)
    rng = np.random.RandomState(seed)
    kp = base[None] + rng.randn(S, 1, 21, 3).astype(np.float32) * 0.002
    kp[:, :, 0] = 0
    return np.ascontiguousarray(kp)


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        if a is not None:
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:16]


def ragged_streams(S, lo=60, hi=300, seed=STREAM_SEED):
    """(keypoints [N,21,3] f32 packed end to end, lengths [S] int64): stream s is the first lengths[s] recorded frames with
    its own 2 mm keypoint offsets (wrist kept at 0), as in `streams`; lengths are seeded, uniform over [lo, hi]."""
    traj = np.load(TRAJECTORY).astype(np.float32)
    rng = np.random.RandomState(seed)
    lengths = rng.randint(lo, hi + 1, size=S).astype(np.int64)
    offs = rng.randn(S, 1, 21, 3).astype(np.float32) * 0.002
    kp = np.concatenate([traj[:n] + offs[s] for s, n in enumerate(lengths)]) if S else np.zeros((0, 21, 3), np.float32)
    kp[:, 0] = 0
    return np.ascontiguousarray(kp), lengths
