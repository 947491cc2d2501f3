"""Streams and the float64 model of the backpropagation-through-the-sequence-solve tests (`dexr_solve_sequences_vjp`),
shared by the host emulation (tests/test_seq_vjp_emulation.py) and the GPU suite (tests/test_gpu_seq_vjp.py).

A stream is solved by the float64 oracle (`OracleSeqRetargeting(mode="converged")`: clipped warm start, converged
minimiser rounded to float32, carried solution, mimic, low-pass filter), recording every frame's solution and the DexPilot
flags it left.  The model then runs the reverse-time recurrence of include/dexr.h independently of the kernel:
  gy += dl/dy_t; gq = init_t ? alpha gy : gy; gy = init_t ? (1 - alpha) gy : 0   (no filter: gq = dl/dy_t)
  gbar = M^T gq + c;  frame VJP `vjp_cases.model_vjp` at (x_t, anchor clip(x_{t-1}), flags_t, gbar)
  fixed_bar_t = H-term + gq[fixed];  c = a_bar * [clip_lo <= x_{t-1} <= clip_hi]
with M = dq/dx of the oracle's scatter + mimic (`full_qpos`), the clip at the oracle's joint limits and the filter the
oracle's `OracleLPFilter`.
"""
import numpy as np

import vjp_cases as V
from helpers import keypoint_trajectory
from oracle.solvers import OracleLPFilter, OracleSeqRetargeting

TAU = V.TAU


def stream_inputs(o, S, T, seed, pinch=False):
    """keypoints [S,T,21,3] (consecutive recorded frames with a little noise, wrist at the origin) and fixed joints
    [S,T,n_fixed] inside their limits (or None).  `pinch`: frames 1 and 2 of every stream bring the index tip within 2 cm of
    the thumb tip (DexPilot flags switch on, then off again at frame 3)."""
    rng = np.random.RandomState(seed)
    traj = keypoint_trajectory().astype(np.float32)
    kp = np.zeros((S, T, 21, 3), np.float32)
    for s in range(S):
        start = rng.randint(0, len(traj) - 3 * T)
        kp[s] = traj[start:start + 3 * T:3] + (rng.randn(T, 1, 3) * 0.002).astype(np.float32)
    kp[:, :, 0] = 0
    if pinch:
        for t in (1, 2):
            if t < T:
                d = kp[:, t, 8] - kp[:, t, 4]
                kp[:, t, 8] = kp[:, t, 4] + 0.02 * d / np.linalg.norm(d, axis=-1, keepdims=True)
    nf = len(o.idx_pin2fixed)
    fixed = None
    if nf:
        lim = o.robot.joint_limits[o.idx_pin2fixed]
        fixed = rng.uniform(lim[:, 0], lim[:, 1], size=(S, T, nf)).astype(np.float32)
    return kp, fixed


def oracle_stream(o, kp, fixed, last0, filter_state0, filter_init0, flags0=None):
    """One stream through OracleSeqRetargeting(mode="converged") from the given state.  Returns dict(qpos [T,n] float32,
    flags [T,len_proj] uint8 or None, robot_qpos [T,dof] float64, last, filter_state)."""
    T = kp.shape[0]
    seq = OracleSeqRetargeting(o, mode="converged")
    seq.last_qpos = np.asarray(last0, np.float32).copy()
    if seq.filter is not None:
        seq.filter.y, seq.filter.is_init = np.asarray(filter_state0, np.float64).copy(), bool(filter_init0)
    if o.type == "dexpilot":
        o.projected[:] = False if flags0 is None else np.asarray(flags0, bool)
    X, F, Y = [], [], []
    for t in range(T):
        Y.append(seq.retarget(o.ref_from_keypoints(kp[t]), np.zeros(0) if fixed is None else fixed[t]))
        X.append(np.asarray(seq.last_qpos, np.float32))
        if o.type == "dexpilot":
            F.append(o.projected.astype(np.uint8))
    return dict(qpos=np.array(X), flags=np.array(F) if F else None, robot_qpos=np.array(Y), last=X[-1],
                filter_state=None if seq.filter is None else seq.filter.y.copy())


def oracle_streams(o, kp, fixed, last0, filter_state0, filter_init0):
    """oracle_stream over S streams, stacked."""
    S = kp.shape[0]
    r = [oracle_stream(o, kp[s], None if fixed is None else fixed[s], last0[s], filter_state0[s], filter_init0[s])
         for s in range(S)]
    return dict(qpos=np.stack([x["qpos"] for x in r]), flags=None if r[0]["flags"] is None else np.stack([x["flags"] for x in r]),
                robot_qpos=np.stack([x["robot_qpos"] for x in r]))


def scatter_jacobians(o):
    """dq/dx [dof,n] and dq/dfixed [dof,n_fixed] of the oracle's scatter + mimic (affine, so exact from unit vectors)."""
    n, nf = o.opt_dof, len(o.idx_pin2fixed)
    q0 = o.full_qpos(np.zeros(n), np.zeros(nf))
    M = np.stack([o.full_qpos(np.eye(n)[j], np.zeros(nf)) - q0 for j in range(n)], axis=1)
    Mf = np.stack([o.full_qpos(np.zeros(n), np.eye(nf)[k]) - q0 for k in range(nf)], axis=1) if nf else np.zeros((len(q0), 0))
    return M, Mf


def model_stream(o, kp, fixed, last0, filter_init0, X, F, g_out=None, g_last=None, g_filter=None):
    """float64 reverse-time recurrence of one stream (module docstring).  Returns dict(keypoints [T,21,3], fixed [T,n_fixed],
    last [n], filter [dof], not_pd [T], skip [T]): `skip` marks frames whose model is ill-conditioned (vjp_cases rules) and,
    because the anchor chain carries their error backwards, every frame before them."""
    T, n = X.shape
    dof = o.robot.dof
    a = o.low_pass_alpha
    use_filter = 0 <= a <= 1
    M, Mf = scatter_jacobians(o)
    lo, hi = np.float32(o.joint_limits[:, 0]).astype(np.float64), np.float32(o.joint_limits[:, 1]).astype(np.float64)
    gy = np.zeros(dof) if g_filter is None else np.asarray(g_filter, np.float64).copy()
    c = np.zeros(n) if g_last is None else np.asarray(g_last, np.float64).copy()
    g_out = np.zeros((T, dof)) if g_out is None else np.asarray(g_out, np.float64)
    kp_bar, fx_bar = np.zeros((T, 21, 3)), np.zeros((T, Mf.shape[1]))
    not_pd, skip = np.zeros(T, bool), np.zeros(T, bool)
    filt = OracleLPFilter(a) if use_filter else None
    for t in range(T - 1, -1, -1):
        if use_filter:
            gy = gy + g_out[t]
            init = t > 0 or bool(filter_init0)
            gq = filt.alpha * gy if init else gy
            gy = (1 - filt.alpha) * gy if init else np.zeros(dof)
        else:
            gq = g_out[t]
        gbar = M.T @ gq + c
        xp = np.asarray(X[t - 1] if t > 0 else last0, np.float64)
        anchor = np.clip(xp, lo, hi)
        fx = np.zeros(0) if fixed is None else fixed[t]
        flags = None if F is None else F[t]
        m = V.model_vjp(o, X[t], gbar, fx, anchor, flags, keypoints=kp[t])
        kp_bar[t], not_pd[t] = m["targets"], m["not_pd"]
        fx_bar[t] = m["fixed"] + Mf.T @ gq
        c = m["last"] * ((xp >= lo) & (xp <= hi))
        skip[t] = m["singular"] or V.near_zone_switch(o, X[t].astype(np.float64), o.ref_from_keypoints(kp[t]), flags, fx)
    skip = np.maximum.accumulate(skip[::-1])[::-1]  # frame t's error reaches every earlier frame through c
    return dict(keypoints=kp_bar, fixed=fx_bar, last=c, filter=gy if use_filter else (np.zeros(dof) if g_filter is None else
                                                                                       np.asarray(g_filter, np.float64)),
                not_pd=not_pd, skip=skip)


def compare_stream(got, model, tau=TAU):
    """One stream's emulated or GPU cotangents (grad_keypoints [T,21,3], grad_fixed [T,n_fixed] or None, grad_last [n],
    grad_filter [dof], status [T]) against model_stream, per frame and per input in units of the model's largest entry.
    Returns the worst ratio to tau."""
    g_kp, g_fx, g_last, g_filter, status = got
    keep = ~model["skip"]
    np.testing.assert_array_equal((status[keep] & V.STATUS_NOT_PD) != 0, model["not_pd"][keep])
    worst = V.errors(g_kp, model["keypoints"], keep)
    if g_fx is not None and model["fixed"].shape[1]:
        worst = max(worst, V.errors(g_fx, model["fixed"], keep))
    if keep[0]:
        worst = max(worst, V.errors(g_last[None], model["last"][None], [True]))
    worst = max(worst, V.errors(g_filter[None], model["filter"][None], [True]))
    assert worst <= tau, worst
    return worst / tau
