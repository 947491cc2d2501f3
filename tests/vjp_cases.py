"""Inputs and the float64 model of the backpropagation-through-the-solve tests (`dexr_solve_vjp`), shared by the host
emulation (tests/test_vjp_emulation.py) and the GPU suite (tests/test_gpu_vjp.py).

The model is the implicit-function theorem at a point x, stated independently of the kernel's formulas:
  * H: the exact Hessian of F = L + norm_delta |x - a|^2, `oracle.solvers._ggn_hessian(obj, x, majoriser=False)`;
  * the active set: the solver's rule (x <= lo and g > -1e-7, or x >= hi and g < 1e-7, at the float32 widened bounds);
  * dg/dtheta by central differences of `FrameObjective.value_and_grad` in theta (keypoints or ref_value, fixed joints,
    anchor), with the DexPilot flags held at the frame's post-solve flags and the targets prepared in float64;
  * theta_bar = -(dg/dtheta)^T v, v_f = H_ff^-1 gbar_f, v = 0 on the active variables.
"""
import numpy as np

import objective_cases as OC
from oracle.objectives import FrameObjective
from oracle.solvers import _ggn_hessian, solve_converged

STATUS_NONFINITE, STATUS_NOT_PD = 1 << 25, 1 << 26
FD_STEP = 1e-6
# frames whose free Hessian has an eigenvalue this close to 0 (relative to the largest) are skipped: whether fp32 finds a pivot
# <= 0 there is a matter of rounding (a joint no residual depends on, without an anchor, has an exactly zero row)
SINGULAR = 1e-6
ZONE_MARGIN = 5e-5  # frames whose Huber distances lie this close to beta are skipped (the central differences would straddle it)

# Emulated / GPU cotangents against the model, in units of the model's |theta_bar|_inf per frame and input.  float32
# kinematics, Hessian and Cholesky against float64.  Worst seen: 2.7e-4 in the host emulation (teleop Shadow vector),
# 3.8e-5 on an H100 (DESIGN.md section 3.8)
TAU = 5e-4


def _prepared(o, ref, flags):
    """float64 targets and weights of `ref` [m,3] with the DexPilot flags held at `flags` (no hysteresis update)."""
    ref = np.asarray(ref, np.float64)
    if o.type == "position":
        return ref, None
    if o.type == "vector":
        return ref * o.scaling, np.ones(o.m)
    len_proj, len_s2 = len(o.projected), len(o.s2_task)
    len_s1 = len_proj - len_s2
    proj = np.asarray(flags, bool)
    w = np.where(proj, np.array([200.0] * len_s1 + [400.0] * len_s2), 1.0)
    w = np.concatenate([w, np.ones(o.num_fingers) * (len_proj + o.num_fingers)])
    dist = np.linalg.norm(ref[:len_proj], axis=1)
    normal = ref * o.scaling
    projv = ref[:len_proj] / (dist[:, None] + 1e-6) * o.projected_dist[:, None]
    tgt = np.concatenate([np.where(proj[:, None], projv, normal[:len_proj]), normal[len_proj:]], axis=0)
    return tgt, w


class _NoAnchor:
    """norm_delta = 0 while a frame without an anchor is modelled."""

    def __init__(self, o, on):
        self.o, self.on, self.nd = o, on, o.norm_delta

    def __enter__(self):
        if self.on:
            self.o.norm_delta = 0.0

    def __exit__(self, *a):
        self.o.norm_delta = self.nd


def _grad(o, x, ref, flags, fixed, last):
    tgt, w = _prepared(o, ref, flags)
    return FrameObjective(o, tgt, w, np.asarray(fixed, float), np.asarray(last, float)).value_and_grad(x)[1]


def near_zone_switch(o, x, ref, flags, fixed):
    """True when a residual's Huber distance (per coordinate for position) lies within ZONE_MARGIN of beta."""
    tgt, w = _prepared(o, ref, flags)
    obj = FrameObjective(o, tgt, w, np.asarray(fixed, float), x)
    pos, _ = obj._kin(np.asarray(x, float), False)
    if o.type == "position":
        d = np.abs(pos - tgt).ravel()
    else:
        d = np.linalg.norm(pos[o.task_sel] - pos[o.origin_sel] - tgt, axis=1)
    return bool(np.any(np.abs(d - o.huber_delta) < ZONE_MARGIN))


def model_vjp(o, x, gbar, fixed, last, flags, ref=None, keypoints=None):
    """float64 VJP of one frame at the float32 point x.  Returns dict(targets [m,3] or [21,3], fixed [n_fixed],
    last [n] or None, not_pd, active [n] bool)."""
    x = np.asarray(x, np.float64)
    gbar = np.asarray(gbar, np.float64)
    no_anchor = last is None
    last_ = x if no_anchor else np.asarray(last, np.float64)
    fixed = np.zeros(0) if fixed is None else np.asarray(fixed, np.float64)
    by_kp = keypoints is not None
    kp = None if keypoints is None else np.asarray(keypoints, np.float64)
    ref = o.ref_from_keypoints(kp) if by_kp else np.asarray(ref, np.float64)
    with _NoAnchor(o, no_anchor):
        tgt, w = _prepared(o, ref, flags)
        obj = FrameObjective(o, tgt, w, fixed, last_)
        g = obj.value_and_grad(x)[1]
        H = _ggn_hessian(obj, x, majoriser=False)
        lo, hi = np.float32(o.lower).astype(np.float64), np.float32(o.upper).astype(np.float64)
        act = ((x <= lo) & (g > -1e-7)) | ((x >= hi) & (g < 1e-7))
        fr = ~act
        v = np.zeros_like(x)
        not_pd = False
        Hff = H[np.ix_(fr, fr)]
        ev = np.linalg.eigvalsh(Hff) if fr.any() else np.ones(1)
        singular = bool(abs(ev[0]) <= SINGULAR * abs(ev).max())
        try:
            Lc = np.linalg.cholesky(Hff)
            v[fr] = np.linalg.solve(Lc.T, np.linalg.solve(Lc, gbar[fr]))
        except np.linalg.LinAlgError:
            not_pd = True

        def cot(theta, grad_of):
            """-(dg/dtheta)^T v over the entries of theta (flat), central differences."""
            out = np.zeros(theta.size)
            if not_pd:
                return out
            flat = theta.ravel()
            for i in range(flat.size):
                tp, tm = flat.copy(), flat.copy()
                tp[i] += FD_STEP
                tm[i] -= FD_STEP
                dg = (grad_of(tp.reshape(theta.shape)) - grad_of(tm.reshape(theta.shape))) / (2 * FD_STEP)
                out[i] = -dg @ v
            return out

        if by_kp:
            used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
            t_bar = np.zeros((21, 3))
            for k in used:
                def gk(p, k=k):
                    kk = kp.copy()
                    kk[k] = p
                    return _grad(o, x, o.ref_from_keypoints(kk), flags, fixed, last_)
                t_bar[k] = cot(kp[k], gk)
        else:
            t_bar = cot(ref, lambda r: _grad(o, x, r, flags, fixed, last_)).reshape(ref.shape)
        f_bar = cot(fixed, lambda fx: _grad(o, x, ref, flags, fx, last_)) if fixed.size else np.zeros(0)
        a_bar = None if no_anchor else cot(last_, lambda a: _grad(o, x, ref, flags, fixed, a))
    return dict(targets=t_bar, fixed=f_bar, last=a_bar, not_pd=not_pd, active=act, singular=singular)


def solved_points(o, n, seed, with_last=True):
    """n frames of OC.oracle_points solved to a KKT point by the float64 oracle (mode B, warm start = anchor or the
    joint-limit middle), rounded to float32, with the DexPilot flags the solve left (from all-false).  Adds
    `qpos` (the rounded minimisers), `flags` (uint8 [n,len_proj] or None) and `gbar` (seeded cotangents)."""
    pts = OC.oracle_points(o, n, seed, with_last=with_last)
    rng = np.random.RandomState(seed + 1)
    nf = len(o.idx_pin2fixed)
    mid = o.joint_limits.mean(1).astype(np.float32)
    X, F = [], []
    for i in range(n):
        if o.type == "dexpilot":
            o.projected[:] = False
        fixed = pts["fixed_qpos"][i] if nf else np.zeros(0, np.float32)
        last = pts["last_qpos"][i] if with_last else mid
        x, _, _ = solve_converged(o, pts["ref_value"][i], fixed, last)
        X.append(x.astype(np.float32))
        if o.type == "dexpilot":
            F.append(o.projected.astype(np.uint8))
    pts["qpos"] = np.array(X)
    pts["flags"] = np.array(F) if F else None
    pts["gbar"] = rng.randn(n, o.opt_dof).astype(np.float32)
    return pts


def model_batch(o, pts, form):
    """model_vjp over the frames of `pts` in input form `form` ("ref_value" / "keypoints"); frames near a Huber zone switch
    and frames with a (nearly) singular free Hessian are marked in `skip`.  Returns dict(targets [B,...], fixed [B,n_fixed], last [B,n] or None, not_pd [B], skip [B],
    n_active)."""
    n = pts["qpos"].shape[0]
    nf = len(o.idx_pin2fixed)
    T, Fx, A, npd, skip, n_act = [], [], [], [], [], 0
    for i in range(n):
        flags = None if pts["flags"] is None else pts["flags"][i]
        fixed = pts["fixed_qpos"][i] if nf else None
        last = None if pts["last_qpos"] is None else pts["last_qpos"][i]
        kw = dict(keypoints=pts["keypoints"][i]) if form == "keypoints" else dict(ref=pts["ref_value"][i])
        m = model_vjp(o, pts["qpos"][i], pts["gbar"][i], fixed, last, flags, **kw)
        T.append(m["targets"])
        Fx.append(m["fixed"])
        A.append(m["last"])
        npd.append(m["not_pd"])
        n_act += int(m["active"].sum())
        skip.append(m["singular"] or near_zone_switch(o, pts["qpos"][i].astype(np.float64), pts["ref_value"][i], flags,
                                                      np.zeros(0) if fixed is None else fixed))
    return dict(targets=np.array(T), fixed=np.array(Fx).reshape(n, nf), last=None if A[0] is None else np.array(A),
                not_pd=np.array(npd), skip=np.array(skip), n_active=n_act)


def errors(got, want, keep):
    """Worst |got - want|_inf / |want|_inf over the kept frames (per frame; frames whose model is exactly 0 need got == 0)."""
    worst = 0.0
    for i in np.flatnonzero(keep):
        a, b = np.asarray(got[i], np.float64).ravel(), np.asarray(want[i], np.float64).ravel()
        scale = np.abs(b).max() if b.size else 0.0
        d = np.abs(a - b).max() if b.size else 0.0
        if scale == 0.0:
            assert d == 0.0, (i, d)
            continue
        worst = max(worst, d / scale)
    return worst


def compare(result, model, pts, tau=TAU):
    """Emulated or GPU outputs (grad_targets, grad_fixed, grad_last, status) against model_batch; asserts tau and the
    status word, returns the worst ratio to tau."""
    g_t, g_f, g_l, status = result
    keep = ~model["skip"]
    np.testing.assert_array_equal(status[keep] & STATUS_NOT_PD != 0, model["not_pd"][keep])
    worst = errors(g_t, model["targets"], keep)
    if g_f is not None and model["fixed"].shape[1]:
        worst = max(worst, errors(g_f, model["fixed"], keep))
    if model["last"] is not None:
        worst = max(worst, errors(g_l, model["last"], keep))
    assert worst <= tau, worst
    return worst / tau
