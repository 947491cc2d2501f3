"""The float64 model of the per-frame Jacobian tests (`dexr_solve_jacobian`), shared by the host emulation
(tests/test_jacobian_emulation.py) and the GPU suite (tests/test_gpu_jacobian.py).

J = dx*/dtheta = -H_ff^-1 dg_f/dtheta at a point x, built from the pieces of the VJP model (tests/vjp_cases.py): its
prepared targets with the DexPilot flags held, its gradient, its no-anchor switch, the exact Hessian
`_ggn_hessian(majoriser=False)`, the solver's active-set rule and the SINGULAR / ZONE_MARGIN skip rules.  dg/dtheta is one
matrix of central differences per input (keypoints or ref_value, fixed joints, anchor) instead of one cotangent per call.
"""
import numpy as np

import vjp_cases as V
from oracle.objectives import FrameObjective

TAU = V.TAU  # in units of the model block's |.|_inf, per frame and block


def _dg(theta, grad_of):
    """dg/dtheta [n, theta.size] by central differences (V.FD_STEP) over the flat entries of theta."""
    flat = np.asarray(theta, np.float64).ravel()
    cols = []
    for i in range(flat.size):
        tp, tm = flat.copy(), flat.copy()
        tp[i] += V.FD_STEP
        tm[i] -= V.FD_STEP
        cols.append((grad_of(tp.reshape(np.shape(theta))) - grad_of(tm.reshape(np.shape(theta)))) / (2 * V.FD_STEP))
    return np.stack(cols, axis=1) if cols else np.zeros((0, 0))


def model_jacobian(o, x, fixed, last, flags, ref=None, keypoints=None):
    """float64 Jacobian of one frame at the float32 point x.  Returns dict(targets [n,m,3] or [n,21,3], fixed [n,n_fixed],
    last [n,n] or None, not_pd, active [n] bool, singular)."""
    x = np.asarray(x, np.float64)
    n = x.size
    no_anchor = last is None
    last_ = x if no_anchor else np.asarray(last, np.float64)
    fixed = np.zeros(0) if fixed is None else np.asarray(fixed, np.float64)
    by_kp = keypoints is not None
    kp = None if keypoints is None else np.asarray(keypoints, np.float64)
    ref = o.ref_from_keypoints(kp) if by_kp else np.asarray(ref, np.float64)
    with V._NoAnchor(o, no_anchor):
        tgt, w = V._prepared(o, ref, flags)
        obj = FrameObjective(o, tgt, w, fixed, last_)
        g = obj.value_and_grad(x)[1]
        H = V._ggn_hessian(obj, x, majoriser=False)
        # the solver's active-set rule at the float32 widened bounds, as in V.model_vjp
        lo, hi = np.float32(o.lower).astype(np.float64), np.float32(o.upper).astype(np.float64)
        act = ((x <= lo) & (g > -1e-7)) | ((x >= hi) & (g < 1e-7))
        fr = ~act
        Hff = H[np.ix_(fr, fr)]
        ev = np.linalg.eigvalsh(Hff) if fr.any() else np.ones(1)
        singular = bool(abs(ev[0]) <= V.SINGULAR * abs(ev).max())
        P = np.zeros((n, n))  # H_ff^-1, zero rows and columns on the active variables
        not_pd = False
        try:
            Lc = np.linalg.cholesky(Hff)
            P[np.ix_(fr, fr)] = np.linalg.solve(Lc.T, np.linalg.solve(Lc, np.eye(int(fr.sum()))))
        except np.linalg.LinAlgError:
            not_pd = True

        def jac(theta, grad_of):
            if not_pd or np.size(theta) == 0:
                return np.zeros((n, np.size(theta)))
            return -P @ _dg(theta, grad_of)

        if by_kp:
            used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
            j_t = np.zeros((n, 21, 3))
            for k in used:
                def gk(p, k=k):
                    kk = kp.copy()
                    kk[k] = p
                    return V._grad(o, x, o.ref_from_keypoints(kk), flags, fixed, last_)
                j_t[:, k] = jac(kp[k], gk)
        else:
            j_t = jac(ref, lambda r: V._grad(o, x, r, flags, fixed, last_)).reshape((n,) + ref.shape)
        j_f = jac(fixed, lambda fx: V._grad(o, x, ref, flags, fx, last_))
        j_a = None if no_anchor else jac(last_, lambda a: V._grad(o, x, ref, flags, fixed, a))
    return dict(targets=j_t, fixed=j_f, last=j_a, not_pd=not_pd, active=act, singular=singular)


def model_batch(o, pts, form):
    """model_jacobian over the frames of `pts` (as from V.solved_points) in input form `form` ("ref_value" / "keypoints");
    frames near a Huber zone switch and frames with a (nearly) singular free Hessian are marked in `skip`.  Returns
    dict(targets [B,n,...], fixed [B,n,n_fixed], last [B,n,n] or None, not_pd [B], skip [B], active [B,n])."""
    B = pts["qpos"].shape[0]
    nf = len(o.idx_pin2fixed)
    T, Fx, A, npd, skip, act = [], [], [], [], [], []
    for i in range(B):
        flags = None if pts["flags"] is None else pts["flags"][i]
        fixed = pts["fixed_qpos"][i] if nf else None
        last = None if pts["last_qpos"] is None else pts["last_qpos"][i]
        kw = dict(keypoints=pts["keypoints"][i]) if form == "keypoints" else dict(ref=pts["ref_value"][i])
        m = model_jacobian(o, pts["qpos"][i], fixed, last, flags, **kw)
        T.append(m["targets"])
        Fx.append(m["fixed"])
        A.append(m["last"])
        npd.append(m["not_pd"])
        act.append(m["active"])
        skip.append(m["singular"] or V.near_zone_switch(o, pts["qpos"][i].astype(np.float64), pts["ref_value"][i], flags,
                                                        np.zeros(0) if fixed is None else fixed))
    n = o.opt_dof
    return dict(targets=np.array(T), fixed=np.array(Fx).reshape(B, n, nf), last=None if A[0] is None else np.array(A),
                not_pd=np.array(npd), skip=np.array(skip), active=np.array(act))


def compare(result, model, tau=TAU):
    """Emulated or GPU Jacobians (jac_targets, jac_fixed, jac_last, status) against model_batch, per frame and block in units
    of the model block's |.|_inf; asserts tau and the status word, returns the worst ratio to tau."""
    j_t, j_f, j_l, status = result
    keep = ~model["skip"]
    np.testing.assert_array_equal(status[keep] & V.STATUS_NOT_PD != 0, model["not_pd"][keep])
    worst = V.errors(j_t, model["targets"], keep)
    if j_f is not None and model["fixed"].shape[2]:
        worst = max(worst, V.errors(j_f, model["fixed"], keep))
    if model["last"] is not None:
        worst = max(worst, V.errors(j_l, model["last"], keep))
    assert worst <= tau, worst
    return worst / tau
