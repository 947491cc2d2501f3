"""The float64 model of the backpropagation through the offline smoother (`dexr_smooth_sequences_packed_vjp`), shared by
the host emulation (tests/test_smooth_vjp_emulation.py), the GPU suite (tests/test_gpu_smooth_vjp.py) and
tools/bench_smooth_vjp.py.

The model is the implicit-function theorem for one stream, stated independently of the kernel's formulas, on
`smooth_cases.Model` (the oracle's per-frame loss with the DexPilot flags held at the causal tape's):
  * G_t = grad_qpos_t + M^T grad_robot_qpos_t, M = d robot_qpos / d x of the oracle's `full_qpos` (affine);
  * the active set: the smoother's rule on the total gradient at X* (x <= lo and g > -1e-7, or x >= hi and g < 1e-7, at the
    float32 widened bounds);
  * H: the stacked Hessian of F over all free variables of the clip, dense: the exact per-frame Hessians of
    `oracle.solvers._ggn_hessian` (zero on a missing frame) + 2 w k_t I on the diagonal, -2 w I beside it; V = H_ff^-1 G_f
    by a dense Cholesky (so only small T);
  * theta_bar_t = -(dg_t/dtheta_t)^T v_t by central differences of the oracle gradient (`vjp_cases._grad`, flags held),
    plus the direct term d robot_qpos / d fixed of the fixed joints, and a_bar = 2 w v_0 where the clip passes the anchor.
Skip rules are those of `vjp_cases` (a nearly singular free Hessian, a frame near a Huber zone switch), applied per stream:
the solve couples every frame of it.  Errors are measured against the model's largest entry per stream and input, since the
cotangents decay along the clip.
"""
import numpy as np

import vjp_cases as V

STATUS_NONFINITE, STATUS_NOT_PD, STATUS_MISSING = 1 << 25, 1 << 26, 1 << 27
# Emulated / GPU cotangents against the model, in units of the model's largest entry per stream and input: twice the
# single-frame VJP's tau.  The stacked solve eliminates up to 60 coupled frames in fp32, and on a 20-60-frame Shadow
# position clip an H100 gave 7.5e-4 (1.5 x vjp_cases.TAU); the packaged 16-lane hands and the structure cases stay below
# 0.1 x vjp_cases.TAU (DESIGN.md section 3.13)
TAU = 2 * V.TAU


def maps(o):
    """M = d robot_qpos / d x [dof,n] and d robot_qpos / d fixed [dof,n_fixed] of the oracle's full_qpos (affine)."""
    n, nf = o.opt_dof, len(o.idx_pin2fixed)
    x0, f0 = np.zeros(n), np.zeros(nf)
    base = np.asarray(o.full_qpos(x0, f0), np.float64)
    Mx = np.stack([np.asarray(o.full_qpos(np.eye(n)[i], f0), np.float64) - base for i in range(n)], axis=1)
    Mf = (np.stack([np.asarray(o.full_qpos(x0, np.eye(nf)[i]), np.float64) - base for i in range(nf)], axis=1)
          if nf else np.zeros((base.size, 0)))
    return Mx, Mf


def model_stream(m, X, keypoints, fixed, flags, anchor_raw, grad_qpos=None, grad_robot_qpos=None):
    """The VJP of one stream at the float32 answer X [T,n].  `m`: its smooth_cases.Model; keypoints [T,21,3], fixed
    [T,n_fixed] or None, flags [T,len_proj] or None, anchor_raw [n] (the unclipped last_qpos) or None, grad_qpos [T,n] /
    grad_robot_qpos [T,dof] or None.  Returns dict(keypoints [T,21,3], fixed [T,n_fixed], last [n] or None, not_pd, skip,
    n_active, V [T,n])."""
    o, T, n, w = m.o, m.T, m.n, m.w
    nf = len(o.idx_pin2fixed)
    X = np.asarray(X, np.float64)
    Mx, Mf = maps(o)
    Gb = np.zeros((T, n))
    direct = np.zeros((T, nf))
    if grad_qpos is not None:
        Gb += np.asarray(grad_qpos, np.float64)
    if grad_robot_qpos is not None:
        grq = np.asarray(grad_robot_qpos, np.float64)
        Gb += grq @ Mx
        direct = grq @ Mf
    fr = [m._frame(t, X[t], True) for t in range(T)]
    g = np.array([r[1] for r in fr]) + m.smooth_grad(X)
    act = ((X <= m.lo) & (g > -1e-7)) | ((X >= m.hi) & (g < 1e-7))
    H = np.zeros((T * n, T * n))
    for t in range(T):
        k = (t > 0 or m.anchor is not None) + (t + 1 < T)
        H[t * n:(t + 1) * n, t * n:(t + 1) * n] = fr[t][2] + 2 * w * k * np.eye(n)
        if t + 1 < T:
            H[t * n:(t + 1) * n, (t + 1) * n:(t + 2) * n] = -2 * w * np.eye(n)
            H[(t + 1) * n:(t + 2) * n, t * n:(t + 1) * n] = -2 * w * np.eye(n)
    free = ~act.ravel()
    Hff = H[np.ix_(free, free)]
    Hff = 0.5 * (Hff + Hff.T)
    ev = np.linalg.eigvalsh(Hff) if free.any() else np.ones(1)
    singular = bool(abs(ev[0]) <= V.SINGULAR * abs(ev).max())
    Vv = np.zeros(T * n)
    not_pd = False
    try:
        L = np.linalg.cholesky(Hff)
        Vv[free] = np.linalg.solve(L.T, np.linalg.solve(L, Gb.ravel()[free]))
    except np.linalg.LinAlgError:
        not_pd = True
    Vm = Vv.reshape(T, n)
    kp_bar = np.zeros((T, 21, 3))
    f_bar = np.zeros((T, nf))
    near = False
    used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
    for t in range(T):
        if m.missing[t]:
            continue
        fl = None if flags is None else flags[t]
        fx = np.zeros(0) if not nf else np.asarray(fixed[t], np.float64)
        kp = np.asarray(keypoints[t], np.float64)
        near = near or V.near_zone_switch(o, X[t], o.ref_from_keypoints(kp), fl, fx)
        if not_pd:
            continue
        v = Vm[t]
        with V._NoAnchor(o, True):
            def cot(theta, grad_of):
                out = np.zeros(theta.size)
                flat = theta.ravel()
                for i in range(flat.size):
                    tp, tm = flat.copy(), flat.copy()
                    tp[i] += V.FD_STEP
                    tm[i] -= V.FD_STEP
                    dg = (grad_of(tp.reshape(theta.shape)) - grad_of(tm.reshape(theta.shape))) / (2 * V.FD_STEP)
                    out[i] = -dg @ v
                return out

            for k in used:
                def gk(p, k=k):
                    kk = kp.copy()
                    kk[k] = p
                    return V._grad(o, X[t], o.ref_from_keypoints(kk), fl, fx, X[t])
                kp_bar[t, k] = cot(kp[k], gk)
            if nf:
                f_bar[t] = cot(fx, lambda f: V._grad(o, X[t], o.ref_from_keypoints(kp), fl, f, X[t]))
        f_bar[t] += direct[t]
    a_bar = None
    if anchor_raw is not None:
        lim = o.joint_limits
        ar = np.asarray(anchor_raw, np.float32)
        passes = (ar >= np.float32(lim[:, 0])) & (ar <= np.float32(lim[:, 1]))
        a_bar = 0.0 if not_pd else 2 * w * Vm[0] * passes
        a_bar = np.zeros(n) if not_pd else a_bar
    return dict(keypoints=kp_bar, fixed=f_bar, last=a_bar, not_pd=not_pd, skip=singular or near, n_active=int(act.sum()),
                V=Vm)


def stream_errors(got, want):
    """|got - want|_inf / |want|_inf over one stream's block of one input (a block whose model is exactly 0 needs got == 0)."""
    a, b = np.asarray(got, np.float64).ravel(), np.asarray(want, np.float64).ravel()
    if b.size == 0:
        return 0.0
    scale, d = np.abs(b).max(), np.abs(a - b).max()
    if scale == 0.0:
        assert d == 0.0, d
        return 0.0
    return d / scale


def compare(result, models, offsets, tau=TAU):
    """Emulated or GPU outputs (grad_keypoints [N,21,3], grad_fixed [N,n_fixed], grad_last [S,n] or None, status [N])
    against a model_stream per stream (None: not checked); asserts tau per stream and input and the NOT_PD verdicts of
    the kept streams.  Returns (worst ratio to tau, number of streams compared)."""
    g_kp, g_f, g_l, status = result
    worst, checked = 0.0, 0
    for s, md in enumerate(models):
        if md is None or md["skip"]:
            continue
        a, b = int(offsets[s]), int(offsets[s + 1])
        assert bool((status[a:b] & STATUS_NOT_PD != 0).all()) == md["not_pd"], (s, md["not_pd"])
        e = stream_errors(g_kp[a:b], md["keypoints"])
        if md["fixed"].size:
            e = max(e, stream_errors(g_f[a:b], md["fixed"]))
        if md["last"] is not None and g_l is not None:
            e = max(e, stream_errors(g_l[s], md["last"]))
        assert e <= tau, (s, e)
        worst = max(worst, e)
        checked += 1
    return worst / tau, checked
