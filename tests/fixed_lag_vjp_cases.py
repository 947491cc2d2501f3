"""The float64 model of the backpropagation through fixed-lag smoothing (`dexr_fixed_lag_step_vjp`), shared by the host
emulation (tests/test_fixed_lag_vjp_emulation.py) and the GPU suite (tests/test_gpu_fixed_lag_vjp.py).

One stream from a fresh state (no held frames), K ticks of lag L, no flush, a loss on the emitted rows only.  Tick k solves
the window of frames c_k .. k (c_k = max(0, k - L)) anchored at the initial anchor when c_k = 0 and at the frame tick k - 1
committed otherwise; it emits (and commits) slot 0 once the window holds L + 1 frames.  The model is stated from the
recurrence, independently of the kernel's bookkeeping: walking the ticks backwards, each emitting window is an offline
smoother clip whose VJP is `smooth_vjp_cases.model_stream` (the implicit-function theorem on the stacked Hessian of
`smooth_cases.Model`), with the emitted row's cotangent plus the carried anchor cotangent on its slot 0; the window's
anchor cotangent feeds slot 0 of the previous tick's window (c_k >= 1) or the initial anchor (c_k = 0).  Every frame uses
the DexPilot flags of the causal walk (the committed flags follow it, tests/test_fixed_lag_emulation.py).

`polished_chain` is the forward in float64: each window re-polished by `smooth_cases.Model.polish`, tick by tick, anchored
at the previous re-polished commit -- the function whose central differences check the model."""
import numpy as np

import smooth_cases as SMC
import smooth_vjp_cases as SVC

TAU = SVC.TAU


def window(k, L):
    """(c_k, m_k): the first frame and the length of tick k's window (fresh state)."""
    c = max(0, k - L)
    return c, k + 1 - c


def clip_anchor(o, a):
    lim = o.joint_limits
    return np.clip(np.asarray(a, np.float64), np.float32(lim[:, 0]).astype(np.float64), np.float32(lim[:, 1]).astype(np.float64))


def model_chain(o, w, kp, fx, flags, a0, Xs, L, gq, grq):
    """The VJP of one stream's K ticks at the window points Xs (a list: Xs[k] [m_k, n], float32 or float64).  kp [K,21,3],
    fx [K,n_fixed] or None, flags [K,len_proj] (the flags each frame uses) or None, a0 [n] the raw initial anchor, gq [K,n],
    grq [K,dof] (rows of non-emitting ticks are not read).  Returns dict(keypoints [K,21,3], fixed [K,n_fixed], last [n],
    skip, not_pd (the emitting ticks whose window is NOT_PD))."""
    K, n = kp.shape[0], o.opt_dof
    nf = len(o.idx_pin2fixed)
    g_kp, g_f, g_last = np.zeros((K, 21, 3)), np.zeros((K, nf)), np.zeros(n)
    abar = np.zeros(n)
    skip, not_pd = False, []
    for k in range(K - 1, -1, -1):
        c, m = window(k, L)
        if m < L + 1:
            continue  # (a pending window carries no loss: only the emitted rows have cotangents here)
        a_raw = a0 if c == 0 else np.asarray(Xs[k - 1][0], np.float64)
        G = np.zeros((m, n))
        GR = np.zeros((m, grq.shape[1]))
        G[0] = np.asarray(gq[k], np.float64) + abar
        GR[0] = grq[k]
        fxw = None if fx is None else fx[c:c + m]
        flw = None if flags is None else flags[c:c + m]
        mw = SMC.Model(o, kp[c:c + m], fxw, flw, clip_anchor(o, a_raw), w)
        md = SVC.model_stream(mw, Xs[k][:m], kp[c:c + m], fxw, flw, a_raw, G, GR)
        skip = skip or md["skip"]
        if md["not_pd"]:
            not_pd.append(k)
        g_kp[c:c + m] += md["keypoints"]
        g_f[c:c + m] += md["fixed"]
        if c > 0:
            abar = md["last"]
        else:
            g_last += md["last"]
    return dict(keypoints=g_kp, fixed=g_f, last=g_last, skip=skip, not_pd=not_pd)


def polished_chain(o, w, kp, fx, flags, a0, L, starts, iters=60):
    """The fixed-lag forward in float64: returns Xs (each tick's re-polished window, float64) from the starting windows
    `starts` (e.g. the float32 tape)."""
    K = kp.shape[0]
    Xs = []
    a = np.asarray(a0, np.float64)
    for k in range(K):
        c, m = window(k, L)
        if c > 0:
            a = Xs[k - 1][0]  # the frame tick k - 1 committed
        mw = SMC.Model(o, kp[c:c + m], None if fx is None else fx[c:c + m], None if flags is None else flags[c:c + m],
                       clip_anchor(o, a), w)
        Xs.append(mw.polish(np.asarray(starts[k][:m], np.float64), iters=iters))
    return Xs


def emitted_loss(o, Xs, fx, L, gq, grq):
    """sum over emitting ticks of <gq_k, x> + <grq_k, robot_qpos(x, fixed of the emitted frame)>."""
    Mx, Mf = SVC.maps(o)
    tot = 0.0
    for k, X in enumerate(Xs):
        c, m = window(k, L)
        if m < L + 1:
            continue
        x = X[0]
        rq = Mx @ x + (0 if fx is None else Mf @ np.asarray(fx[c], np.float64))
        tot += float(np.asarray(gq[k], np.float64) @ x + np.asarray(grq[k], np.float64) @ rq)
    return tot


def compare(got_kp, got_f, got_last, md, tau=TAU):
    """Emulated or GPU gradients of one stream against model_chain; returns the worst error in units of tau."""
    e = SVC.stream_errors(got_kp, md["keypoints"])
    if md["fixed"].size:
        e = max(e, SVC.stream_errors(got_f, md["fixed"]))
    e = max(e, SVC.stream_errors(got_last, md["last"]))
    assert e <= tau, e
    return e / tau
