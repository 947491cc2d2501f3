"""The float64 model of the backpropagation through acceleration-penalised fixed-lag smoothing
(`dexr_fixed_lag_step_accel_vjp`), shared by the host emulation (tests/test_fixed_lag_accel_vjp_emulation.py) and the GPU
suite (tests/test_gpu_fixed_lag_accel_vjp.py).

One stream from a state with an empty window, anchor a0, pre-anchor p0 and flag hp0, K ticks of lag L, no flush; a loss on
the emitted rows and, optionally, on the final last_qpos and prev_qpos.  Tick k solves the window of frames c_k .. k (c_k =
max(0, k - L)) anchored at A_k with the pre-anchor P_k when H_k = 1 (c_k = 0: a0, p0, hp0; c_k = 1: X^{k-1}[0], a0, 1;
c_k >= 2: X^{k-1}[0], X^{k-2}[0], 1).  Each emitting window is the accel smoother's clip of
`fixed_lag_accel_cases.Model` (the pre-anchor row included), whose VJP is `smooth_accel_cases.model_vjp` (the dense stacked
Hessian); the pre-anchor's cotangent is -(d g / d p)^T V from the same difference rows where the clip passes p.  The
reverse walk carries C1 (the cotangent of X^k[0]) and C2 (that of X^{k-1}[0]) as dexr.h states.

`polished_chain` is the forward in float64: each window re-polished by the model tick by tick, anchored at the previous
re-polished commits -- the function whose central differences check the model."""
import numpy as np

import fixed_lag_accel_cases as FAC
import fixed_lag_vjp_cases as FLC
import smooth_accel_cases as SAC
import smooth_vjp_cases as SVC

TAU = SVC.TAU
window = FLC.window


def _passes(o, q):
    lim = o.joint_limits
    q = np.asarray(q, np.float32)
    return (q >= np.float32(lim[:, 0])) & (q <= np.float32(lim[:, 1]))


def anchors(k, L, a0, p0, hp0, commit):
    """(A_k, P_k, H_k) of tick k (raw); commit(j) is X^j[0]."""
    c, _ = window(k, L)
    if c == 0:
        return a0, p0, bool(hp0)
    return commit(k - 1), (a0 if c == 1 else commit(k - 2)), True


def window_model(o, w, c, kp, fx, flags, A, P, H, k, L):
    cc, m = window(k, L)
    return FAC.Model(o, kp[cc:cc + m], None if fx is None else fx[cc:cc + m], None if flags is None else flags[cc:cc + m],
                     FAC.clipped(o, A), w, c, pre=FAC.clipped(o, P) if H else None)


def model_chain(o, w, c, kp, fx, flags, a0, p0, hp0, Xs, L, gq, grq, glast=None, gprev=None):
    """The VJP of one stream's K ticks at the window points Xs (Xs[k] [m_k, n]).  kp [K,21,3], fx [K,n_fixed] or None,
    flags [K,len_proj] or None, a0 / p0 [n] the raw anchor and pre-anchor, hp0 the flag, gq [K,n] / grq [K,dof] (rows of
    non-emitting ticks are not read), glast / gprev [n] the cotangents of the final last_qpos / prev_qpos (None = 0).
    Returns dict(keypoints [K,21,3], fixed [K,n_fixed], last [n], prev [n], skip, not_pd)."""
    K, n = kp.shape[0], o.opt_dof
    nf = len(o.idx_pin2fixed)
    g_kp, g_f = np.zeros((K, 21, 3)), np.zeros((K, nf))
    g_last, g_prev = np.zeros(n), np.zeros(n)
    cend = max(0, K - L)
    c1, c2 = np.zeros(n), np.zeros(n)
    gl = np.zeros(n) if glast is None else np.asarray(glast, np.float64)
    gp_ = np.zeros(n) if gprev is None else np.asarray(gprev, np.float64)
    # the final last_qpos / prev_qpos: commits cend - 1 and cend - 2 (-1: a0, -2: p0)
    for i, g in ((cend - 1, gl), (cend - 2, gp_)):
        if i == -2:
            g_prev += g
        elif i == -1:
            g_last += g
        elif i == cend - 1:
            c1 = c1 + g
        else:
            c2 = c2 + g
    commit = (lambda j: np.asarray(Xs[j][0], np.float64))
    skip, not_pd = False, []
    for k in range(K - 1, -1, -1):
        cc, m = window(k, L)
        if m < L + 1:
            continue
        A, P, H = anchors(k, L, np.asarray(a0, np.float64), np.asarray(p0, np.float64), hp0, commit)
        mw = window_model(o, w, c, kp, fx, flags, A, P, H, k, L)
        G = np.zeros((m, n))
        GR = np.zeros((m, grq.shape[1]))
        G[0] = np.asarray(gq[k], np.float64) + c1
        GR[0] = grq[k]
        fxw = None if fx is None else fx[cc:cc + m]
        flw = None if flags is None else flags[cc:cc + m]
        md = SAC.model_vjp(mw, Xs[k][:m], kp[cc:cc + m], fxw, flw, A, G, GR)
        skip = skip or md["skip"]
        if md["not_pd"]:
            not_pd.append(k)
        g_kp[cc:cc + m] += md["keypoints"]
        g_f[cc:cc + m] += md["fixed"]
        ga = md["last"]
        gp = np.zeros(n)
        if H and not md["not_pd"]:
            T = mw.T
            dgp = 2.0 * mw.D[:, :T].T @ (mw.Wr * mw.D[:, T + 1])  # d(smooth_grad)_t / d p, [T] scalars
            gp = -(dgp @ md["V"]) * _passes(o, P)
        if cc > 0:
            c1 = c2 + ga
        else:
            g_last += ga
        if cc > 1:
            c2 = gp
        elif cc == 1:
            g_last += gp
        else:
            g_prev += gp
    return dict(keypoints=g_kp, fixed=g_f, last=g_last, prev=g_prev, skip=skip, not_pd=not_pd)


def polished_chain(o, w, c, kp, fx, flags, a0, p0, hp0, L, starts, iters=60):
    """The accelerated fixed-lag forward in float64: each tick's window re-polished from `starts` (e.g. the tape)."""
    Xs = []
    a0, p0 = np.asarray(a0, np.float64), np.asarray(p0, np.float64)
    for k in range(kp.shape[0]):
        _, m = window(k, L)
        A, P, H = anchors(k, L, a0, p0, hp0, lambda j: Xs[j][0])
        mw = window_model(o, w, c, kp, fx, flags, A, P, H, k, L)
        Xs.append(mw.polish(np.asarray(starts[k][:m], np.float64), iters=iters))
    return Xs


def chain_loss(o, Xs, fx, L, gq, grq, a0, p0, glast=None, gprev=None):
    """FLC.emitted_loss plus <glast, final last_qpos> + <gprev, final prev_qpos> (the last two commits, a0 and p0 before
    the first)."""
    tot = FLC.emitted_loss(o, Xs, fx, L, gq, grq)
    K = len(Xs)
    commits = [np.asarray(p0, np.float64), np.asarray(a0, np.float64)] + [Xs[k][0] for k in range(L, K)]
    for g, q in ((glast, commits[-1]), (gprev, commits[-2])):
        if g is not None:
            tot += float(np.asarray(g, np.float64) @ q)
    return tot


def compare(got_kp, got_f, got_last, got_prev, md, tau=TAU):
    """Emulated or GPU gradients of one stream against model_chain; returns the worst error in units of tau."""
    e = FLC.compare(got_kp, got_f, got_last, md, tau)
    e2 = SVC.stream_errors(got_prev, md["prev"])
    assert e2 <= tau, e2
    return max(e, e2 / tau)
