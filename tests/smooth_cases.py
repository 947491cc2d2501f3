"""The float64 model of the offline smoother (`dexr_smooth_sequences_packed`), shared by the host emulation
(tests/test_smooth_emulation.py), the GPU suite (tests/test_gpu_smooth.py) and tools/bench_smooth.py.

The model states the smoothed problem of one stream independently of the kernel, from the oracle:
  F(X) = sum_t L_t(x_t) + w sum_{t>=1} |x_t - x_{t-1}|^2 + w |x_0 - a|^2,   x_t in [lo, hi]
with L_t the oracle's `FrameObjective` value (norm_delta 0, targets prepared in float64 with the DexPilot flags the frame
uses held fixed, `vjp_cases._prepared`), no L_t on a missing frame (a non-finite keypoint or fixed joint), a the clipped
anchor (or no anchor term) and [lo, hi] the solver's float32 widened bounds.  `Model.polish` is a float64 projected Newton
method on the stacked problem: the exact Hessians of `oracle.solvers._ggn_hessian`, block-Thomas elimination along the
clip, a backtracking projected step, so it runs at T = 300.
"""
import numpy as np

import vjp_cases as V
from oracle.objectives import FrameObjective
from oracle.solvers import _ggn_hessian

STATUS_MISSING = 1 << 27
PARITY = 1e-4  # rad: how far the float64 polish may move the smoothed answer (the project's parity bar)


class Model:
    """One stream: keypoints [T,21,3], fixed [T,n_fixed] or None, flags [T,len_proj] (the flags frame t uses) or None,
    anchor [n] (clipped) or None, smoothing weight w."""

    def __init__(self, o, keypoints, fixed, flags, anchor, w):
        self.o, self.w = o, float(w)
        self.T = keypoints.shape[0]
        self.n = o.opt_dof
        self.anchor = None if anchor is None else np.asarray(anchor, np.float64)
        self.lo = np.float32(o.lower).astype(np.float64)
        self.hi = np.float32(o.upper).astype(np.float64)
        nf = len(o.idx_pin2fixed)
        self.missing = np.zeros(self.T, bool)
        self.objs = []
        for t in range(self.T):
            fx = np.zeros(0) if fixed is None or nf == 0 else np.asarray(fixed[t], np.float64)
            kp = np.asarray(keypoints[t], np.float64)
            miss = not (np.isfinite(kp).all() and np.isfinite(fx).all())
            self.missing[t] = miss
            if miss:
                self.objs.append(None)
                continue
            tgt, wts = V._prepared(o, o.ref_from_keypoints(kp), None if flags is None else flags[t])
            self.objs.append(FrameObjective(o, tgt, wts, fx, np.zeros(self.n)))

    def _frame(self, t, x, hess):
        """L_t, its gradient and (hess) exact Hessian at x (zeros for a missing frame)."""
        if self.objs[t] is None:
            return 0.0, np.zeros(self.n), (np.zeros((self.n, self.n)) if hess else None)
        with V._NoAnchor(self.o, True):
            v, g = self.objs[t].value_and_grad(x)
            H = _ggn_hessian(self.objs[t], x, majoriser=False) if hess else None
        return v, g, H

    def value(self, X):
        X = np.asarray(X, np.float64)
        f = sum(self._frame(t, X[t], False)[0] for t in range(self.T))
        f += self.w * float(((X[1:] - X[:-1]) ** 2).sum())
        if self.anchor is not None:
            f += self.w * float(((X[0] - self.anchor) ** 2).sum())
        return f

    def smooth_grad(self, X):
        """Gradient of the smoothness terms."""
        G = np.zeros_like(X)
        d = X[1:] - X[:-1]
        G[1:] += 2 * self.w * d
        G[:-1] -= 2 * self.w * d
        if self.anchor is not None:
            G[0] += 2 * self.w * (X[0] - self.anchor)
        return G

    def grad(self, X):
        X = np.asarray(X, np.float64)
        return np.array([self._frame(t, X[t], False)[1] for t in range(self.T)]) + self.smooth_grad(X)

    def polish(self, X0, iters=30):
        """Projected Newton from X0 (clipped to the bounds); returns the float64 minimiser."""
        X = np.clip(np.asarray(X0, np.float64), self.lo, self.hi)
        T, n, w2 = self.T, self.n, 2 * self.w
        f = self.value(X)
        for _ in range(iters):
            fr = [self._frame(t, X[t], True) for t in range(T)]
            g = np.array([r[1] for r in fr]) + self.smooth_grad(X)
            free = ~(((X <= self.lo) & (g > 0)) | ((X >= self.hi) & (g < 0)))
            Zs, ys = [], []
            for t in range(T):  # block Thomas, Z_t the inverse of S_t over the free variables (zero elsewhere)
                k = (t > 0 or self.anchor is not None) + (t + 1 < T)
                S = fr[t][2] + w2 * k * np.eye(n)
                y = -g[t].copy()
                if t > 0:
                    S = S - w2 * w2 * Zs[-1]
                    y = y + w2 * Zs[-1] @ ys[-1]
                f_ = free[t]
                Z = np.zeros((n, n))
                Sf = S[np.ix_(f_, f_)]
                Sf = 0.5 * (Sf + Sf.T)
                ev = np.linalg.eigvalsh(Sf) if f_.any() else np.ones(1)
                if ev[0] <= 1e-12 * max(abs(ev).max(), 1.0):  # indefinite: a gradient step on this frame's block
                    Sf = Sf + (1e-12 * abs(ev).max() - ev[0] + 1e-9) * np.eye(f_.sum())
                Z[np.ix_(f_, f_)] = np.linalg.inv(Sf)
                Zs.append(Z)
                ys.append(np.where(f_, y, 0.0))
            D = np.zeros((T, n))
            dn = np.zeros(n)
            for t in range(T - 1, -1, -1):
                dn = Zs[t] @ (ys[t] + (w2 * dn if t + 1 < T else 0.0))
                D[t] = dn
            step = 1.0
            while step > 1e-6:
                Xn = np.clip(X + step * D, self.lo, self.hi)
                fn = self.value(Xn)
                if fn < f:
                    break
                step *= 0.5
            else:
                return X
            moved = np.abs(Xn - X).max()
            X, f = Xn, fn
            if moved < 1e-12:
                break
        return X


def stream_models(o, keypoints, offsets, fixed, flags, anchors, w):
    """A Model per packed stream: keypoints [N,21,3], offsets [S+1], fixed [N,n_fixed] or None, flags [N,len_proj] (the
    flags each frame uses: the causal tape's) or None, anchors [S,n] (clipped) or None."""
    out = []
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        out.append(Model(o, keypoints[a:b], None if fixed is None else fixed[a:b], None if flags is None else flags[a:b],
                         None if anchors is None else anchors[s], w))
    return out


def clipped_anchor(o, last_qpos):
    """clip(a) at the oracle's joint limits, as the smoother clips the anchor (float32 bounds)."""
    lim = o.joint_limits
    return np.clip(np.asarray(last_qpos, np.float32), np.float32(lim[:, 0]), np.float32(lim[:, 1])).astype(np.float64)


def interpolation(x_prev, x_next, gap, has_prev=True, has_next=True):
    """What the smoothness terms alone give a gap of `gap` frames between x_prev and x_next: the linear interpolation, or
    the one neighbour repeated."""
    if has_prev and has_next:
        s = np.arange(1, gap + 1)[:, None] / (gap + 1)
        return x_prev[None] + s * (x_next - x_prev)[None]
    return np.repeat((x_prev if has_prev else x_next)[None], gap, axis=0)
