"""The float64 model of the acceleration-penalised smoother (`dexr_smooth_sequences_packed_accel`) and of its
backpropagation (`dexr_smooth_sequences_packed_accel_vjp`), shared by the host emulation
(tests/test_smooth_accel_emulation.py), the GPU suite (tests/test_gpu_smooth_accel.py) and tools/bench_smooth_accel.py.

The model states the problem of one stream independently of the kernel's elimination:
  F_c(X) = F(X) + c sum_{triples (t-1, t, t+1)} |x_{t+1} - 2 x_t + x_{t-1}|^2,
F the smoother's objective of `smooth_cases.Model` (the oracle's per-frame loss, flags held at the causal tape's), the clipped
anchor standing in for frame -1 when it is given.  The smoothness terms are written as weighted difference rows over
(x_0 .. x_{T-1}, a): velocity rows (x_t - x_{t-1}, weight w), the anchor row (x_0 - a, weight w) and the triples' rows
(coefficients 1, -2, 1, weight c), so their gradient and Hessian follow from that one matrix.  `polish` is a dense damped
projected Newton method on the stacked problem (so only short clips); `model_vjp` is the implicit-function VJP with the
dense stacked Hessian, the anchor's share taken from the rows' derivative in a.
"""
import numpy as np

import smooth_cases as SMC
import smooth_vjp_cases as SVC
import vjp_cases as V

PARITY = SMC.PARITY
TAU = SVC.TAU


class Model(SMC.Model):
    """One stream of the acceleration-penalised smoother: smooth_cases.Model plus the acceleration weight c."""

    def __init__(self, o, keypoints, fixed, flags, anchor, w, c):
        super().__init__(o, keypoints, fixed, flags, anchor, w)
        self.c = float(c)
        T, has_a = self.T, self.anchor is not None
        rows, wts = [], []

        def row(coefs, weight):
            r = np.zeros(T + 1)  # column T: the anchor
            for t, v in coefs:
                r[T if t < 0 else t] += v
            rows.append(r)
            wts.append(weight)

        for t in range(1, T):
            row([(t, 1.0), (t - 1, -1.0)], self.w)
        if has_a and T > 0:
            row([(0, 1.0), (-1, -1.0)], self.w)
        for s in range(0 if has_a else 1, T - 1):
            row([(s + 1, 1.0), (s, -2.0), (s - 1, 1.0)], self.c)
        self.D = np.array(rows).reshape(-1, T + 1)
        self.Wr = np.array(wts)

    def _residuals(self, X):
        a = self.anchor if self.anchor is not None else np.zeros(self.n)
        Y = np.concatenate([np.asarray(X, np.float64).reshape(self.T, self.n), a[None]])
        return self.D @ Y

    def smooth_value(self, X):
        R = self._residuals(X)
        return float((self.Wr[:, None] * R * R).sum())

    def accel_value(self, X):
        """sum over the triples of |second difference|^2 (the term c weighs)."""
        R = self._residuals(X)
        acc = np.abs(self.D).sum(1) == 4.0
        return float((R[acc] ** 2).sum())

    def value(self, X):
        X = np.asarray(X, np.float64)
        return sum(self._frame(t, X[t], False)[0] for t in range(self.T)) + self.smooth_value(X)

    def smooth_grad(self, X):
        R = self._residuals(X)
        return 2.0 * self.D[:, :self.T].T @ (self.Wr[:, None] * R)

    def smooth_hessian(self):
        """[T,T]: the smoothness Hessian is this matrix times I_n."""
        Dx = self.D[:, :self.T]
        return 2.0 * Dx.T @ (self.Wr[:, None] * Dx)

    def smooth_grad_anchor(self):
        """d(smooth_grad)_t / d a as [T] scalars, each multiplying I_n."""
        return 2.0 * self.D[:, :self.T].T @ (self.Wr * self.D[:, self.T])

    def hessian(self, X):
        """The dense stacked Hessian of F_c [T n, T n] (exact per-frame Hessians)."""
        T, n = self.T, self.n
        H = np.kron(self.smooth_hessian(), np.eye(n))
        for t in range(T):
            H[t * n:(t + 1) * n, t * n:(t + 1) * n] += self._frame(t, X[t], True)[2]
        return H

    def polish(self, X0, iters=40):
        """Dense damped projected Newton from X0 (clipped to the bounds); returns the float64 minimiser."""
        X = np.clip(np.asarray(X0, np.float64), self.lo, self.hi)
        T, n = self.T, self.n
        if T == 0:
            return X
        f = self.value(X)
        for _ in range(iters):
            g = self.grad(X)
            free = (~(((X <= self.lo) & (g > 0)) | ((X >= self.hi) & (g < 0)))).ravel()
            H = self.hessian(X)
            Hf = H[np.ix_(free, free)]
            Hf = 0.5 * (Hf + Hf.T)
            D = np.zeros(T * n)
            if free.any():
                ev = np.linalg.eigvalsh(Hf)
                if ev[0] <= 1e-12 * max(abs(ev).max(), 1.0):  # indefinite: damp to positive definite
                    Hf = Hf + (1e-12 * abs(ev).max() - ev[0] + 1e-9) * np.eye(free.sum())
                D[free] = np.linalg.solve(Hf, -g.ravel()[free])
            D = D.reshape(T, n)
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


def stream_models(o, keypoints, offsets, fixed, flags, anchors, w, c):
    """A Model per packed stream (arguments as smooth_cases.stream_models, plus c)."""
    out = []
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        out.append(Model(o, keypoints[a:b], None if fixed is None else fixed[a:b], None if flags is None else flags[a:b],
                         None if anchors is None else anchors[s], w, c))
    return out


def jitter(q, offsets):
    """Mean |second difference| of qpos over the frames of every stream that have two neighbours (DESIGN.md 3.14)."""
    d = []
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        if b - a >= 3:
            d.append(np.abs(q[a + 2:b] - 2 * q[a + 1:b - 1] + q[a:b - 2]).ravel())
    return float(np.concatenate(d).mean()) if d else 0.0


def model_vjp(m, X, keypoints, fixed, flags, anchor_raw, grad_qpos=None, grad_robot_qpos=None):
    """The VJP of one stream at the float32 answer X [T,n] (arguments and result as smooth_vjp_cases.model_stream; `m`: its
    Model here).  The active set is the smoother's rule on the total gradient of F_c; V = H_ff^-1 G_f with the dense stacked
    Hessian of F_c; the anchor's cotangent is -(d g / d a)^T V where the clip passes it."""
    o, T, n = m.o, m.T, m.n
    nf = len(o.idx_pin2fixed)
    X = np.asarray(X, np.float64)
    Mx, Mf = SVC.maps(o)
    Gb = np.zeros((T, n))
    direct = np.zeros((T, nf))
    if grad_qpos is not None:
        Gb += np.asarray(grad_qpos, np.float64)
    if grad_robot_qpos is not None:
        grq = np.asarray(grad_robot_qpos, np.float64)
        Gb += grq @ Mx
        direct = grq @ Mf
    g = m.grad(X)
    act = ((X <= m.lo) & (g > -1e-7)) | ((X >= m.hi) & (g < 1e-7))
    free = ~act.ravel()
    Hff = m.hessian(X)[np.ix_(free, free)]
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
        a_bar = np.zeros(n) if not_pd else -(m.smooth_grad_anchor() @ Vm) * passes
    return dict(keypoints=kp_bar, fixed=f_bar, last=a_bar, not_pd=not_pd, skip=singular or near, n_active=int(act.sum()),
                V=Vm)
