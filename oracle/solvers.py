"""Oracle solvers and the sequence wrapper.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates, relative to the reference repository:
  src/dex_retargeting/optimizer.py:77-102   Optimizer.retarget: nlopt LD_SLSQP from last_qpos inside
        [lo-1e-3, hi+1e-3], stop on ftol_abs, result cast to float32, RuntimeError -> last_qpos.
        nlopt is absent offline; scipy.optimize SLSQP (same Kraft SLSQP code base, different stop
        test plumbing) is the stand-in -- "restated reference path".
  src/dex_retargeting/seq_retarget.py:112-134  SeqRetargeting.retarget: clip warm start to the
        un-widened limits, solve, keep the UNFILTERED solution as the next warm start, scatter to
        the full qpos, mimic forward, low-pass filter
  src/dex_retargeting/optimizer_utils.py:1-17  LPFilter
  tests/test_optimizer.py:27-81            seeded problem generators (sample_qpos etc.)
"""
import numpy as np
from scipy.optimize import minimize

from .objectives import OracleOptimizer


def solve_reference(opt: OracleOptimizer, ref_value, fixed_qpos, last_qpos, maxiter=1000):
    """Mode A.  Returns (qpos float32, n objective evaluations)."""
    obj = opt.make_objective(ref_value, fixed_qpos, last_qpos)
    x0 = np.asarray(last_qpos, dtype=np.float64)
    try:
        res = minimize(obj.value_and_grad, x0, jac=True, method="SLSQP",
                       bounds=list(zip(opt.lower, opt.upper)), options=dict(ftol=opt.ftol, maxiter=maxiter))
        x = res.x
    except Exception as e:  # the reference prints and returns last_qpos (optimizer.py:99-102)
        print(e)
        x = x0
    return np.asarray(x, dtype=np.float32), obj.n_eval


def projected_gradient_norm(x, g, lo, hi, tol=1e-9):
    """inf-norm of the KKT residual for a box-constrained minimum."""
    pg = g.copy()
    pg[(x <= lo + tol) & (g > 0)] = 0.0
    pg[(x >= hi - tol) & (g < 0)] = 0.0
    return float(np.abs(pg).max()) if pg.size else 0.0


def _consistent_value_and_grad(obj):
    def f(x):
        v, g = obj.value_and_grad(x)
        return v + obj.o.norm_delta * float(((x - obj.last) ** 2).sum()), g

    return f


def polish(obj, x, lo, hi, iters=200, tol=1e-13):
    """Float64 projected, damped Newton on F = L + norm_delta |x - x_last|^2 with the exact Hessian.
    Used to drive a good iterate to a KKT point; returns (x, kkt residual)."""
    o = obj.o
    f = _consistent_value_and_grad(obj)
    x = np.clip(np.asarray(x, float), lo, hi)
    fx, g = f(x)
    lam = 1e-6
    for _ in range(iters):
        if projected_gradient_norm(x, g, lo, hi) < tol:
            break
        H = _ggn_hessian(obj, x)
        free = ~(((x <= lo) & (g > 0)) | ((x >= hi) & (g < 0)))
        improved = False
        for _try in range(30):
            A = H + lam * np.diag(np.abs(np.diag(H)) + 1e-9)
            A = A[np.ix_(free, free)]
            try:
                np.linalg.cholesky(A)  # the exact Hessian can be indefinite away from a minimum
                step = -np.linalg.solve(A, g[free])
            except np.linalg.LinAlgError:
                lam *= 10
                continue
            xn = x.copy()
            xn[free] += step
            xn = np.clip(xn, lo, hi)
            fn, gn = f(xn)
            if fn <= fx:
                x, fx, g = xn, fn, gn
                lam = max(lam * 0.2, 1e-12)
                improved = True
                break
            lam *= 10
        if not improved:
            break
    return x, projected_gradient_norm(x, g, lo, hi)


def _fold(o, Hq):
    """pinocchio-order (dof x dof) -> variable order (n x n): M^T Hq M with q = M x + c (mimic map)."""
    M = np.zeros((o.robot.dof, o.opt_dof))
    M[o.idx_pin2target, np.arange(o.opt_dof)] = 1.0
    if o.adaptor is not None:
        a = o.adaptor
        for i in range(len(a.idx_pin2mimic)):
            M[a.idx_pin2mimic[i], a.idx_target2source[i]] = a.multipliers[i]
    return M.T @ Hq @ M


def _ggn_hessian(obj, x, majoriser=False):
    """Exact Hessian of the consistent objective: loss curvature through the Jacobian + the kinematic
    second-derivative term + the regulariser.  `majoriser` (position loss only): beyond the quadratic
    zone a coordinate contributes the curvature 1/|d| of the Huber majoriser instead of the exact 0."""
    o = obj.o
    pos, J = obj._kin(x, True)
    n = o.opt_dof
    H = 2.0 * o.norm_delta * np.eye(n)
    beta = o.huber_delta
    _, gpos = obj._loss(pos, True)
    H += _fold(o, o.robot.link_position_hessian_contraction(o.link_ids, gpos))
    if o.type == "position":
        d = pos - obj.target
        a = np.abs(d)
        w = np.where(a < beta, 1.0 / beta, 1.0 / np.maximum(a, beta) if majoriser else 0.0) / d.size
        H += np.einsum("lc,lci,lcj->ij", w, J, J)
        return H
    Jv = J[o.task_sel] - J[o.origin_sel]  # (m,3,n)
    diff = pos[o.task_sel] - pos[o.origin_sel] - obj.target
    dist = np.linalg.norm(diff, axis=1)
    for k in range(o.m):
        wk = obj.weights[k] / o.m
        if dist[k] < beta:
            Hr = np.eye(3) / beta
        else:
            u = diff[k] / dist[k]
            Hr = (np.eye(3) - np.outer(u, u)) / dist[k]
        H += wk * Jv[k].T @ Hr @ Jv[k]
    return H


def solve_converged(opt: OracleOptimizer, ref_value, fixed_qpos, last_qpos, x_init=None, update_state=True):
    """Mode B.  Minimise the consistent objective from `last_qpos` (or `x_init`): SLSQP at a tight
    tolerance to pick the basin the way the reference's solver class would, then polish to a KKT
    point.  Returns (x float64, kkt residual, F(x))."""
    obj = opt.make_objective(ref_value, fixed_qpos, last_qpos, update_state)
    f = _consistent_value_and_grad(obj)
    x0 = np.asarray(last_qpos if x_init is None else x_init, dtype=np.float64)
    x0 = np.clip(x0, opt.lower, opt.upper)
    res = minimize(f, x0, jac=True, method="SLSQP", bounds=list(zip(opt.lower, opt.upper)),
                   options=dict(ftol=1e-9, maxiter=300))
    x, kkt = polish(obj, res.x, opt.lower, opt.upper)
    return x, kkt, obj.consistent(x)


class OracleLPFilter:
    """optimizer_utils.py:1-17."""

    def __init__(self, alpha):
        self.alpha, self.y, self.is_init = alpha, None, False

    def next(self, x):
        if not self.is_init:
            self.y, self.is_init = x, True
            return self.y.copy()
        self.y = self.y + self.alpha * (x - self.y)
        return self.y.copy()


class OracleSeqRetargeting:
    """seq_retarget.py:12-157 (without warm_start) over either solver mode."""

    def __init__(self, opt: OracleOptimizer, mode="reference"):
        self.opt, self.mode = opt, mode
        self.joint_limits = opt.joint_limits
        self.last_qpos = self.joint_limits.mean(1).astype(np.float32)
        a = opt.low_pass_alpha
        self.filter = OracleLPFilter(a) if 0 <= a <= 1 else None
        self.n_eval = 0

    def set_qpos(self, robot_qpos):
        self.last_qpos = np.asarray(robot_qpos)[self.opt.idx_pin2target]

    def retarget(self, ref_value, fixed_qpos=np.array([])):
        o = self.opt
        last = np.clip(self.last_qpos, self.joint_limits[:, 0], self.joint_limits[:, 1])
        ref32, fixed32 = np.asarray(ref_value).astype(np.float32), np.asarray(fixed_qpos).astype(np.float32)
        if self.mode == "reference":
            qpos, ne = solve_reference(o, ref32, fixed32, last)
            self.n_eval += ne
        else:
            x, _, _ = solve_converged(o, ref32, fixed32, last)
            qpos = x.astype(np.float32)
        self.last_qpos = qpos
        robot_qpos = np.zeros(o.robot.dof)
        robot_qpos[o.idx_pin2fixed] = fixed_qpos
        robot_qpos[o.idx_pin2target] = qpos
        if o.adaptor is not None:
            robot_qpos = o.adaptor.forward_qpos(robot_qpos)
        if self.filter is not None:
            robot_qpos = self.filter.next(robot_qpos)
        return robot_qpos


# ------------------------------------------------------------------ tests/test_optimizer.py protocol
def sample_qpos(opt: OracleOptimizer, rng_module=np.random):
    """tests/test_optimizer.py:27-42 (uses the global numpy RNG exactly like the reference)."""
    eps = 1e-5
    lim = opt.robot.joint_limits
    q = rng_module.uniform(lim[:, 0], lim[:, 1])
    if opt.adaptor is not None:
        q = opt.adaptor.forward_qpos(q)
    init = np.clip(q + rng_module.randn(opt.robot.dof) * 0.5, lim[:, 0] + eps, lim[:, 1] - eps)
    return q, init


def generate_problem(opt: OracleOptimizer, rng_module=np.random):
    """tests/test_optimizer.py:56-81: (q*, init in pinocchio order, reachable target)."""
    q, init = sample_qpos(opt, rng_module)
    opt.robot.compute_forward_kinematics(q)
    pos = opt.robot.link_positions(opt.link_ids)
    if opt.type == "position":
        target = pos
    else:
        target = pos[opt.task_sel] - pos[opt.origin_sel]
    return q, init, target
