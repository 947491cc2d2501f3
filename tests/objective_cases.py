"""Inputs and float64 expectations of the objective-evaluation tests (`dexr_eval_objective`), shared by the host emulation
(tests/test_objective_emulation.py) and the GPU suite (tests/test_gpu_objective.py)."""
import numpy as np

from helpers import GOLDEN, keypoint_trajectory

VEC = np.load(GOLDEN / "reference_vectors.npz")
REF_CASES = sorted({k.split("/")[0] for k in VEC.files if k.endswith("/values")})

# Against values the reference's own closure returned (tests/golden/reference_vectors.npz).  Worst seen, in the host emulation
# and on an H100 alike: loss 5.8e-6 relative, gradient 1.2e-5 of |g_ref|_inf (Inspire position with mimic joints and a
# free-flying base: float32 link positions of a few metres)
REF_LOSS_RTOL, REF_LOSS_ATOL = 1e-5, 1e-9
REF_GRAD_RTOL, REF_GRAD_ATOL = 5e-5, 1e-7  # of |g_ref|_inf


def reference_frames(case):
    """The fixture's problems with each of their 3 points as one frame, DexPilot flags starting at 0.  Returns dict(key, qpos,
    ref_value, fixed_qpos (None without fixed joints), last_qpos, values, grads, projected (flags after the call, uint8, or
    None))."""
    refs, fixed, last, pts = (VEC[f"{case}/{k}"] for k in ("ref_value", "fixed_qpos", "last_qpos", "points"))
    n, P = pts.shape[:2]
    rep = lambda a: np.ascontiguousarray(np.repeat(a, P, axis=0), dtype=np.float32)  # noqa: E731
    proj = VEC[f"{case}/projected"] if f"{case}/projected" in VEC.files else None
    return dict(key=str(VEC[f"{case}/key"]), qpos=np.ascontiguousarray(pts.reshape(n * P, -1), dtype=np.float32),
                ref_value=rep(refs), fixed_qpos=rep(fixed) if fixed.shape[1] else None, last_qpos=rep(last),
                values=VEC[f"{case}/values"].reshape(-1), grads=VEC[f"{case}/grads"].reshape(n * P, -1),
                projected=None if proj is None else np.repeat(proj, P, axis=0).astype(np.uint8))


def initial_flags(opt, B):
    return np.zeros((B, len(opt.projected)), np.uint8) if opt.retargeting_type == "DEXPILOT" else None


def reference_errors(loss, grad, values, grads):
    """Worst relative loss error and worst gradient error in units of |g_ref|_inf; asserts the tolerances above."""
    dl = np.abs(loss.astype(np.float64) - values)
    assert np.all(dl <= REF_LOSS_RTOL * np.abs(values) + REF_LOSS_ATOL), (loss, values)
    gmax = np.abs(grads).max(1)
    dg = np.abs(grad.astype(np.float64) - grads).max(1)
    assert np.all(dg <= REF_GRAD_RTOL * gmax + REF_GRAD_ATOL), dg / gmax
    return float((dl / np.maximum(np.abs(values), 1e-30)).max()), float((dg / np.maximum(gmax, 1e-30)).max())


def oracle_points(o, n, seed, with_last=True):
    """n seeded frames of optimizer `o` (oracle): recorded human keypoints [n,21,3] (their gather = ref_value), joint vectors
    drawn up to 0.2 rad / m beyond the bounds, anchors 0.05 from them (or None), fixed joints inside their limits."""
    rng = np.random.RandomState(seed)
    traj = keypoint_trajectory().astype(np.float32)
    kp = np.ascontiguousarray(traj[rng.randint(0, len(traj), n)] + (rng.randn(n, 1, 3) * 0.002).astype(np.float32))
    kp[:, 0] = 0
    ref = np.stack([o.ref_from_keypoints(k) for k in kp]).astype(np.float32)
    lo, hi = o.joint_limits[:, 0] - 0.2, o.joint_limits[:, 1] + 0.2
    x = rng.uniform(lo, hi, size=(n, o.opt_dof)).astype(np.float32)
    last = (x + 0.05 * rng.randn(n, o.opt_dof)).astype(np.float32) if with_last else None
    lim = o.robot.joint_limits[o.idx_pin2fixed]
    fixed = rng.uniform(lim[:, 0], lim[:, 1], size=(n, len(o.idx_pin2fixed))).astype(np.float32)
    return dict(keypoints=kp, ref_value=ref, qpos=x, last_qpos=last, fixed_qpos=fixed if fixed.shape[1] else None)


def oracle_expect(o, pts):
    """float64 loss, cost, grad (and the DexPilot flags after the call, starting from 0) of oracle_points' frames."""
    n = pts["qpos"].shape[0]
    nf = len(o.idx_pin2fixed)
    L, Cst, G, P = np.zeros(n), np.zeros(n), np.zeros((n, o.opt_dof)), []
    for i in range(n):
        x = pts["qpos"][i].astype(np.float64)
        last = pts["qpos"][i] if pts["last_qpos"] is None else pts["last_qpos"][i]
        fixed = pts["fixed_qpos"][i] if nf else np.zeros(0)
        if o.type == "dexpilot":
            o.projected[:] = False
        obj = o.make_objective(pts["ref_value"][i], fixed, last, update_state=True)
        L[i], G[i] = obj.value_and_grad(x)
        Cst[i] = obj.consistent(x)
        if o.type == "dexpilot":
            P.append(o.projected.astype(np.uint8))
    return L, Cst, G, (np.array(P) if P else None)


# Against the float64 oracle at arbitrary points (float32 kinematics and targets on the library's side).  Worst seen: host
# emulation over every configuration and structure case 3.5e-7 (loss, cost) and 1.3e-6 (gradient); H100, bench-batch
# sample 3.2e-6 and 3.6e-6
ORC_RTOL, ORC_ATOL = 2e-5, 1e-8
ORC_GRAD_RTOL, ORC_GRAD_ATOL = 5e-5, 1e-7


def oracle_errors(loss, cost, grad, L, Cst, G):
    """Asserts loss, cost (relative) and grad (in units of |g|_inf) against the oracle; returns the worst of each."""
    el = np.abs(loss - L) / np.maximum(np.abs(L), 1e-30)
    ec = np.abs(cost - Cst) / np.maximum(np.abs(Cst), 1e-30)
    assert np.all(np.abs(loss - L) <= ORC_RTOL * np.abs(L) + ORC_ATOL), el.max()
    assert np.all(np.abs(cost - Cst) <= ORC_RTOL * np.abs(Cst) + ORC_ATOL), ec.max()
    gmax = np.abs(G).max(1)
    dg = np.abs(grad - G).max(1)
    assert np.all(dg <= ORC_GRAD_RTOL * gmax + ORC_GRAD_ATOL), (dg / gmax).max()
    return float(el.max()), float(ec.max()), float((dg / np.maximum(gmax, 1e-30)).max())


def ulp(v):
    return np.spacing(np.abs(np.asarray(v, np.float32)))


def projected_gradient(g, x, lo, hi):
    """The gradient without its outward components at active bounds (a minimiser inside [lo, hi] makes this 0)."""
    out = ((x <= lo) & (g > 0)) | ((x >= hi) & (g < 0))
    return np.where(out, 0.0, g)


# One configuration per solver instantiation and loss (and the mimic + free-flying-base position hand): solve, then evaluate
SOLVER_CASES = ["teleop/allegro_hand_right", "teleop/leap_hand_right_dexpilot", "teleop/ability_hand_right",
                "teleop/shadow_hand_right", "offline/shadow_hand_right", "teleop/schunk_svh_hand_right",
                "offline/inspire_hand_right"]
PGRAD_BOUND = 5e-5  # |projected gradient|_inf at a converged solve; worst seen 3.8e-6 (emulation), 8.7e-6 (H100)


def check_after_solve(o, q, status, cost, proj_solve, cost0, cost_eval, grad, proj_eval):
    """The evaluation at a solve's answer, anchored at the solve's warm start, against what the solve reported.  The solve
    carries its cost as F + dF from step to step: a few ulp of drift per accepted step, ulp of the larger F of the two points
    a step joins, so at most of the cost at the (clipped) warm start, `cost0`.  Returns the worst cost drift (in ulp of
    the solve's cost) and the worst projected gradient on converged frames."""
    iters = (status & 0xFFFF).astype(np.float64)
    bound = 4 * ulp(np.maximum(cost0, cost)) * (iters + 1)
    drift = np.abs(cost_eval.astype(np.float64) - cost)
    assert np.all(drift <= bound), drift / ulp(cost)
    if proj_solve is not None:
        np.testing.assert_array_equal(proj_eval, proj_solve)
    conv = (status >> 23) & 3 == 0
    assert conv.mean() > 0.5
    pg = projected_gradient(grad, q, np.float32(o.lower), np.float32(o.upper))
    worst = float(np.abs(pg[conv]).max())
    assert worst < PGRAD_BOUND, worst
    return float((drift / ulp(cost)).max()), worst
