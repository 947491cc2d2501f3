"""Float64 model of the solver's first damped Newton step, and the frames it is checked on (shared by
tests/test_newton_step_emulation.py and tests/test_gpu_newton_step.py).

Every other solver test checks where the iteration ENDS.  A converged minimiser pins the gradient, but not the Newton system
Solver::solve builds and factorises at every iteration: a wrong curvature term, mimic fold, factorisation or damping shift
only makes convergence slower.  With params.max_iters = 1 and the starting damping given per frame (damping_io /
damping_state), the returned point is clip(x + s, lo, hi), s the first trial's solution of the damped system, whenever that
trial was accepted (no rejects): the step itself becomes visible through the public API.

The model restates dex_retargeting_b200/csrc/dexr_kernels.cuh:719-1221 (the first pass of the iteration loop of
Solver::solve, up to the first trial point):
  :643-648    warm start: xin = last_qpos (clipped to clip_lo / clip_hi with clip_init), anchor x0 = xin, x = clip(xin, lo, hi)
  :743-848    residual passes: Jacobian rows, loss gradient, loss curvature through the Jacobian -- the majoriser 1/max(|r|, beta)
              per coordinate for the position loss (:778-789), the exact norm-Huber curvature for vector / DexPilot on the
              first iteration (`exact`, :790-802)
  :849-864    merged residual passes reduced over the windows, and over the two half-warps in the scarce-streams mode
  :865-887    kinematic curvature a_i . t_c (ancestor half "up", descendant half "dn")
  :888-931    mimic fold H_x = M^T H_q M, g_x = M^T g_q
  :932-957    regulariser gradient 2 nd (x - x0), active set (|g| threshold kGradNoise = 1e-7), freeze of fixed / mimic lanes
  :970-978    diagonal: regulariser 2 nd and damping lam (|H_ii + 2 nd| + 1e-6) added at pivot time
  :983-1183   block, dense and arrow / Schur factorisation and the substitutions
  :1184-1221  positive-definite fallback (not modelled: frames that could reach it do not qualify) and the trial point
              clip(x + s, lo, hi)
Deliberate model choice: kFarResidual (:81) is 1e30, so the kinematic curvature is always in; the model always adds it."""
from dataclasses import dataclass
from typing import Optional

import numpy as np

import structure_cases as SC
from helpers import keypoint_trajectory, synth_problems

GRAD_NOISE = 1e-7         # kGradNoise: active-set threshold on |g|
BOUND_GRAD_MARGIN = 1e-5  # a variable on a bound with |g| below this could fall on either side of the threshold in fp32
PD_MARGIN = 1e-3          # lambda_min(A_ff), Jacobi-scaled, below this could reach the kernel's positive-definite fallback
LAMS = {"near": (1e-6, 1e-2, 1.0), "far": (1.0, 10.0), "bounds": (1e-2, 1.0), "dexpilot": (1e-6, 1e-2, 1.0)}
# Worst ratio of the correct solver: 7.4e-5 in the host emulation, 1.3e-4 on an H100 80GB HBM3 (700 W power limit), both on
# bw8_88_vector and Shadow position on its free-floating base; 9e-5 and below elsewhere -- float32 noise in g and H,
# amplified where the damped system is ill conditioned.  A broken term moves the step by 1e-3 to 1 of its length.
TAU = 2e-3
N = dict(near=24, far=12, bounds=12, dexpilot=12)
SEEDS = dict(near=11, far=12, bounds=13, dexpilot=14)
FLOORS = dict(near=0.75, far=0.5, bounds=0.5, dexpilot=0.5)  # least fraction of the frames that must qualify
# The exact model of these two is indefinite near the pose at lam <= 1e-2 on most frames (those take the positive-definite
# fallback and do not qualify): a free-floating base under the position loss, and 31 joints for three residual vectors.
NEAR_FLOORS = {"offline/shadow_hand_right": 0.4, "dof31_vector": 0.3}
SHIPPED = [  # key, use_arrow: every solver instantiation and mode
    ("teleop/allegro_hand_right", True),        # Solver<16, 4>
    ("teleop/leap_hand_right_dexpilot", True),  # Solver<16, 0>, DexPilot
    ("teleop/ability_hand_right", True),        # Solver<16, 0>, mimic
    ("teleop/shadow_hand_right", False),        # Solver<32, 0>
    ("teleop/schunk_svh_hand_right", True),     # Solver<32, 0>, 11 mimic joints
    ("teleop/shadow_hand_right", True),         # Solver<32, -1>: arrow, trunk of 2
    ("offline/shadow_hand_right", True),        # Solver<32, -1>: arrow, trunk of 8, position loss
]
SHIPPED_RUNS = [(k, a, r) for k, a in SHIPPED for r in ("near", "far", "bounds")] + [("teleop/leap_hand_right_dexpilot", True, "dexpilot")]
# (tests/structure_cases.py; no bounds regime for the 1-DoF robot: its only variable would be held on the bound)
STRUCT_RUNS = [(c.id, r) for c in SC.CASES for r in ("near", "bounds") if not (r == "bounds" and c.expect["dof"] == 1)] + \
    [(c, "dexpilot") for c in ("dexpilot_2fingers", "dexpilot_3fingers")]
STREAM_RUNS = [("teleop/allegro_hand_right", False), ("teleop/leap_hand_right_dexpilot", True), ("teleop/ability_hand_right", True)]


@dataclass
class Frames:
    regime: str
    refs: np.ndarray      # [B, n_res, 3] float32
    fixed: np.ndarray     # [B, n_fixed] float32
    last: np.ndarray      # [B, n] float32 warm starts
    lam: np.ndarray       # [B] float32 starting damping
    flags: Optional[np.ndarray] = None  # [B, len_proj] uint8 DexPilot flags the frames start with
    clip_init: bool = False


def _bound_problems(o, n, rng, init_noise, target_noise):
    """synth_problems, except that a quarter of the variables (at least one) of every frame sit 0.01-0.05 outside a joint
    limit both in the pose that makes the targets and in the warm start.  With clip_init off they start on the bound, and
    the loss and the regulariser anchor both pull outward: they stay active."""
    lim, tl = o.robot.joint_limits, o.joint_limits
    cand = np.flatnonzero(np.abs(tl).max(1) < 10.0)  # (not the unlimited joints of a free-floating base)
    k = max(1, o.opt_dof // 4)
    refs, fixed, last = [], [], []
    for _ in range(n):
        q = rng.uniform(lim[:, 0], lim[:, 1])
        x, fx = q[o.idx_pin2target], q[o.idx_pin2fixed]
        init = np.clip(x + rng.randn(o.opt_dof) * init_noise, tl[:, 0] + 1e-5, tl[:, 1] - 1e-5)
        for j in rng.choice(cand, min(k, len(cand)), replace=False):
            d = rng.uniform(0.01, 0.05)
            x[j] = init[j] = tl[j, 0] - d if rng.rand() < 0.5 else tl[j, 1] + d
        o.robot.compute_forward_kinematics(o.full_qpos(x, fx))
        pos = o.robot.link_positions(o.link_ids)
        ref = pos if o.type == "position" else pos[o.task_sel] - pos[o.origin_sel]
        refs.append((ref + rng.randn(*ref.shape) * target_noise).astype(np.float32))
        fixed.append(fx.astype(np.float32))
        last.append(init.astype(np.float32))
    return np.array(refs), np.array(fixed).reshape(n, -1), np.array(last)


def make_frames(o, regime, n, seed):
    """`n` frames of one regime.
    near:     warm start 0.01 rad from the pose that made the targets, 1 mm target noise, lam 1e-6 / 1e-2 / 1
    far:      0.05 rad, 1 cm (the host emulation suite's problems), lam 1 / 10
    bounds:   near problems with a quarter of the variables outside the joint limits (_bound_problems), clip_init off,
              lam 1e-2 / 1
    dexpilot: near problems with random projection flags preset per frame (200 / 400 weights, projected targets).
    Vector and DexPilot targets except the far ones are divided by the config's scaling factor, which the objective applies
    again: the minimiser is then near the pose."""
    rng = np.random.RandomState(seed)
    init_noise, target_noise = (0.05, 0.01) if regime == "far" else (0.01, 0.001)
    if regime == "bounds":
        refs, fixed, last = _bound_problems(o, n, rng, init_noise, target_noise)
    else:
        refs, fixed, last, _ = synth_problems(o, n, rng, init_noise=init_noise, target_noise=target_noise)
    if regime != "far" and o.type != "position":
        refs = (refs / np.float32(o.scaling)).astype(np.float32)
    lams = LAMS[regime]
    lam = np.array([lams[i % len(lams)] for i in range(n)], np.float32)
    flags = None
    if o.type == "dexpilot":
        lp = len(o.projected)
        flags = rng.randint(0, 2, size=(n, lp)).astype(np.uint8) if regime == "dexpilot" else np.zeros((n, lp), np.uint8)
    return Frames(regime, refs, fixed, last, lam, flags)


def objective(o, fr, i):
    """The frame's FrameObjective, anchored at xin (the clipped last_qpos with clip_init), and xin."""
    xin = fr.last[i].astype(np.float32)
    if fr.clip_init:
        xin = np.clip(xin, o.joint_limits[:, 0].astype(np.float32), o.joint_limits[:, 1].astype(np.float32))
    if o.type == "dexpilot":
        o.projected[:] = fr.flags[i].astype(bool)
    return o.make_objective(fr.refs[i], fr.fixed[i], xin, update_state=False), xin


def newton_step(o, fr, i):
    """The first trial of Solver::solve on frame i, in float64.  Returns a dict: x_start, g, active, A_ff, s, x1 and the
    qualification of the frame (pd: A_ff clear of the fallback; margin: no variable on a bound near the threshold)."""
    from oracle.solvers import _ggn_hessian

    obj, xin = objective(o, fr, i)
    lo, hi = o.lower.astype(np.float32), o.upper.astype(np.float32)
    xs = np.clip(xin, lo, hi)
    x = xs.astype(np.float64)
    _, g = obj.value_and_grad(x)  # J^T dL/dp + 2 nd (x - xin), J through the mimic map
    nd = o.norm_delta
    H = _ggn_hessian(obj, x, majoriser=o.type == "position") - 2.0 * nd * np.eye(o.opt_dof)
    on_lo, on_hi = xs <= lo, xs >= hi
    active = (on_lo & (g > -GRAD_NOISE)) | (on_hi & (g < GRAD_NOISE))
    free = ~active
    lam = float(fr.lam[i])
    d = np.diag(H)
    A = H + np.diag(2.0 * nd + lam * (np.abs(d + 2.0 * nd) + 1e-6))
    Aff = A[np.ix_(free, free)]
    s = np.zeros(o.opt_dof)
    if free.any():
        s[free] = -np.linalg.solve(Aff, g[free])
    x1 = np.clip(x + s, lo.astype(np.float64), hi.astype(np.float64))
    # Cholesky's breakdown and rounding do not change under a symmetric diagonal scaling: judge the scaled matrix (the
    # free-floating base's translations and the finger joints differ by 1e3 in their diagonal entries)
    sc = 1.0 / np.sqrt(np.abs(np.diag(Aff)))
    pd = bool(free.any()) and np.linalg.eigvalsh(Aff * np.outer(sc, sc)).min() > PD_MARGIN
    margin = not np.any((on_lo | on_hi) & (np.abs(g) < BOUND_GRAD_MARGIN))
    return dict(obj=obj, xin=xin, x_start=xs, g=g, active=active, A_ff=Aff, s=s, x1=x1, pd=pd, margin=margin)


def check_frames(o, fr, q, status, cost=None, full=None, tau=1e-4):
    """Per frame: the model's step, whether the frame qualifies (no rejects, A_ff positive definite with margin, no bound
    variable near the active-set threshold) and, for every qualifying frame, the assertions on the kernel's answer.
    Returns (qualifying mask, ratio max|x1_kernel - x1_model| / max|x1_model - x_start| per frame, nan where not
    qualifying, number of active variables per frame).  `cost` / `full`: the reported cost and full joint vector, or None
    where the entry point has none."""
    B = len(q)
    ok = np.zeros(B, bool)
    ratio = np.full(B, np.nan)
    n_act = np.zeros(B, int)
    for i in range(B):
        st = int(status[i])
        assert (st >> 25) & 1 == 0, f"frame {i}: non-finite flag"
        m = newton_step(o, fr, i)
        step = np.abs(m["x1"] - m["x_start"]).max()
        if ((st >> 16) & 0x7f) != 0 or not m["pd"] or not m["margin"] or step == 0.0:
            continue
        ok[i] = True
        n_act[i] = int(m["active"].sum())
        assert st & 0xffff == 1, f"frame {i}: {st & 0xffff} iterations with max_iters = 1"
        qi = np.asarray(q[i], np.float32)
        # (less one float32 ulp of the returned value: the kernel rounds x + s to float32, which alone is 1e-5 of a 1e-2 step)
        ulp = np.spacing(np.abs(m["x1"]).astype(np.float32)).astype(np.float64)
        ratio[i] = np.maximum(np.abs(qi.astype(np.float64) - m["x1"]) - ulp, 0.0).max() / step
        assert ratio[i] <= tau, f"frame {i} ({fr.regime}, lam {fr.lam[i]:g}): step off by {ratio[i]:.2e} of its length (tau {tau:g})"
        np.testing.assert_array_equal(qi[m["active"]], m["x_start"][m["active"]], err_msg=f"frame {i}: active variables moved")
        if cost is not None:
            want = m["obj"].consistent(qi.astype(np.float64))
            assert abs(float(cost[i]) - want) <= 2e-4 * abs(want) + 1e-8, f"frame {i}: cost {float(cost[i])!r} vs {want!r}"
        if full is not None:
            want = o.full_qpos(qi.astype(np.float64), fr.fixed[i])
            fi = np.asarray(full[i], np.float32)
            np.testing.assert_array_equal(fi[o.idx_pin2target], qi, err_msg=f"frame {i}: robot qpos of the variables")
            np.testing.assert_array_equal(fi[o.idx_pin2fixed], fr.fixed[i], err_msg=f"frame {i}: robot qpos of the fixed joints")
            np.testing.assert_allclose(fi, want, rtol=0, atol=2e-6, err_msg=f"frame {i}: robot qpos (mimic joints)")
    return ok, ratio, n_act


def assert_regime(o, fr, q, status, cost, full, label):
    """check_frames, then the least fraction of qualifying frames (and, for the bounds regime, that they hold variables
    on a bound): a case can never pass with nothing checked."""
    ok, ratio, n_act = check_frames(o, fr, q, status, cost, full, TAU)
    print(f"{label} {fr.regime}: {ok.sum()}/{len(ok)} qualify, worst ratio {np.nanmax(ratio) if ok.any() else float('nan'):.2e} "
          f"(tau {TAU:g}), {n_act[ok].sum()} active variables")
    floor = NEAR_FLOORS.get(label, FLOORS["near"]) if fr.regime == "near" else FLOORS[fr.regime]
    assert ok.mean() >= floor, f"{label} {fr.regime}: only {ok.sum()} of {len(ok)} frames qualify (floor {floor})"
    if fr.regime == "bounds":
        assert n_act[ok].sum() > 0, f"{label}: no qualifying frame holds a variable on a bound"


def stream_frames(o, S, seed=21):
    """S streams of one step for the sequences entry: recorded keypoints [S, 1, 21, 3], and the warm start 0.02 rad from
    the oracle's minimiser from mid-range (clip_init, as the sequences kernel always clips)."""
    from oracle.solvers import solve_converged

    rng = np.random.RandomState(seed)
    kp = keypoint_trajectory()
    kps = np.stack([kp[60 + 97 * s] for s in range(S)]).astype(np.float32)[:, None]
    refs = np.stack([o.ref_from_keypoints(k[0]) for k in kps]).astype(np.float32)
    nf = len(o.idx_pin2fixed)
    last = np.zeros((S, o.opt_dof), np.float32)
    for s in range(S):
        if o.type == "dexpilot":
            o.projected[:] = False
        xb = solve_converged(o, refs[s], np.zeros(nf), o.joint_limits.mean(1), update_state=False)[0]
        last[s] = np.clip(xb + 0.02 * rng.randn(o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    lams = LAMS["near"]
    lam = np.array([lams[s % len(lams)] for s in range(S)], np.float32)
    flags = np.zeros((S, len(o.projected)), np.uint8) if o.type == "dexpilot" else None
    return kps, Frames("near", refs, np.zeros((S, nf), np.float32), last, lam, flags, clip_init=True)
