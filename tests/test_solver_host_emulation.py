"""The CUDA solver SOURCE executed on the host (no GPU): tests/emu compiles dex_retargeting_b200/csrc/dexr_kernels.cuh with
g++ through a warp shim -- 32 cooperatively scheduled fibers, the warp collectives as rendezvous points, shared memory as a
NaN-poisoned buffer -- and runs Solver<G, BW>::solve exactly as dexr_frames_kernel does (one frame per group of G lanes).
What this checks: the logic of every solver instantiation (block, dense 16 / 32 lanes, arrow, mimic fold, DexPilot state),
the warp-convergence of every collective, the shared-memory ordering (lanes run one after another between collectives, so a
missing __syncwarp reads stale or NaN data here) and the compile-time experiment switches, all against the float64 oracle.
What it cannot check: GPU arithmetic in the last bits, the TMA ring / kernels of dexr.cu, performance (the -m gpu tests do)."""
import numpy as np
import pytest

import emu_host
from helpers import build_oracle, build_product, keypoint_trajectory, synth_problems

TOL = 1e-4  # rad / m, BASELINE.json's joint-space tolerance

CASES = [  # key, use_arrow, frames
    ("teleop/allegro_hand_right", True, 5),          # Solver<16, 4>: block-diagonal, two frames per warp, odd count
    ("teleop/leap_hand_right_dexpilot", True, 5),    # Solver<16, 0>: dense, DexPilot weights / projected targets
    ("teleop/ability_hand_right", True, 4),          # Solver<16, 0>: mimic fold
    ("teleop/shadow_hand_right", True, 3),           # Solver<32, -1>: arrow, trunk of 2 wrist joints
    ("teleop/shadow_hand_right", False, 3),          # Solver<32, 0>: the same problems through the dense factorisation
    ("offline/shadow_hand_right", True, 2),          # Solver<32, -1>: position loss, free-flying base (trunk of 8)
    ("teleop/schunk_svh_hand_right", True, 2),       # Solver<32, 0>: 20 lanes, 11 mimic joints
]
VARIANTS = [("DEXR_EXP_FASTSINCOS",)]
_cache = {}


def problems(key, n):
    o = build_oracle(key)
    refs, fixed, x0, _ = synth_problems(o, n, np.random.RandomState(3), init_noise=0.05, target_noise=0.01)
    return o, refs, fixed, x0


def oracle_solutions(key, n):
    from oracle.solvers import solve_converged

    if (key, n) not in _cache:
        o, refs, fixed, x0 = problems(key, n)
        X = []
        for i in range(n):
            if o.type == "dexpilot":
                o.projected[:] = False
            xb, kkt, _ = solve_converged(o, refs[i], fixed[i], x0[i], update_state=False)
            assert kkt < 1e-6
            X.append(xb)
        _cache[key, n] = np.array(X)
    return _cache[key, n]


def emulate(key, n, use_arrow, defines=()):
    o, refs, fixed, x0 = problems(key, n)
    opt = build_product(key).optimizer
    proj = np.zeros((n, len(o.projected)), np.uint8) if o.type == "dexpilot" else None
    q, status, cost = emu_host.solve_frames(opt, x0, ref_value=refs, fixed_qpos=fixed if fixed.size else None, projected=proj,
                                           defines=defines, use_arrow=use_arrow)
    return o, refs, fixed, x0, q, status, cost, proj


@pytest.mark.parametrize("key,use_arrow,n", CASES)
def test_solver_source_matches_oracle(key, use_arrow, n):
    o, refs, fixed, x0, q, status, cost, proj = emulate(key, n, use_arrow)
    assert np.all((status >> 24) == 0), "flagged frames"
    XB = oracle_solutions(key, n)
    dq = np.abs(q - XB).max(1)
    assert dq.max() < TOL, dq
    for i in range(n):  # the reported cost is the consistent objective at the returned point
        if o.type == "dexpilot":
            o.projected[:] = False
        obj = o.make_objective(refs[i], fixed[i], x0[i], update_state=(o.type == "dexpilot"))
        assert cost[i] == pytest.approx(obj.consistent(q[i].astype(np.float64)), rel=2e-4, abs=1e-8)
        if o.type == "dexpilot":
            np.testing.assert_array_equal(proj[i], o.projected.astype(np.uint8))


@pytest.mark.parametrize("defines", VARIANTS, ids=lambda d: "+".join(x.replace("DEXR_EXP_", "").lower() for x in d))
@pytest.mark.parametrize("key,use_arrow,n", CASES)
def test_experiment_switches(key, use_arrow, n, defines):
    """Every compile-time experiment (csrc/dexr_kernels.cuh "Experiment switches") solves the same problems:
    DEXR_EXP_FASTSINCOS takes another iteration path and must land on the oracle's minimiser."""
    _, _, _, _, q0, s0, c0, p0 = emulate(key, n, use_arrow)
    o, refs, fixed, x0, q, status, cost, proj = emulate(key, n, use_arrow, defines)
    assert np.all((status >> 24) == 0)
    assert np.abs(q - oracle_solutions(key, n)).max() < TOL
    assert (status & 0xffff).sum() <= (s0 & 0xffff).sum() + 2  # not slower in iterations on these problems
    if proj is not None:
        np.testing.assert_array_equal(proj, p0)


def test_keypoint_gather_and_clip_on_recorded_frames():
    """In-kernel gather from the 21 keypoints (prepare_targets) = the caller-side gather, on recorded human frames with the
    warm start clipped to the joint limits (SeqRetargeting.retarget's prelude)."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    kp = keypoint_trajectory()[::40][:4].astype(np.float32)
    refs = np.stack([o.ref_from_keypoints(k) for k in kp]).astype(np.float32)
    x0 = np.tile(seq.joint_limits.mean(1).astype(np.float32), (len(kp), 1))
    x0[1] = seq.joint_limits[:, 1] + 0.2  # outside the limits: clipped before the solve
    qa, sa, _ = emu_host.solve_frames(seq.optimizer, x0, keypoints=kp, clip_init=True)
    qb, sb, _ = emu_host.solve_frames(seq.optimizer, x0, ref_value=refs, clip_init=True)
    np.testing.assert_array_equal(qa, qb)
    np.testing.assert_array_equal(sa, sb)
    assert np.all(qa <= seq.joint_limits[:, 1] + 1e-3 + 1e-6) and np.all(qa >= seq.joint_limits[:, 0] - 1e-3 - 1e-6)


def test_non_finite_input_is_flagged_and_isolated():
    """A NaN keypoint flags its frame (status bit 25) and returns the warm start; the other frame of the warp is unaffected."""
    key = "teleop/allegro_hand_right"
    o, refs, fixed, x0 = problems(key, 2)
    opt = build_product(key).optimizer
    q_ok, s_ok, _ = emu_host.solve_frames(opt, x0, ref_value=refs)
    bad = refs.copy()
    bad[0, 1, 2] = np.nan
    q, s, _ = emu_host.solve_frames(opt, x0, ref_value=bad)
    assert (s[0] >> 25) & 1 and not (s[1] >> 24)
    np.testing.assert_array_equal(q[0], x0[0])
    np.testing.assert_array_equal(q[1], q_ok[1])


@pytest.mark.parametrize("key,vs_oracle", [("teleop/allegro_hand_right", True), ("teleop/leap_hand_right_dexpilot", False),
                                           ("teleop/schunk_svh_hand_right", True)])
def test_streams_recurrence(key, vs_oracle):
    """The stream recurrence around the same solve() (warm start carried in the lane's register, clip, unfiltered solution =
    next warm start, low-pass filter, DexPilot flags in place: solve_stream, which dexr_sequences_kernel runs) equals the
    frame-by-frame twin through the frames entry bit for bit, and the oracle's SeqRetargeting where basins are unambiguous."""
    from oracle.solvers import OracleSeqRetargeting

    seq = build_product(key)
    opt = seq.optimizer
    S, T = 3, 8
    kp = keypoint_trajectory()
    kps = np.stack([kp[s:s + 2 * T:2] for s in (0, 150, 400)]).astype(np.float32)
    got, status, state = emu_host.solve_sequences(seq, kps)
    assert np.all((status >> 24) == 0)
    # frame-by-frame twin
    last = np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1))
    proj = np.zeros((S, opt._objective_spec().len_proj), np.uint8) if opt.retargeting_type == "DEXPILOT" else None
    damping = np.zeros(S, np.float32)  # the streams' carried damping (dexr_frames_t.damping_io), updated in place
    y = None
    for t in range(T):
        q, _, _ = emu_host.solve_frames(opt, last, keypoints=kps[:, t], projected=proj, clip_init=True, damping=damping)
        last = q
        full = np.zeros((S, opt.robot.dof), np.float32)
        full[:, opt.idx_pin2target] = q
        if opt.adaptor is not None:
            full = np.stack([opt.adaptor.forward_qpos(r.astype(np.float64)) for r in full]).astype(np.float32)
        y = full if y is None else y + np.float32(seq.low_pass_alpha) * (full - y)
        np.testing.assert_allclose(got[:, t], y, atol=2e-6, err_msg=f"{key} step {t}")
    np.testing.assert_array_equal(state["last_qpos"], last)
    np.testing.assert_array_equal(state["damping"], damping)
    assert np.all(damping >= np.float32(opt.lambda0))
    if proj is not None:
        np.testing.assert_array_equal(state["projected"], proj)
    if vs_oracle:
        want = np.zeros((S, T, opt.robot.dof))
        for s in range(S):
            oseq = OracleSeqRetargeting(build_oracle(key), mode="converged")
            for t in range(T):
                want[s, t] = oseq.retarget(oseq.opt.ref_from_keypoints(kps[s, t]))
        assert np.abs(got - want).max() < TOL
    # the state is complete: two calls = one call
    out1, _, st = emu_host.solve_sequences(seq, kps[:, :3])
    out2, _, st = emu_host.solve_sequences(seq, kps[:, 3:], state=st)
    np.testing.assert_array_equal(np.concatenate([out1, out2], axis=1), got)
    # and with every experiment switch on: same streams within the solver tolerance
    exp, st_e, _ = emu_host.solve_sequences(seq, kps, defines=VARIANTS[-1])
    assert np.all((st_e >> 24) == 0)
    if vs_oracle:
        assert np.abs(exp - want).max() < TOL


def test_position_noise_floor_keeps_newton_steps_near_the_minimiser():
    """Shadow position on a free-flying base: link positions of ~0.5 m resolve F ~ 1.3e-3 to ~2e-8 only, ten times coarser
    than a relative floor on |F|.  Before the position-noise floor (and the term-by-term objective differences) frame 38 of
    this batch rejected its converging Newton step on a noise bump, escalated the damping and stopped on a damped step
    4e-4 rad from the minimiser (arrow elimination order).  Every frame must end on the oracle's minimiser, in both
    elimination orders, with the same iteration counts."""
    from oracle.solvers import solve_converged

    key = "offline/shadow_hand_right"
    opt, o = build_product(key).optimizer, build_oracle(key)
    refs, fixed, x0, _ = synth_problems(o, 48, np.random.RandomState(5), init_noise=0.05, target_noise=0.01)
    sel = [36, 37, 38, 39]
    XB = np.array([solve_converged(o, refs[i], fixed[i], x0[i], update_state=False)[0] for i in sel])
    qa, sa, _ = emu_host.solve_frames(opt, x0[sel], ref_value=refs[sel], use_arrow=True)
    qd, sd, _ = emu_host.solve_frames(opt, x0[sel], ref_value=refs[sel], use_arrow=False)
    assert np.abs(qa - XB).max() < 1e-5 and np.abs(qd - XB).max() < 1e-5
    np.testing.assert_array_equal(sa & 0xffff, sd & 0xffff)


def test_trusted_steps_are_verified_by_the_gradient():
    """Steps whose predicted decrease is below what fp32 resolves in F are taken on trust; round 1 kept the damping for them, and
    frames that had collected a large damping early crept towards the minimiser until max_iters (bit 24: 13 of 65 536 LEAP
    DexPilot bench frames, 583 of 614 400 stream frames in the round-1 kernel).  Now the gradient of the next iteration says whether a
    trusted step was good (relax the damping) or whether the KKT residual sits at its fp32 floor (end the frame, bit 23).
    Frame 2452 of the DexPilot bench workload used to stop at 64 iterations 4.3e-4 rad from the oracle."""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    import workloads as W
    from oracle.solvers import solve_converged

    seq = W.build(W.LEAP_DEXPILOT_KEY)
    kp, x0, _, _ = W.frames(seq, 65536, W.SHADOW_SEED)
    idx = [2452, 5297, 5325]
    proj = np.zeros((len(idx), 6), np.uint8)
    q, st, _ = emu_host.solve_frames(seq.optimizer, x0[idx], keypoints=kp[idx], projected=proj)
    assert np.all((st >> 24) == 0) and (st & 0xffff).max() < 40, st & 0xffff
    o = build_oracle(W.LEAP_DEXPILOT_KEY)
    for j, i in enumerate(idx):
        o.projected[:] = False
        xb = solve_converged(o, o.ref_from_keypoints(kp[i]), np.zeros(0), x0[i], update_state=False)[0]
        assert np.abs(q[j] - xb).max() < TOL, (i, np.abs(q[j] - xb).max())


def test_out_of_reach_targets_do_not_cycle():
    """Targets at twice the robot's reach (tests/test_gpu_parity.py::test_bounds_are_respected_and_active): relaxing the damping
    after every trusted step that shrank the gradient drove one frame into a two-cycle (overshoot, damped step, overshoot ...)
    until max_iters; a trusted step that GROWS the gradient now blocks further relaxation until F verifies a decrease."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    refs, fixed, x0, _ = synth_problems(o, 16, np.random.RandomState(9), init_noise=0.05)
    refs = (refs * 1.25).astype(np.float32)
    q, st, _ = emu_host.solve_frames(seq.optimizer, x0, ref_value=refs)
    assert np.all((st >> 24) == 0), st >> 23


@pytest.mark.parametrize("key,hand", [("teleop/allegro_hand_right", "right"), ("teleop/leap_hand_right_dexpilot", "right"),
                                      ("teleop/shadow_hand_left", "left"), ("offline/leap_hand_left", "left")])
def test_fused_keypoint_preprocessing_matches_detector_oracle(key, hand):
    """`dexr_params_t.preprocess`: raw detector landmarks (recorded hand frames under random camera poses) go straight into
    the solver, which applies single_hand_detector.py:100-103, 130-158 in its prelude.  Against oracle/preprocess.py (the
    reference's SVD-based frame estimate, float64) followed by the oracle's converged solve, vector, DexPilot and position
    targets, both hands."""
    from oracle.preprocess import preprocess
    from oracle.solvers import solve_converged

    seq, o = build_product(key), build_oracle(key)
    rng = np.random.RandomState(12)
    base = keypoint_trajectory()[::23][:12].astype(np.float64)
    if hand == "left":
        base = base * np.array([-1.0, 1.0, 1.0])  # mirror the recorded right hand
    B = base.shape[0]
    q4 = rng.randn(B, 4)
    q4 /= np.linalg.norm(q4, axis=1, keepdims=True)
    w, x, y, z = q4.T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                  np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                  np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], 1)
    raw = (np.einsum("bij,bkj->bki", R, base) + rng.randn(B, 1, 3) * 0.3).astype(np.float32)
    x0 = np.tile(seq.joint_limits.mean(1).astype(np.float32), (B, 1))
    nf = len(seq.optimizer.idx_pin2fixed)
    fixed = np.zeros((B, nf), np.float32) if nf else None
    proj = np.zeros((B, len(o.projected)), np.uint8) if o.type == "dexpilot" else None
    q, st, _ = emu_host.solve_frames(seq.optimizer, x0, keypoints=raw, fixed_qpos=fixed, projected=proj, raw_hand=hand)
    assert np.all((st >> 24) == 0)
    inside = 0
    for b in range(B):
        kp, _ = preprocess(raw[b], hand)
        if o.type == "dexpilot":
            o.projected[:] = False
        xb = solve_converged(o, o.ref_from_keypoints(kp.astype(np.float32)), np.zeros(nf), x0[b], update_state=False)[0]
        inside += np.abs(q[b] - xb).max() < TOL
    assert inside >= B - 2, inside  # mid-range cold start on recorded frames: an occasional other basin


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "teleop/ability_hand_right", "teleop/allegro_hand_right"])
def test_two_half_warps_on_one_stream_match_the_single_group(key):
    """Scarce streams (dexr_sequences_kernel with one stream per warp): the second 16-lane group of the warp works on the SAME
    stream and takes every other merged residual pass; the partial gradient / Hessian sums are added across the halves.  Same
    mathematics, another summation order: the trajectories agree to rounding and the DexPilot flags exactly."""
    seq = build_product(key)
    kp = keypoint_trajectory()[None, 100:140].astype(np.float32)
    kp = np.concatenate([kp, kp[:, ::-1]], 0)  # two streams
    a, sa, st_a = emu_host.solve_sequences(seq, kp)
    b, sb, st_b = emu_host.solve_sequences(seq, kp, duo=True)
    assert np.all((sb >> 24) == 0)
    d = np.abs(a - b).max(2)
    assert np.median(d) < 1e-6 and (d < 1e-4).mean() > 0.97, (np.median(d), d.max())
    if st_a["projected"] is not None:
        np.testing.assert_array_equal(st_a["projected"], st_b["projected"])


def test_stop_one_iteration_ahead_stays_inside_the_step_tolerance():
    """kStopAhead (dexr_kernels.cuh): a frame whose last two first-trial steps contract fast enough ends without the iteration
    that would only confirm it.  On the first 512 frames bench.py times that must (a) save iterations -- the round-2 solver
    before it took 3.21 per frame -- and (b) leave every frame within the step tolerance (1e-5 rad) of the oracle's converged
    minimiser, ten times inside the parity bar."""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    import parity as P
    import workloads as W

    seq = W.build(W.METRIC_KEY)
    kp, x0, _, _ = W.frames(seq, 65536, W.METRIC_SEED)
    n = 512
    q, st, _ = emu_host.solve_frames(seq.optimizer, x0[:n], keypoints=kp[:n])
    assert np.all((st >> 24) == 0)
    it = st & 0xffff
    assert it.mean() < 2.7, it.mean()
    dq = np.abs(q - P.fixture()["metric/q"][:n]).max(1)
    assert dq.max() < 1e-5 and np.median(dq) < 5e-7, (dq.max(), np.median(dq))


def test_a_stream_carries_its_damping():
    """kCarry: fed frame by frame, a stream that hands the solver's damping from one frame to the next (damping_io) pays fewer
    rejected steps than the same stream with every frame starting at lambda0, and ends at the same joint angles wherever both
    stay in one basin; the carried value never drops below lambda0."""
    seq = build_product("teleop/leap_hand_right_dexpilot")
    opt = seq.optimizer
    kp = keypoint_trajectory()[:120].astype(np.float32)
    S = 1

    def run(carry):
        last = np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1))
        proj = np.zeros((S, opt._objective_spec().len_proj), np.uint8)
        damping = np.zeros(S, np.float32) if carry else None
        rejects, out, seen = 0, [], []
        for t in range(kp.shape[0]):
            q, st, _ = emu_host.solve_frames(opt, last, keypoints=kp[t][None], projected=proj, clip_init=True, damping=damping)
            assert (st >> 24) == 0
            rejects += int((st[0] >> 16) & 0x7f)
            last = q
            out.append(q[0].copy())
            if carry:
                seen.append(float(damping[0]))
        return rejects, np.array(out), seen

    r_carry, q_carry, seen = run(True)
    r_plain, q_plain, _ = run(False)
    assert min(seen) >= np.float32(opt.lambda0) and max(seen) > np.float32(opt.lambda0)  # some stretch needed more damping
    assert r_carry <= r_plain, (r_carry, r_plain)
    same = np.abs(q_carry - q_plain).max(1) < TOL
    assert same.mean() > 0.5, same.mean()


def test_position_optimizer_initial_damping_on_bench_frames():
    """PositionOptimizer starts at lambda0 = 1e-3 (optimizer.py): on the first 256 config-3 frames bench.py times (Shadow hand
    on a free-flying base, arrow factorisation) every frame still ends in the oracle's minimum, in fewer iterations than from
    1e-2 (3.96 iterations per frame before, 3.29 after)."""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    import parity as P
    import workloads as W

    seq = W.build(W.SHADOW_POS_KEY)
    assert seq.optimizer.lambda0 == 1e-3
    kp, x0, fixed, _ = W.frames(seq, 65536, W.SHADOW_SEED, narrow_dummy=True)
    n = 256
    q, st, _ = emu_host.solve_frames(seq.optimizer, x0[:n], keypoints=kp[:n], fixed_qpos=None if fixed is None else fixed[:n])
    assert np.all((st >> 24) == 0)
    assert (st & 0xffff).mean() < 3.6, (st & 0xffff).mean()
    dq = np.abs(q - P.fixture()["shadow_narrow/q"][:n]).max(1)
    assert dq.max() < TOL and np.median(dq) < 2e-6, (dq.max(), np.median(dq))
