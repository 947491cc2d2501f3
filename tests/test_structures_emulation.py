"""The solver source (host emulation, tests/emu) on synthetic robots at the edges of the table format (tests/structure_cases.py):
block width 8, several objective links per joint up to the maximum, n_links = n_res = 16, fixed joints in fingers and
trunks, mimic groups of four with negative multipliers and offsets, mimic sources after their mimic joint / across fingers /
in the trunk, prismatic joints in block and arrow fingers, 1 to 31 DoF, DexPilot on two- and three-finger hands.  Each case
against the float64 oracle's converged minimiser (mode B): |dq|_inf < 1e-4, no flagged frame, the reported cost is the
objective at the returned point, DexPilot flags equal to the oracle's."""
import numpy as np
import pytest

import emu_host
import structure_cases as SC
from helpers import keypoint_trajectory

TOL = 1e-4
N_FRAMES = 5


def _oracle_b(o, refs, fixed, x0, flags=None):
    """Mode B per frame, and the DexPilot flags each frame leaves behind when it starts from `flags`."""
    from oracle.solvers import solve_converged

    X, P = [], []
    for i in range(len(x0)):
        if o.type == "dexpilot":
            o.projected[:] = flags[i].astype(bool)
        xb, kkt, _ = solve_converged(o, refs[i], fixed[i], x0[i], update_state=False)
        assert kkt < 1e-6
        X.append(xb)
        if o.type == "dexpilot":
            o.projected[:] = flags[i].astype(bool)
            o.prepare(refs[i], update_state=True)
            P.append(o.projected.astype(np.uint8))
    return np.array(X), (np.array(P) if P else None)


@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.id)
def test_structure_case_matches_oracle(case, tmp_path):
    seq, o = SC.build(case, tmp_path)
    opt = seq.optimizer
    refs, fixed, x0 = SC.problems(o, N_FRAMES)
    assert fixed.shape == (N_FRAMES, case.expect["n_fixed"])
    if fixed.size:  # per-frame values inside the limits, not one constant
        lim = o.robot.joint_limits[o.idx_pin2fixed]
        assert np.all(fixed >= lim[:, 0] - 1e-6) and np.all(fixed <= lim[:, 1] + 1e-6) and np.ptp(fixed, axis=0).min() > 0
    flags = SC.initial_flags(o, N_FRAMES)
    proj = None if flags is None else flags.copy()
    q, status, cost = emu_host.solve_frames(opt, x0, ref_value=refs, fixed_qpos=fixed if fixed.size else None, projected=proj)
    assert np.all((status >> 24) == 0), status
    XB, PB = _oracle_b(o, refs, fixed, x0, flags)
    dq = np.abs(q - XB).max(1)
    assert dq.max() < TOL, dq
    for i in range(N_FRAMES):  # the reported cost is the consistent objective at the returned point
        if o.type == "dexpilot":
            o.projected[:] = flags[i].astype(bool)
        obj = o.make_objective(refs[i], fixed[i], x0[i], update_state=False)
        assert cost[i] == pytest.approx(obj.consistent(q[i].astype(np.float64)), rel=2e-4, abs=1e-8)
    if proj is not None:
        np.testing.assert_array_equal(proj, PB)


def test_dexpilot_cases_set_and_clear_flags(tmp_path):
    """The DexPilot cases only check the hysteresis if their frames both set and clear projection flags, and keep a set
    flag inside the band between project_dist and escape_dist."""
    for cid in ("dexpilot_2fingers", "dexpilot_3fingers"):
        _, o = SC.build(SC.BY_ID[cid], tmp_path)
        refs, fixed, x0 = SC.problems(o, N_FRAMES)
        flags = SC.initial_flags(o, N_FRAMES)
        _, PB = _oracle_b(o, refs, fixed, x0, flags)
        s1 = PB[:, 0]
        assert s1[0] == 1 and s1[1] == 1 and s1[2] == 0 and s1[4] == 0, (cid, flags[:, 0], s1)  # set / kept / cleared / not set
        if len(o.projected) > 1:
            assert PB[0, -1] == 1, (cid, PB)  # an S2 pair (both thumb pairs projected, close enough) is projected too


@pytest.mark.parametrize("cid", ["mimic_fixed_dense16", "mimic_fixed_dense32"])
def test_streams_with_fixed_and_mimic_joints(cid, tmp_path):
    """dexr_sequences_kernel's recurrence with fixed joints ([S,T,n_fixed] per step) and mimic joints, one case per solver
    instantiation that takes them (16 and 32 lanes, dense): equal to the frame-by-frame twin through the frames entry, and
    every step's solution is the oracle's converged minimiser from the stream's own (clipped) warm start."""
    from oracle.solvers import solve_converged

    case = SC.BY_ID[cid]
    seq, o = SC.build(case, tmp_path)
    opt = seq.optimizer
    S, T, nf = 2, 6, case.expect["n_fixed"]
    kp = keypoint_trajectory()
    kps = np.stack([kp[s:s + 3 * T:3] for s in (20, 300)]).astype(np.float32)
    lim = o.robot.joint_limits[o.idx_pin2fixed]
    fixed = np.random.RandomState(7).uniform(lim[:, 0], lim[:, 1], size=(S, T, nf)).astype(np.float32)
    got, status, state = emu_host.solve_sequences(seq, kps, fixed_qpos=fixed)
    assert np.all((status >> 24) == 0)
    last = np.tile(seq.joint_limits.mean(1).astype(np.float32), (S, 1))
    damping = np.zeros(S, np.float32)
    y, inside = None, []
    for t in range(T):
        x_in = np.clip(last, seq.joint_limits[:, 0], seq.joint_limits[:, 1])
        q, _, _, full = emu_host.solve_frames(opt, last, keypoints=kps[:, t], fixed_qpos=fixed[:, t], clip_init=True, damping=damping,
                                              want_robot_qpos=True)
        np.testing.assert_array_equal(full[:, o.idx_pin2fixed], fixed[:, t])  # the caller's values, untouched
        y = full if y is None else y + np.float32(seq.low_pass_alpha) * (full - y)
        np.testing.assert_allclose(got[:, t], y, atol=2e-6, err_msg=f"step {t}")
        for s in range(S):
            xb = solve_converged(o, o.ref_from_keypoints(kps[s, t]), fixed[s, t], x_in[s], update_state=False)[0]
            inside.append(np.abs(q[s] - xb).max() < TOL)
        last = q
    np.testing.assert_array_equal(state["last_qpos"], last)
    assert np.mean(inside) >= 0.9, np.mean(inside)
