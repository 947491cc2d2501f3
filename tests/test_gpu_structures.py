"""The CUDA solver on synthetic robots at the edges of the table format (tests/structure_cases.py): block width 8 (dense
factorisation of a block-diagonal table), 2-4 objective links per joint, n_links = n_res = 16, fixed joints in fingers and
trunks, mimic groups of four / negative multipliers / sources after their mimic joint / across fingers / in the trunk /
prismatic mimics, 1 to 31 DoF, prismatic joints in block and arrow fingers, DexPilot on two- and three-finger hands.
Frames against the float64 oracle, sequences against their frame-by-frame twin, and a mixed-robot launch against
per-robot launches."""
import numpy as np
import pytest

import structure_cases as SC
from helpers import build_oracle, build_product, keypoint_trajectory

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_gpu_parity import gpu_solve  # noqa: E402

TOL = 1e-4
N_FRAMES = 24


def _set_flags(o, flags, i):
    if o.type == "dexpilot":
        o.projected[:] = flags[i].astype(bool)


def _check(o, res, refs, fixed, x0, flags, min_same_basin):
    """test_gpu_parity.check_against_oracle with per-frame initial DexPilot flags: every frame is the oracle's converged
    minimiser (mode B) or a verified other minimiser, the reported cost is the objective at the returned point and the
    flags each frame leaves behind are the oracle's."""
    from oracle.solvers import polish, solve_converged

    q = res["q"].astype(np.float64)
    assert np.all((res["status"] >> 24) == 0), "solver flagged frames"
    assert np.all(q >= o.lower - 1e-6) and np.all(q <= o.upper + 1e-6)
    dq = np.zeros(len(q))
    for i in range(len(q)):
        _set_flags(o, flags, i)
        xb, kkt, _ = solve_converged(o, refs[i], fixed[i], x0[i], update_state=False)
        assert kkt < 1e-6
        dq[i] = np.abs(q[i] - xb).max()
        _set_flags(o, flags, i)
        obj = o.make_objective(refs[i], fixed[i], x0[i], update_state=False)
        if dq[i] >= TOL:
            xp, kkt = polish(obj, q[i], o.lower, o.upper)
            assert kkt < 1e-6 and np.abs(xp - q[i]).max() < TOL, f"frame {i}: GPU answer is not a minimiser (moved {np.abs(xp - q[i]).max():.2e})"
        assert res["cost"][i] == pytest.approx(obj.consistent(q[i]), rel=2e-4, abs=1e-8)
        if flags is not None:
            o.projected[:] = flags[i].astype(bool)
            o.prepare(refs[i], update_state=True)
            np.testing.assert_array_equal(res["projected"][i], o.projected.astype(np.uint8), err_msg=f"frame {i}")
    same = dq < TOL
    print(f"same basin {same.mean():.4f} of {len(same)} (floor {min_same_basin}), |dq| median {np.median(dq):.1e} "
          f"max inside {dq[same].max() if same.any() else float('nan'):.1e}")
    assert same.mean() >= min_same_basin, f"only {same.mean():.3f} of frames in the oracle's basin"
    return dq


@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.id)
def test_structure_case_frames_match_oracle(case, tmp_path):
    seq, o = SC.build(case, tmp_path)
    opt = seq.optimizer
    refs, fixed, x0 = SC.problems(o, N_FRAMES)
    flags = SC.initial_flags(o, N_FRAMES)
    res = gpu_solve(opt, refs, fixed, x0, want_proj=flags is not None, proj_init=None if flags is None else flags.copy())
    info = opt.engine().launch_info()
    assert info["lanes_per_frame"] == (16 if case.expect["dof"] <= 16 else 32)
    dq = _check(o, res, refs, fixed, x0, flags, min_same_basin=0.9)
    assert np.median(dq) < 2e-5


def _fixed_streams(o, S, T, nf, seed=7):
    lim = o.robot.joint_limits[o.idx_pin2fixed]
    return np.random.RandomState(seed).uniform(lim[:, 0], lim[:, 1], size=(S, T, nf)).astype(np.float32)


@pytest.mark.parametrize("cid", ["mimic_fixed_dense16", "mimic_fixed_dense32", "fixed_dense16", "bw8_88_vector",
                                 "bw8_6288_position", "links_block4_position", "links_arrow_vector", "dexpilot_3fingers"])
def test_structure_case_sequences_match_frame_by_frame(cid, tmp_path, monkeypatch):
    """dexr_solve_sequences (fixed joints as [S,T,n_fixed]) == the same recurrence driven frame by frame through the frames
    kernel: warm starts, carried damping and DexPilot flags bit for bit, filtered outputs to the filter's rounding.
    DEXR_SEQ_DUO=0: one group per stream, the summation order of the frames kernel."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    dev = torch.device("cuda", 0)
    case = SC.BY_ID[cid]
    seq, o = SC.build(case, tmp_path)
    opt = seq.optimizer
    S, T, nf = 3, 12, case.expect["n_fixed"]
    kp = keypoint_trajectory()
    kps = np.stack([kp[s:s + 2 * T:2] for s in (0, 150, 400)]).astype(np.float32)
    tk = torch.from_numpy(kps).to(dev)
    fixed = torch.from_numpy(_fixed_streams(o, S, T, nf)).to(dev) if nf else None
    status = torch.zeros((S, T), dtype=torch.int32, device=dev)
    out, state = seq.retarget_sequences(tk, fixed_qpos=fixed, status_out=status)
    torch.cuda.synchronize()
    # (no non-finite flag; bit 24 is allowed: from the mid-range cold start of a stream, the first frame of a position stream
    # with far-away recorded targets on bw8_6288_position / links_block4_position runs into max_iters in the emulation)
    assert int((status >> 25).max()) == 0
    got = out.cpu().numpy()
    st = seq.make_stream_state(S)
    y = None
    for t in range(T):
        rq = torch.zeros((S, opt.robot.dof), dtype=torch.float32, device=dev)
        q = opt.retarget_batch(keypoints=tk[:, t].contiguous(), fixed_qpos=fixed[:, t].contiguous() if nf else None,
                               last_qpos=st.last_qpos, robot_qpos_out=rq, projected=st.projected, clip_init=True, damping=st.damping)
        st.last_qpos = q
        y = rq if y is None else y + seq.filter.alpha * (rq - y)
        torch.cuda.synchronize()
        np.testing.assert_allclose(got[:, t], y.cpu().numpy(), atol=2e-6, err_msg=f"{cid} step {t}")
    np.testing.assert_array_equal(state.last_qpos.cpu().numpy(), st.last_qpos.cpu().numpy())
    np.testing.assert_array_equal(state.damping.cpu().numpy(), st.damping.cpu().numpy())
    if st.projected is not None:
        np.testing.assert_array_equal(state.projected.cpu().numpy(), st.projected.cpu().numpy())


@pytest.mark.parametrize("mode", ["streams", "persistent"])
def test_mixed_launch_with_structure_cases(mode, tmp_path, monkeypatch):
    """One retarget_batch_mixed call over a block-width-8 robot, a robot with fixed and mimic joints, a 32-lane robot with
    four links on one joint and a shipped hand equals one retarget_batch launch per robot bit for bit, in both
    DEXR_MULTI_MODEs."""
    from dex_retargeting_b200.optimizer import retarget_batch_mixed

    monkeypatch.setenv("DEXR_MULTI_MODE", mode)
    dev = torch.device("cuda", 0)
    robots = [SC.build(SC.BY_ID[c], tmp_path) for c in ("bw8_5344_position", "mimic_fixed_dense32", "links_dense32_position")]
    robots.append((build_product("teleop/allegro_hand_right"), build_oracle("teleop/allegro_hand_right")))
    jobs = []
    for i, ((seq, o), n) in enumerate(zip(robots, (300, 77, 130, 500))):
        refs, fixed, x0 = SC.problems(o, n, seed=30 + i)
        kw = dict(ref_value=torch.from_numpy(refs).to(dev), last_qpos=torch.from_numpy(x0).to(dev),
                  fixed_qpos=torch.from_numpy(fixed).to(dev) if fixed.shape[1] else None,
                  status_out=torch.zeros((n,), dtype=torch.int32, device=dev), cost_out=torch.zeros((n,), device=dev))
        jobs.append((seq.optimizer, kw))

    def clone(kw):
        return {k: (v.clone() if hasattr(v, "clone") else v) for k, v in kw.items()}

    ref = []
    for opt, kw in jobs:
        k2 = clone(kw)
        ref.append((opt.retarget_batch(**k2), k2))
    mixed = [(opt, clone(kw)) for opt, kw in jobs]
    outs = retarget_batch_mixed(mixed)
    torch.cuda.synchronize()
    for (q_ref, k_ref), q_mix, (_, k_mix) in zip(ref, outs, mixed):
        assert torch.equal(q_ref, q_mix)
        assert torch.equal(k_ref["status_out"], k_mix["status_out"])
        assert torch.equal(k_ref["cost_out"], k_mix["cost_out"])
        assert int((k_mix["status_out"] >> 24).max()) == 0
