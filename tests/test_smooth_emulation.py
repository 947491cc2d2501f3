"""Offline smoothing (`dexr_smooth_sequences_packed`) through the host emulation of the kernel's own driver (tests/emu runs
smooth_packed_stream of dexr_kernels.cuh on the fiber warp) on block 16, dense 16, arrow 32 and dense 32 fixtures (the smoother
runs every robot on the dense Solver of its lane count), all three losses, with and without mimic and fixed joints, with and
without an anchor, with variables at their bounds: the float64 model of tests/smooth_cases.py (minimiser, descent), the
one-frame and unweighted reductions, missing frames, DexPilot flags that switch, the stream layout (positions, lengths 0 and
1, malformed offsets, non-finite starts), the argument checks, the workspace size, the register budget and a dry run of
tests/test_gpu_smooth.py."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_packed_host as P
import emu_smooth_host as SM
import seq_vjp_cases as SV
import smooth_cases as SMC
import structure_cases as SC
from emu_eval_host import EmulationError
from emu_seq_vjp_host import fresh_state
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID
STATUS_MAXITER, STATUS_NONFINITE, STATUS_MISSING = 1 << 24, 1 << 25, 1 << 27

# (name, kind of the table, how to build it)
CASES = [
    ("allegro_vector", "<16,4>", ("teleop/allegro_hand_right", None)),
    ("leap_dexpilot", "<16,0>", ("teleop/leap_hand_right_dexpilot", None)),
    ("mimic_fixed_dense16", "<16,0>", "mimic_fixed_dense16"),
    ("shadow_position", "<32,-1>", ("offline/shadow_hand_right", None)),
    ("mimic_fixed_dense32", "<32,0>", "mimic_fixed_dense32"),
]
IDS = [c[0] for c in CASES]


def _setup(case, tmp_path):
    name, kind, spec = case
    if isinstance(spec, str):
        seq, o = SC.build(SC.BY_ID[spec], tmp_path)
    else:
        seq, o = build_product(*spec), build_oracle(*spec)
    assert SC.solver_kind(seq.optimizer.build_table()) == kind, (name, kind)
    return seq, o


def _inputs(o, lengths, seed, pinch=False):
    T = max(int(max(lengths)), 1)
    kp, fixed = SV.stream_inputs(o, len(lengths), T, seed, pinch=pinch)
    pk = np.concatenate([kp[s, :n] for s, n in enumerate(lengths)]).reshape(-1, 21, 3)
    pf = None if fixed is None else np.concatenate([fixed[s, :n] for s, n in enumerate(lengths)]).reshape(-1, fixed.shape[2])
    return pk, pf


def _causal(seq, o, pk, pf, lengths, seed):
    """The causal taped packed solve from a seeded state: (state before, tape)."""
    rng = np.random.RandomState(seed)
    st0 = fresh_state(seq, len(lengths))
    st0["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(len(lengths), o.opt_dof),
                                    o.joint_limits[:, 0], o.joint_limits[:, 1])
    st = {k: None if v is None else v.copy() for k, v in st0.items()}
    _, _, _, tape = P.solve_packed(seq, pk, P.offsets_of(lengths), state=st, fixed_qpos=pf, record=True)
    return st0, tape


def _smooth(seq, pk, pf, lengths, st0, qinit, anchor=True, **kw):
    return SM.smooth_packed(seq, pk, P.offsets_of(lengths), qinit, last_qpos=st0["last_qpos"] if anchor else None,
                            projected=st0["projected"], fixed_qpos=pf, **kw)


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _check_minimiser(models, q, cost, qinit, offs):
    for s, m in enumerate(models):
        a, b = offs[s], offs[s + 1]
        if b == a:
            continue
        X = q[a:b].astype(np.float64)
        Xp = m.polish(X)
        assert np.abs(Xp - X).max() <= SMC.PARITY, (s, np.abs(Xp - X).max())
        f = m.value(X)
        assert m.value(Xp) >= f - 1e-6 * abs(f), s
        assert cost[s] <= m.value(qinit[a:b]) * (1 + 1e-6), s  # descent from the start, in float64
        assert cost[s] == pytest.approx(f, rel=2e-5, abs=1e-9), s


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_answer_is_the_float64_minimiser(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    lengths = [5, 8]
    pk, pf = _inputs(o, lengths, 3)
    st0, tape = _causal(seq, o, pk, pf, lengths, 4)
    q, rq, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"])
    assert not (status & (STATUS_MAXITER | STATUS_NONFINITE | STATUS_MISSING)).any()
    offs = P.offsets_of(lengths)
    models = SMC.stream_models(o, pk, offs, pf, tape["projected"], SMC.clipped_anchor(o, st0["last_qpos"]), _nd(seq))
    _check_minimiser(models, q, cost, tape["qpos"], offs)
    # robot_qpos is the scatter + mimic of the answer (no filter)
    for i in range(len(q)):
        want = o.full_qpos(q[i].astype(np.float64), np.zeros(0) if pf is None else pf[i].astype(np.float64))
        np.testing.assert_allclose(rq[i], want, atol=1e-6)


@pytest.mark.parametrize("case", CASES[:4], ids=IDS[:4])
def test_without_an_anchor_and_at_the_bounds(case, tmp_path):
    """No anchor term; the start pushed onto the bounds of some variables (the active set decides which stay).  The Shadow
    hand on its free-flying base starts from the causal tape with max_iters = 1000: without an anchor its clip's placement
    lies in a valley where F changes by 5e-5 relative over 0.16 rad, and the method needs a few hundred accepted iterations
    there; F is checked for optimality, the position not (DESIGN.md 3.12)."""
    seq, o = _setup(case, tmp_path)
    lengths = [6]
    pk, pf = _inputs(o, lengths, 5)
    st0, tape = _causal(seq, o, pk, pf, lengths, 6)
    qinit = tape["qpos"].copy()
    lo, hi = np.float32(o.lower), np.float32(o.upper)
    gap = np.minimum(qinit[0] - lo, hi - qinit[0])
    prm = seq.optimizer.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    if case[0] == "shadow_position":
        prm.max_iters = 1000
    else:
        for j in np.argsort(gap)[:2]:  # the two variables nearest a bound start on it
            qinit[:, j] = lo[j] if qinit[0, j] - lo[j] < hi[j] - qinit[0, j] else hi[j]
    q, _, status, cost = _smooth(seq, pk, pf, lengths, st0, qinit, anchor=False, params=prm)
    assert not (status & STATUS_MAXITER).any()
    offs = P.offsets_of(lengths)
    models = SMC.stream_models(o, pk, offs, pf, tape["projected"], None, _nd(seq))
    if case[0] != "shadow_position":
        _check_minimiser(models, q, cost, qinit, offs)
        return
    # the valley is too flat for a displacement bar (F agrees to 1e-11 while the position moves by 1e-2 rad): optimality in F
    m, X = models[0], q.astype(np.float64)
    f = m.value(X)
    assert m.value(m.polish(X)) >= f - 1e-7 * f
    assert cost[0] <= m.value(qinit) * (1 + 1e-6)


@pytest.mark.parametrize("case", CASES[::2], ids=IDS[::2])
def test_reductions(case, tmp_path):
    """T = 1 streams are the single-frame minimisers with norm_delta = w and last_qpos = clip(a); with w = 0 and no anchor
    every frame is its own minimiser."""
    seq, o = _setup(case, tmp_path)
    lengths = [1, 1, 1]
    pk, pf = _inputs(o, lengths, 7)
    st0, tape = _causal(seq, o, pk, pf, lengths, 8)
    w = 2.5 * _nd(seq)
    q, _, _, _ = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], smooth_weight=w)
    offs = P.offsets_of(lengths)
    for s, m in enumerate(SMC.stream_models(o, pk, offs, pf, tape["projected"], SMC.clipped_anchor(o, st0["last_qpos"]), w)):
        X = q[s:s + 1].astype(np.float64)
        assert np.abs(m.polish(X) - X).max() <= SMC.PARITY
    lengths = [4]
    pk, pf = _inputs(o, lengths, 9)
    st0, tape = _causal(seq, o, pk, pf, lengths, 10)
    q, _, _, _ = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], anchor=False, smooth_weight=0.0)
    for t in range(4):
        m = SMC.Model(o, pk[t:t + 1], None if pf is None else pf[t:t + 1],
                      None if tape["projected"] is None else tape["projected"][t:t + 1], None, 0.0)
        X = q[t:t + 1].astype(np.float64)
        assert np.abs(m.polish(X) - X).max() <= SMC.PARITY, t


@pytest.mark.parametrize("case", CASES[:2] + CASES[4:], ids=IDS[:2] + IDS[4:])
def test_missing_frames_are_interpolated(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    T = 14
    pk, pf = _inputs(o, [T, T], 11)
    drop = np.array([0, 1, 5, 6, 7, 12, 13])  # leading, interior and trailing gaps
    pk[drop] = np.nan
    pk[T + 4] = np.nan  # the second stream, without an anchor run below, keeps a one-frame gap
    st0, tape = _causal(seq, o, pk, pf, [T, T], 12)
    q, _, status, _ = _smooth(seq, pk, pf, [T, T], st0, tape["qpos"])
    miss = np.zeros(2 * T, bool)
    miss[drop] = True
    miss[T + 4] = True
    np.testing.assert_array_equal((status & STATUS_MISSING) != 0, miss)
    q = q.astype(np.float64)
    a = SMC.clipped_anchor(o, st0["last_qpos"])
    np.testing.assert_allclose(q[0:2], SMC.interpolation(a[0], q[2], 2), atol=1e-5)
    np.testing.assert_allclose(q[5:8], SMC.interpolation(q[4], q[8], 3), atol=1e-5)
    np.testing.assert_allclose(q[12:14], SMC.interpolation(q[11], None, 2, has_next=False), atol=1e-5)
    np.testing.assert_allclose(q[T + 4:T + 5], SMC.interpolation(q[T + 3], q[T + 5], 1), atol=1e-5)
    # a leading gap without an anchor repeats the first observed frame
    q2, _, status2, _ = _smooth(seq, pk[:T], None if pf is None else pf[:T], [T], st0, tape["qpos"][:T], anchor=False)
    np.testing.assert_allclose(q2[0:2].astype(np.float64), SMC.interpolation(None, q2[2].astype(np.float64), 2, has_prev=False),
                               atol=1e-5)


def test_dexpilot_flags_that_switch(tmp_path):
    """A pinch switches the flags on at frame 1 and off at frame 3: the model held at the causal tape's flags agrees."""
    seq, o = _setup(CASES[1], tmp_path)
    lengths = [6]
    pk, pf = _inputs(o, lengths, 13, pinch=True)
    st0, tape = _causal(seq, o, pk, pf, lengths, 14)
    assert tape["projected"].any() and not tape["projected"].all()
    q, _, _, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"])
    offs = P.offsets_of(lengths)
    models = SMC.stream_models(o, pk, offs, pf, tape["projected"], SMC.clipped_anchor(o, st0["last_qpos"]), _nd(seq))
    _check_minimiser(models, q, cost, tape["qpos"], offs)


@pytest.mark.parametrize("case", CASES[1:2] + CASES[4:], ids=IDS[1:2] + IDS[4:])
def test_layout(case, tmp_path):
    """A stream's outputs are bit-identical alone and anywhere in a batch; lengths 0 and 1; a non-finite start."""
    seq, o = _setup(case, tmp_path)
    lengths = [3, 0, 1, 4]
    pk, pf = _inputs(o, lengths, 15)
    st0, tape = _causal(seq, o, pk, pf, lengths, 16)
    q, rq, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"])
    offs = P.offsets_of(lengths)
    assert np.isnan(cost[1])  # a stream of length 0 writes nothing
    for s in (0, 2, 3):
        a, b = offs[s], offs[s + 1]
        sub = {k: None if v is None else v[s:s + 1] for k, v in st0.items()}
        q1, rq1, st1, c1 = _smooth(seq, pk[a:b], None if pf is None else pf[a:b], [b - a], sub, tape["qpos"][a:b])
        np.testing.assert_array_equal(q1, q[a:b])
        np.testing.assert_array_equal(rq1, rq[a:b])
        np.testing.assert_array_equal(st1, status[a:b])
        np.testing.assert_array_equal(c1, cost[s:s + 1])
    # reversed batch order: the same bits
    order = [3, 2, 1, 0]
    rl = [lengths[s] for s in order]
    idx = np.concatenate([np.arange(offs[s], offs[s + 1]) for s in order]).astype(int)
    sub = {k: None if v is None else v[order] for k, v in st0.items()}
    qr, _, sr, cr = _smooth(seq, pk[idx], None if pf is None else pf[idx], rl, sub, tape["qpos"][idx])
    np.testing.assert_array_equal(qr, q[idx])
    np.testing.assert_array_equal(sr, status[idx])
    # a non-finite start: that stream gets qpos_init back and NONFINITE; the others are unchanged
    qinit = tape["qpos"].copy()
    qinit[offs[3] + 1, 0] = np.nan
    qn, _, sn, cn = _smooth(seq, pk, pf, lengths, st0, qinit)
    np.testing.assert_array_equal(qn[offs[3]:], qinit[offs[3]:])
    assert (sn[offs[3]:] == STATUS_NONFINITE).all() and np.isnan(cn[3])
    np.testing.assert_array_equal(qn[:offs[3]], q[:offs[3]])
    np.testing.assert_array_equal(sn[:offs[3]], status[:offs[3]])


def test_malformed_offsets_touch_nothing(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    pk, pf = _inputs(o, [4], 17)
    st0, tape = _causal(seq, o, pk, pf, [4], 18)
    st2 = {k: None if v is None else np.repeat(v, 3, axis=0) for k, v in st0.items()}
    bad = np.array([0, 5, 2, -1], np.int64)  # past N, decreasing, negative: every stream reads as empty
    q, rq, status, cost = SM.smooth_packed(seq, pk, bad, tape["qpos"], last_qpos=st2["last_qpos"], fixed_qpos=pf)
    assert np.isnan(q).all() and (status == -1).all() and np.isnan(cost).all()


def test_argument_checks(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    pk, pf = _inputs(o, [3], 19)
    st0, tape = _causal(seq, o, pk, pf, [3], 20)
    offs = P.offsets_of([3])

    def err(**kw):
        with pytest.raises(EmulationError) as e:
            SM.smooth_packed(seq, pk, offs, tape["qpos"], last_qpos=st0["last_qpos"], **kw)
        assert e.value.code == N_INVALID
        return e.value.msg

    assert "required" in err(null=("qpos_init",))
    assert "required" in err(null=("keypoints",))
    assert "required" in err(null=("qpos_out",))
    assert "offsets" in err(null=("offsets",))
    assert "workspace" in err(workspace_bytes=SM.workspace_bytes(seq, 3) - 4)
    assert "workspace" in err(null=("workspace",))
    assert "smooth_weight" in err(smooth_weight=float("nan"))
    prm = seq.optimizer.params(raw_hand=None)
    prm.preprocess = 1
    assert "preprocess" in err(params=prm)
    assert "sizes" in err(num_streams=-1)


def test_fixed_joints_are_required(tmp_path):
    seq, o = _setup(CASES[2], tmp_path)
    pk, pf = _inputs(o, [2], 21)
    assert pf is not None
    with pytest.raises(EmulationError, match="fixed"):
        SM.smooth_packed(seq, pk, P.offsets_of([2]), np.zeros((2, o.opt_dof), np.float32), null=("fixed_qpos",))


@pytest.mark.parametrize("case", [CASES[0], CASES[3]], ids=[IDS[0], IDS[3]])
def test_workspace_size(case, tmp_path):
    """(G^2 + 5 G) floats per frame, G the robot's lane count; the library reports the same."""
    seq, o = _setup(case, tmp_path)
    G = 16 if seq.optimizer.build_table().dof <= 16 else 32
    assert SM.workspace_bytes(seq, 10) == 10 * (G * G + 5 * G) * 4
    assert SM.workspace_bytes(seq, 0) == 0
    from dex_retargeting_b200 import _native as N

    lib = N.load()
    assert lib.dexr_smooth_workspace_bytes(None, 10) == 0


def test_smooth_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v`: both dexr_smooth_kernel instantiations spill nothing."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    smooth = {k: v for k, v in stores.items() if "dexr_smooth_kernel" in k}
    assert len(smooth) == 2, sorted(stores)
    assert all(v == 0 for v in smooth.values()), smooth


def test_gpu_smooth_file_passes_against_the_emulation():
    """tests/test_gpu_smooth.py dry-run on the CPU (tests/tools/emu_gpu_smooth.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_smooth.py")], capture_output=True,
                         text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
