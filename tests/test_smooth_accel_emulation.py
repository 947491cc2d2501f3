"""Offline smoothing with an acceleration penalty (`dexr_smooth_sequences_packed_accel` and its `_vjp`) through the host
emulation of the kernels' own code (tests/emu runs smooth_packed_stream<G, true> and smooth_vjp_packed_stream<G, true> of
dexr_kernels.cuh on the fiber warp), on the packaged configs (DexPilot included) and on structure cases at 16 and 32 lanes:
the float64 model of tests/smooth_accel_cases.py (minimiser, descent, the VJP), the model's own VJP against central
differences of re-polished minimisers, the penalty property, streams of 0-3 frames, missing frames, the stream layout,
c = 0 against the velocity-only smoother bit for bit, the argument checks, the workspace size, the register budget and a
dry run of tests/test_gpu_smooth_accel.py."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_packed_host as P
import emu_smooth_accel_host as AH
import emu_smooth_host as SM
import emu_smooth_vjp_host as SVH
import seq_vjp_cases as SV
import smooth_accel_cases as AC
import smooth_cases as SMC
import smooth_vjp_cases as SVC
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
    ("mimic_dense16", "<16,0>", "mimic_dense16"),  # the mimic fold reads other lanes' H_q columns
    ("shadow_position", "<32,-1>", ("offline/shadow_hand_right", None)),
    ("mimic_fixed_dense32", "<32,0>", "mimic_fixed_dense32"),
    ("prismatic_arrow", "<32,-1>", "prismatic_arrow"),
]
IDS = [c[0] for c in CASES]
BY_NAME = dict(zip(IDS, CASES))


def _pick(*names):
    """(cases, ids) for pytest.mark.parametrize."""
    return dict(argvalues=[BY_NAME[n] for n in names], ids=list(names))


NO_SHADOW = [n for n in IDS if n != "shadow_position"]
# the acceleration weight of most checks, in units of the robot's norm_delta (the velocity weight w by default)
C_REL = 5.0


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


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _smooth(seq, pk, pf, lengths, st0, qinit, c, anchor=True, **kw):
    return AH.smooth_packed(seq, pk, P.offsets_of(lengths), qinit, c, last_qpos=st0["last_qpos"] if anchor else None,
                            projected=st0["projected"], fixed_qpos=pf, **kw)


def _models(o, pk, pf, lengths, tape, st0, w, c, anchor=True):
    anch = SMC.clipped_anchor(o, st0["last_qpos"]) if anchor else None
    return AC.stream_models(o, pk, P.offsets_of(lengths), pf, tape["projected"], anch, w, c)


def _check_minimiser(models, q, cost, qinit, offs):
    for s, m in enumerate(models):
        a, b = offs[s], offs[s + 1]
        if b == a:
            continue
        X = q[a:b].astype(np.float64)
        Xp = m.polish(X)
        assert np.abs(Xp - X).max() <= AC.PARITY, (s, np.abs(Xp - X).max())
        f = m.value(X)
        assert m.value(Xp) >= f - 1e-6 * abs(f), s
        assert cost[s] <= m.value(qinit[a:b]) * (1 + 1e-6), s  # F_c does not rise above the start's (float64)
        assert cost[s] == pytest.approx(f, rel=2e-5, abs=1e-9), s


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_answer_is_the_float64_minimiser(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    lengths = [5, 8]
    pk, pf = _inputs(o, lengths, 3)
    st0, tape = _causal(seq, o, pk, pf, lengths, 4)
    c = C_REL * _nd(seq)
    q, rq, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], c)
    assert not (status & (STATUS_MAXITER | STATUS_NONFINITE | STATUS_MISSING)).any()
    offs = P.offsets_of(lengths)
    _check_minimiser(_models(o, pk, pf, lengths, tape, st0, _nd(seq), c), q, cost, tape["qpos"], offs)
    for i in range(len(q)):  # robot_qpos is the scatter + mimic of the answer (no filter)
        want = o.full_qpos(q[i].astype(np.float64), np.zeros(0) if pf is None else pf[i].astype(np.float64))
        np.testing.assert_allclose(rq[i], want, atol=1e-6)


@pytest.mark.parametrize("case", **_pick(*NO_SHADOW))
def test_without_an_anchor_and_at_the_bounds(case, tmp_path):
    """No anchor term (no triple before frame 1); the two variables nearest a bound start on it."""
    seq, o = _setup(case, tmp_path)
    lengths = [6]
    pk, pf = _inputs(o, lengths, 5)
    st0, tape = _causal(seq, o, pk, pf, lengths, 6)
    qinit = tape["qpos"].copy()
    lo, hi = np.float32(o.lower), np.float32(o.upper)
    gap = np.minimum(qinit[0] - lo, hi - qinit[0])
    for j in np.argsort(gap)[:2]:
        qinit[:, j] = lo[j] if qinit[0, j] - lo[j] < hi[j] - qinit[0, j] else hi[j]
    c = C_REL * _nd(seq)
    q, _, status, cost = _smooth(seq, pk, pf, lengths, st0, qinit, c, anchor=False)
    assert not (status & STATUS_MAXITER).any()
    _check_minimiser(_models(o, pk, pf, lengths, tape, st0, _nd(seq), c, anchor=False), q, cost, qinit,
                     P.offsets_of(lengths))


@pytest.mark.parametrize("case", **_pick("allegro_vector", "mimic_dense16", "mimic_fixed_dense32"))
def test_zero_velocity_weight(case, tmp_path):
    """w = 0 with c > 0: the acceleration term alone couples the frames."""
    seq, o = _setup(case, tmp_path)
    lengths = [6, 4]
    pk, pf = _inputs(o, lengths, 7)
    st0, tape = _causal(seq, o, pk, pf, lengths, 8)
    c = 2 * C_REL * _nd(seq)
    q, _, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], c, smooth_weight=0.0)
    assert not (status & STATUS_MAXITER).any()
    _check_minimiser(_models(o, pk, pf, lengths, tape, st0, 0.0, c), q, cost, tape["qpos"], P.offsets_of(lengths))


@pytest.mark.parametrize("anchor", [True, False], ids=["anchor", "no_anchor"])
@pytest.mark.parametrize("case", **_pick("allegro_vector", "leap_dexpilot", "mimic_fixed_dense32"))
def test_streams_of_zero_to_three_frames(case, anchor, tmp_path):
    """Lengths 0-3 follow from the definition: with an anchor a 2-frame stream has one triple, without one a stream needs 3
    frames for its first; a 0-frame stream writes nothing."""
    seq, o = _setup(case, tmp_path)
    lengths = [2, 0, 1, 3]
    pk, pf = _inputs(o, lengths, 9)
    st0, tape = _causal(seq, o, pk, pf, lengths, 10)
    c = 4 * C_REL * _nd(seq)
    q, _, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], c, anchor=anchor)
    assert np.isnan(cost[1])
    assert not (status & (STATUS_MAXITER | STATUS_NONFINITE)).any()
    models = _models(o, pk, pf, lengths, tape, st0, _nd(seq), c, anchor=anchor)
    assert [int(np.abs(m.D).sum(1).tolist().count(4.0)) for m in models] == ([1, 0, 0, 2] if anchor else [0, 0, 0, 1])
    _check_minimiser(models, q, cost, tape["qpos"], P.offsets_of(lengths))


@pytest.mark.parametrize("case", **_pick("allegro_vector", "leap_dexpilot", "mimic_fixed_dense32"))
def test_missing_frames_follow_the_model(case, tmp_path):
    """Leading, interior and trailing gaps: their values are what the smoothness terms give (the model with no data term
    there), which for c > 0 is not the linear interpolation."""
    seq, o = _setup(case, tmp_path)
    T = 12
    pk, pf = _inputs(o, [T], 11)
    drop = np.array([0, 1, 5, 6, 7, 11])
    pk[drop] = np.nan
    st0, tape = _causal(seq, o, pk, pf, [T], 12)
    c = C_REL * _nd(seq)
    q, _, status, cost = _smooth(seq, pk, pf, [T], st0, tape["qpos"], c)
    miss = np.zeros(T, bool)
    miss[drop] = True
    np.testing.assert_array_equal((status & STATUS_MISSING) != 0, miss)
    _check_minimiser(_models(o, pk, pf, [T], tape, st0, _nd(seq), c), q, cost, tape["qpos"], P.offsets_of([T]))
    q = q.astype(np.float64)
    assert np.abs(q[5:8] - SMC.interpolation(q[4], q[8], 3)).max() > 1e-4


@pytest.mark.parametrize("case", **_pick("leap_dexpilot", "mimic_fixed_dense32"))
def test_layout_and_nonfinite_isolation(case, tmp_path):
    """A stream's outputs are bit-identical alone and anywhere in a batch; a non-finite start changes only its stream."""
    seq, o = _setup(case, tmp_path)
    lengths = [3, 0, 1, 5]
    pk, pf = _inputs(o, lengths, 15)
    st0, tape = _causal(seq, o, pk, pf, lengths, 16)
    c = C_REL * _nd(seq)
    q, rq, status, cost = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], c)
    offs = P.offsets_of(lengths)
    for s in (0, 2, 3):
        a, b = offs[s], offs[s + 1]
        sub = {k: None if v is None else v[s:s + 1] for k, v in st0.items()}
        q1, rq1, st1, c1 = _smooth(seq, pk[a:b], None if pf is None else pf[a:b], [b - a], sub, tape["qpos"][a:b], c)
        np.testing.assert_array_equal(q1, q[a:b])
        np.testing.assert_array_equal(rq1, rq[a:b])
        np.testing.assert_array_equal(st1, status[a:b])
        np.testing.assert_array_equal(c1, cost[s:s + 1])
    qinit = tape["qpos"].copy()
    qinit[offs[3] + 1, 0] = np.nan
    qn, _, sn, cn = _smooth(seq, pk, pf, lengths, st0, qinit, c)
    np.testing.assert_array_equal(qn[offs[3]:], qinit[offs[3]:])
    assert (sn[offs[3]:] == STATUS_NONFINITE).all() and np.isnan(cn[3])
    np.testing.assert_array_equal(qn[:offs[3]], q[:offs[3]])
    np.testing.assert_array_equal(sn[:offs[3]], status[:offs[3]])
    # the VJP: a non-finite cotangent makes its stream NaN and NONFINITE, the others keep their bits
    gq = np.random.RandomState(17).randn(len(q), o.opt_dof).astype(np.float32)
    kw = dict(last_qpos=st0["last_qpos"], projected=st0["projected"], fixed_qpos=pf)
    g = AH.smooth_vjp_packed(seq, pk, offs, q, c, grad_qpos=gq, **kw)
    gq[offs[3] + 2, 1] = np.inf
    gn = AH.smooth_vjp_packed(seq, pk, offs, q, c, grad_qpos=gq, **kw)
    assert np.isnan(gn[0][offs[3]:]).all() and np.isnan(gn[2][3]).all() and (gn[3][offs[3]:] == STATUS_NONFINITE).all()
    np.testing.assert_array_equal(gn[0][:offs[3]], g[0][:offs[3]])
    np.testing.assert_array_equal(gn[2][:3], g[2][:3])


def test_malformed_offsets_touch_nothing(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    pk, pf = _inputs(o, [4], 17)
    st0, tape = _causal(seq, o, pk, pf, [4], 18)
    st2 = {k: None if v is None else np.repeat(v, 3, axis=0) for k, v in st0.items()}
    bad = np.array([0, 5, 2, -1], np.int64)  # past N, decreasing, negative: every stream reads as empty
    c = C_REL * _nd(seq)
    q, rq, status, cost = AH.smooth_packed(seq, pk, bad, tape["qpos"], c, last_qpos=st2["last_qpos"], fixed_qpos=pf)
    assert np.isnan(q).all() and (status == -1).all() and np.isnan(cost).all()
    g_kp, _, g_l, vst = AH.smooth_vjp_packed(seq, pk, bad, tape["qpos"], c, last_qpos=st2["last_qpos"], fixed_qpos=pf,
                                             grad_qpos=np.ones((4, o.opt_dof), np.float32))
    assert np.isnan(g_kp).all() and (vst == -1).all() and (g_l == 0).all()


@pytest.mark.parametrize("case", **_pick("allegro_vector", "leap_dexpilot", "mimic_fixed_dense32"))
def test_zero_accel_weight_is_the_smoother_bit_for_bit(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    lengths = [4, 6]
    pk, pf = _inputs(o, lengths, 19)
    st0, tape = _causal(seq, o, pk, pf, lengths, 20)
    offs = P.offsets_of(lengths)
    kw = dict(last_qpos=st0["last_qpos"], projected=st0["projected"], fixed_qpos=pf)
    want = SM.smooth_packed(seq, pk, offs, tape["qpos"], **kw)
    got = AH.smooth_packed(seq, pk, offs, tape["qpos"], 0.0, workspace_bytes=SM.workspace_bytes(seq, len(pk)), **kw)
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)
    gq = np.random.RandomState(21).randn(len(pk), o.opt_dof).astype(np.float32)
    want = SVH.smooth_vjp_packed(seq, pk, offs, want[0], grad_qpos=gq, **kw)
    got = AH.smooth_vjp_packed(seq, pk, offs, got[0], 0.0, grad_qpos=gq, **kw)
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)


def _vjp_run(seq, o, lengths, seed, c, anchor=True):
    pk, pf = _inputs(o, lengths, seed)
    st0, tape = _causal(seq, o, pk, pf, lengths, seed + 1)
    q, _, status, _ = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], c, anchor=anchor)
    rng = np.random.RandomState(seed + 2)
    gq = rng.randn(len(pk), o.opt_dof).astype(np.float32)
    grq = rng.randn(len(pk), seq.optimizer.robot.dof).astype(np.float32)
    last = st0["last_qpos"] if anchor else None
    res = AH.smooth_vjp_packed(seq, pk, P.offsets_of(lengths), q, c, last_qpos=last, projected=st0["projected"],
                               fixed_qpos=pf, grad_qpos=gq, grad_robot_qpos=grq)
    models = []
    offs = P.offsets_of(lengths)
    for s, m in enumerate(_models(o, pk, pf, lengths, tape, st0, _nd(seq), c, anchor=anchor)):
        a, b = offs[s], offs[s + 1]
        fl = None if tape["projected"] is None else tape["projected"][a:b]
        fx = None if pf is None else pf[a:b]
        models.append(AC.model_vjp(m, q[a:b], pk[a:b], fx, fl, None if last is None else last[s], gq[a:b], grq[a:b]))
    return res, models, offs, status


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_vjp_is_the_model(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    res, models, offs, status = _vjp_run(seq, o, [5, 3, 2], 23, C_REL * _nd(seq))
    assert not (status & STATUS_MAXITER).any()
    ratio, checked = SVC.compare(res, models, offs, tau=AC.TAU)
    assert checked >= 2, case
    if res[1].size:
        assert np.abs(res[1]).max() > 0


@pytest.mark.parametrize("case", **_pick("allegro_vector", "leap_dexpilot"))
def test_vjp_without_an_anchor_and_at_w0(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    res, models, offs, _ = _vjp_run(seq, o, [4, 3], 25, C_REL * _nd(seq), anchor=False)
    assert SVC.compare(res, models, offs, tau=AC.TAU)[1] >= 1
    assert res[2] is None


def _polished_loss(o, kp, fixed, flags, anchor, w, c, X0, gq):
    m = AC.Model(o, kp, fixed, flags, anchor, w, c)
    return float((m.polish(X0, iters=60) * gq).sum())


@pytest.mark.parametrize("case", **_pick("allegro_vector", "mimic_fixed_dense16"))
def test_vjp_model_against_central_differences(case, tmp_path):
    """l(X*) = <G, X*> with X* re-polished in float64 at theta +- h delta (keypoints, fixed joints, anchor): the model's
    cotangents give the same directional derivative.  The clips have variables at their bounds, held there by a gradient
    far above what the perturbation moves, so the active set stays."""
    seq, o = _setup(case, tmp_path)
    T = 4
    pk, pf = _inputs(o, [T], 35)
    st0, tape = _causal(seq, o, pk, pf, [T], 36)
    w, c = _nd(seq), C_REL * _nd(seq)
    anchor = SMC.clipped_anchor(o, st0["last_qpos"])[0]
    flags = tape["projected"]
    m = AC.Model(o, pk, pf, flags, anchor, w, c)
    X = m.polish(tape["qpos"].astype(np.float64), iters=60)
    rng = np.random.RandomState(29)
    gq = rng.randn(T, o.opt_dof)
    md = AC.model_vjp(m, X, pk, pf, flags, st0["last_qpos"][0], grad_qpos=gq)
    g = m.grad(X)
    act = ((X <= m.lo) & (g > -1e-7)) | ((X >= m.hi) & (g < 1e-7))
    assert not md["not_pd"] and md["n_active"] > 0 and np.abs(g[~act]).max() < 1e-9 and np.abs(g[act]).min() > 5e-4
    used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
    dk = np.zeros_like(pk, dtype=np.float64)
    dk[:, used] = rng.randn(T, len(used), 3)
    df = None if pf is None else rng.randn(*pf.shape)
    da = rng.randn(o.opt_dof)
    want = float((md["keypoints"] * dk).sum() + (md["last"] * da).sum() + (0.0 if df is None else (md["fixed"] * df).sum()))
    h = 1e-4
    kp64 = pk.astype(np.float64)
    f64 = None if pf is None else pf.astype(np.float64)
    lp = _polished_loss(o, kp64 + h * dk, None if pf is None else f64 + h * df, flags, anchor + h * da, w, c, X, gq)
    lm = _polished_loss(o, kp64 - h * dk, None if pf is None else f64 - h * df, flags, anchor - h * da, w, c, X, gq)
    got = (lp - lm) / (2 * h)
    assert got == pytest.approx(want, rel=2e-3, abs=1e-6), (got, want)


@pytest.mark.parametrize("case", **_pick("allegro_vector", "leap_dexpilot"))
def test_penalty_property(case, tmp_path):
    """sum |second difference|^2 at the answer does not increase as c grows (the model's minimisers and the emulation's
    answers, all in one basin: each is within the parity bar of the model's polish from it)."""
    seq, o = _setup(case, tmp_path)
    lengths = [8]
    pk, pf = _inputs(o, lengths, 31)
    st0, tape = _causal(seq, o, pk, pf, lengths, 32)
    nd = _nd(seq)
    emu_acc, model_acc = [], []
    for rel in (0.0, 1.0, 10.0, 100.0):
        q, _, _, _ = _smooth(seq, pk, pf, lengths, st0, tape["qpos"], rel * nd)
        m = _models(o, pk, pf, lengths, tape, st0, nd, rel * nd)[0]
        X = q.astype(np.float64)
        Xp = m.polish(X)
        assert np.abs(Xp - X).max() <= AC.PARITY
        emu_acc.append(m.accel_value(X))
        model_acc.append(m.accel_value(Xp))
    assert all(b <= a * (1 + 1e-6) for a, b in zip(model_acc, model_acc[1:])), model_acc
    assert all(b <= a * (1 + 1e-4) for a, b in zip(emu_acc, emu_acc[1:])), emu_acc
    assert model_acc[-1] < 0.5 * model_acc[0]


def test_argument_checks(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    pk, pf = _inputs(o, [3], 33)
    st0, tape = _causal(seq, o, pk, pf, [3], 34)
    offs = P.offsets_of([3])
    c = C_REL * _nd(seq)

    def err(fn, *a, **kw):
        with pytest.raises(EmulationError) as e:
            fn(*a, **kw)
        assert e.value.code == N_INVALID
        return e.value.msg

    fwd = lambda cc, **kw: AH.smooth_packed(seq, pk, offs, tape["qpos"], cc, last_qpos=st0["last_qpos"], **kw)  # noqa: E731
    bwd = lambda cc, **kw: AH.smooth_vjp_packed(seq, pk, offs, tape["qpos"], cc, last_qpos=st0["last_qpos"],  # noqa: E731
                                                grad_qpos=np.ones((3, o.opt_dof), np.float32), **kw)
    for fn in (fwd, bwd):
        for bad in (-1e-3, float("nan"), float("inf"), -float("inf")):
            assert "accel_weight" in err(fn, bad)
        assert "dexr_smooth_accel_workspace_bytes" in err(fn, c, workspace_bytes=AH.workspace_bytes(seq, 3) - 4)
        assert "workspace" in err(fn, c, workspace_bytes=SM.workspace_bytes(seq, 3))
        assert "workspace" in err(fn, c, null=("workspace",))
        assert "offsets" in err(fn, c, null=("offsets",))
        assert "sizes" in err(fn, c, num_streams=-1)
        assert "smooth_weight" in err(fn, c, smooth_weight=float("nan"))
        fn(0.0, workspace_bytes=SM.workspace_bytes(seq, 3))  # c = 0: the smoother's own workspace suffices
    assert "required" in err(fwd, c, null=("qpos_init",))
    assert "required" in err(bwd, c, null=("grad_keypoints",))


@pytest.mark.parametrize("case", **_pick("allegro_vector", "shadow_position"))
def test_workspace_size(case, tmp_path):
    """(2 G^2 + 5 G) floats per frame: the smoother's block and the coupling block E_t."""
    seq, o = _setup(case, tmp_path)
    G = 16 if seq.optimizer.build_table().dof <= 16 else 32
    assert AH.workspace_bytes(seq, 10) == 10 * (2 * G * G + 5 * G) * 4
    assert AH.workspace_bytes(seq, 10) >= SM.workspace_bytes(seq, 10)
    assert AH.workspace_bytes(seq, 0) == 0
    from dex_retargeting_b200 import _native as N

    assert N.load().dexr_smooth_accel_workspace_bytes(None, 10) == 0


def test_accel_kernels_register_budget(tmp_path):
    """`-Xptxas -v`: the four acceleration kernels; the 32-lane ones spill nothing, the 16-lane ones (128 registers under
    their launch bounds) at most 8 bytes of stores (DESIGN.md 3.16)."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    acc = {k: v for k, v in stores.items() if "dexr_smooth_accel" in k}
    assert len(acc) == 4, sorted(stores)
    for k, v in acc.items():
        assert v <= (8 if "ILi16E" in k else 0), (k, v)


def test_gpu_smooth_accel_file_passes_against_the_emulation():
    """tests/test_gpu_smooth_accel.py dry-run on the CPU (tests/tools/emu_gpu_smooth_accel.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_smooth_accel.py")], capture_output=True,
                         text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
