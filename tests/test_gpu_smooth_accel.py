"""Offline smoothing with an acceleration penalty on the GPU (`dexr_smooth_sequences_packed_accel` and its `_vjp` through
SeqRetargeting.smooth_packed_sequences(_vjp)(..., accel_weight=c) and objective.differentiable_smooth_packed_sequences): the
float64 model of tests/smooth_accel_cases.py on ragged LEAP DexPilot, Allegro vector and Shadow position clips
(tools/workloads.py `ragged_streams`) and on structure cases with fixed, mimic and prismatic joints; c = 0 against the
velocity-only calls bit for bit; stream bits independent of the neighbours and of S; the GPU against the host emulation;
autograd against the direct call; writes inside their buffers; asynchronous calls."""
import sys
from pathlib import Path

import numpy as np
import pytest

import smooth_accel_cases as AC
import smooth_cases as SMC
import smooth_vjp_cases as SVC
import structure_cases as SC
from helpers import build_oracle, build_product

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
STRUCTURES = ["fixed_dense16", "mimic_dense16", "mimic_fixed_dense32", "prismatic_arrow"]
# clips of the model check (lengths uniform over [LO, HI]) and how many of the shortest the float64 model checks.  The CPU
# dry run (tests/tools/emu_gpu_smooth_accel.py) shrinks them.
STREAMS, LO, HI = 24, 20, 40
CHECKED = 3
NEIGHBOURS = (48, 5, 30)  # clips and their length range of the layout checks
SENTINEL = 64  # rows of sentinels before and after every output block
C_REL = 5.0  # the acceleration weight, in units of the robot's norm_delta
STATUS_MAXITER, STATUS_NONFINITE, STATUS_NOT_PD = 1 << 24, 1 << 25, 1 << 26


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _fixed(o, Nf, seed):
    nf = len(o.idx_pin2fixed)
    if not nf:
        return None
    lim = o.robot.joint_limits[o.idx_pin2fixed]
    return np.random.RandomState(seed).uniform(lim[:, 0], lim[:, 1], size=(Nf, nf)).astype(np.float32)


def _c(seq):
    return C_REL * float(seq.optimizer.params().norm_delta)


def _run(seq, o, kp, lengths, fixed, seed, c):
    """The smoother with accel_weight c from the causal tape of a fresh state (anchor moved off the middle), then its VJP of
    seeded cotangents."""
    layout = seq.pack_streams(lengths)
    st = seq.make_stream_state(len(lengths))
    rng = np.random.RandomState(seed)
    lim = o.joint_limits
    st.last_qpos.copy_(_t(np.clip(lim.mean(1) + 0.1 * rng.randn(len(lengths), o.opt_dof), lim[:, 0], lim[:, 1])
                          .astype(np.float32)))
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(kp), layout, st.__class__(
        **{k: (None if getattr(st, k) is None else getattr(st, k).clone()) for k in st._FIELDS}), fixed_qpos=_t(fixed),
        tape=tape)
    rq, q, status = seq.smooth_packed_sequences(_t(kp), layout, st, fixed_qpos=_t(fixed), accel_weight=c)
    Nf = int(np.sum(lengths))
    gq = rng.randn(Nf, o.opt_dof).astype(np.float32)
    grq = rng.randn(Nf, seq.optimizer.robot.dof).astype(np.float32)
    vst = torch.empty(Nf, dtype=torch.int32, device=_dev())
    g_kp, g_f, g_l = seq.smooth_packed_sequences_vjp(_t(kp), layout, q, st.last_qpos, st.projected, _t(gq), _t(grq),
                                                     fixed_qpos=_t(fixed), status_out=vst, accel_weight=c)
    return dict(kp=kp, fixed=fixed, layout=layout, state=st, q=_np(q), rq=_np(rq), status=_np(status), gq=gq, grq=grq,
                qinit=_np(tape.qpos), flags=_np(tape.projected), res=(_np(g_kp), _np(g_f), _np(g_l), _np(vst)), c=c,
                offs=np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64))


def _model(seq, o, r, s):
    a, b = int(r["offs"][s]), int(r["offs"][s + 1])
    fl = None if r["flags"] is None else r["flags"][a:b]
    fx = None if r["fixed"] is None else r["fixed"][a:b]
    anch = SMC.clipped_anchor(o, _np(r["state"].last_qpos))
    return AC.Model(o, r["kp"][a:b], fx, fl, anch[s], float(seq.optimizer.params().norm_delta), r["c"])


def _check(seq, o, r, streams):
    """Forward: the float64 polish barely moves the answer, finds no lower F_c, and the answer descends from its start.
    Backward: the model's VJP at tau.  Returns the number of clips compared."""
    last = _np(r["state"].last_qpos)
    models = [None] * (len(r["offs"]) - 1)
    for s in streams:
        a, b = int(r["offs"][s]), int(r["offs"][s + 1])
        m = _model(seq, o, r, s)
        X = r["q"][a:b].astype(np.float64)
        Xp = m.polish(X)
        assert np.abs(Xp - X).max() <= AC.PARITY, (s, np.abs(Xp - X).max())
        f = m.value(X)
        assert m.value(Xp) >= f - 1e-6 * abs(f), s
        assert f <= m.value(r["qinit"][a:b]) * (1 + 1e-6), s
        fl = None if r["flags"] is None else r["flags"][a:b]
        fx = None if r["fixed"] is None else r["fixed"][a:b]
        models[s] = AC.model_vjp(m, r["q"][a:b], r["kp"][a:b], fx, fl, last[s], r["gq"][a:b], r["grq"][a:b])
    return SVC.compare(r["res"], models, r["offs"], tau=AC.TAU)


def _maxiter(r, s):
    return bool(r["status"][r["offs"][s]] & STATUS_MAXITER)


@pytest.mark.parametrize("key", KEYS)
def test_matches_the_model_on_ragged_clips(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(STREAMS, LO, HI, 41)
    r = _run(seq, o, kp, lengths, _fixed(o, int(lengths.sum()), 1), 42, _c(seq))
    assert not (r["status"] & STATUS_NONFINITE).any() and not (r["res"][3] & STATUS_NONFINITE).any()
    cand = [s for s in np.argsort(lengths, kind="stable")
            if not _maxiter(r, s) and not (r["res"][3][r["offs"][s]] & STATUS_NOT_PD)]
    ratio, checked = _check(seq, o, r, cand[:CHECKED])
    assert checked >= 1, key
    print(f"{key}: worst {ratio:.3f} of tau over {checked} clips")


@pytest.mark.parametrize("case", STRUCTURES)
def test_matches_the_model_on_structure_cases(case, tmp_path):
    seq, o = SC.build(SC.BY_ID[case], tmp_path)
    lengths = np.array([4, 7, 2], np.int64)
    kp, _ = W.ragged_streams(3, 7, 7, 43)
    kp = np.concatenate([kp[int(o_):int(o_) + int(n)] for o_, n in zip(np.arange(3) * 7, lengths)])
    fixed = _fixed(o, int(lengths.sum()), 2)
    r = _run(seq, o, kp, lengths, fixed, 44, _c(seq))
    ratio, checked = _check(seq, o, r, [s for s in range(3) if not _maxiter(r, s)])
    assert checked >= 1, case
    if fixed is not None:
        assert np.abs(r["res"][1]).max() > 0
    print(f"{case}: worst {ratio:.3f} of tau over {checked} clips")


@pytest.mark.parametrize("key", KEYS)
def test_zero_accel_weight_is_the_smoother_bit_for_bit(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(6, 5, 20, 45)
    fixed = _fixed(o, int(lengths.sum()), 3)
    r = _run(seq, o, kp, lengths, fixed, 46, 0.0)
    st = r["state"]
    rq, q, status = seq.smooth_packed_sequences(_t(kp), r["layout"], st, fixed_qpos=_t(fixed))
    for got, want in zip((r["rq"], r["q"], r["status"]), (rq, q, status)):
        np.testing.assert_array_equal(got, _np(want))
    vst = torch.empty(len(kp), dtype=torch.int32, device=_dev())
    g = seq.smooth_packed_sequences_vjp(_t(kp), r["layout"], q, st.last_qpos, st.projected, _t(r["gq"]), _t(r["grq"]),
                                        fixed_qpos=_t(fixed), status_out=vst)
    for got, want in zip(r["res"], tuple(g) + (vst,)):
        if want is not None:
            np.testing.assert_array_equal(got, _np(want))


@pytest.mark.parametrize("key", KEYS)
def test_stream_bits_do_not_depend_on_packing(key):
    """A stream's forward and backward bits are the same alone (S = 1) and among its neighbours."""
    seq, o = build_product(key, device=0), build_oracle(key)
    S, lo, hi = NEIGHBOURS
    kp, lengths = W.ragged_streams(S, lo, hi, 47)
    whole = _run(seq, o, kp, lengths, _fixed(o, int(lengths.sum()), 4), 48, _c(seq))
    offs = whole["offs"]
    for s in (0, S // 3, S - 1):
        a, b = offs[s], offs[s + 1]
        lay = seq.pack_streams(lengths[s:s + 1])
        fx = None if whole["fixed"] is None else whole["fixed"][a:b]
        st = whole["state"]
        sub = st.__class__(**{k: (None if getattr(st, k) is None else getattr(st, k)[s:s + 1].clone()) for k in st._FIELDS})
        rq, q, status = seq.smooth_packed_sequences(_t(kp[a:b]), lay, sub, fixed_qpos=_t(fx), qpos_init=_t(whole["qinit"][a:b]),
                                                    accel_weight=whole["c"])
        np.testing.assert_array_equal(_np(q), whole["q"][a:b])
        np.testing.assert_array_equal(_np(status), whole["status"][a:b])
        g = seq.smooth_packed_sequences_vjp(_t(kp[a:b]), lay, _t(whole["q"][a:b]), st.last_qpos[s:s + 1],
                                            None if st.projected is None else st.projected[s:s + 1],
                                            _t(whole["gq"][a:b]), _t(whole["grq"][a:b]), fixed_qpos=_t(fx),
                                            accel_weight=whole["c"])
        np.testing.assert_array_equal(_np(g[0]), whole["res"][0][a:b])
        np.testing.assert_array_equal(_np(g[2])[0], whole["res"][2][s])


@pytest.mark.parametrize("key", KEYS[:2])
def test_gpu_matches_the_emulation(key):
    import emu_smooth_accel_host as AH

    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(3, 4, 8, 49)
    r = _run(seq, o, kp, lengths, None, 50, _c(seq))
    last, proj = _np(r["state"].last_qpos), _np(r["state"].projected)
    q, _, status, _ = AH.smooth_packed(seq, kp, r["offs"], r["qinit"], r["c"], last_qpos=last, projected=proj)
    np.testing.assert_array_equal(status >> 24, r["status"] >> 24)  # the verdict bits; iteration counts may differ
    assert np.abs(q - r["q"]).max() <= 1e-4
    emu = AH.smooth_vjp_packed(seq, kp, r["offs"], r["q"], r["c"], last_qpos=last, projected=proj, grad_qpos=r["gq"],
                               grad_robot_qpos=r["grq"])
    np.testing.assert_array_equal(emu[3], r["res"][3])
    for s in range(len(lengths)):
        a, b = r["offs"][s], r["offs"][s + 1]
        assert SVC.stream_errors(r["res"][0][a:b], emu[0][a:b]) <= 1e-3, s
        assert SVC.stream_errors(r["res"][2][s], emu[2][s]) <= 1e-3, s


@pytest.mark.parametrize("key", KEYS[1:])
def test_autograd_is_the_direct_call(key):
    from dex_retargeting_b200.objective import differentiable_smooth_packed_sequences

    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(4, 10, 20, 51)
    fixed = _fixed(o, int(lengths.sum()), 5)
    r = _run(seq, o, kp, lengths, fixed, 52, _c(seq))
    kpt = _t(kp).requires_grad_(True)
    st = r["state"]
    last = st.last_qpos.clone().requires_grad_(True)
    view = st.__class__(last_qpos=last, filter_state=st.filter_state, filter_init=st.filter_init, projected=st.projected,
                        damping=st.damping)
    rq, q, status = differentiable_smooth_packed_sequences(seq, kpt, r["layout"], view, fixed_qpos=_t(fixed),
                                                           accel_weight=r["c"])
    np.testing.assert_array_equal(_np(q), r["q"])
    ((rq * _t(r["grq"])).sum() + (q * _t(r["gq"])).sum()).backward()
    np.testing.assert_array_equal(_np(kpt.grad), r["res"][0])
    np.testing.assert_array_equal(_np(last.grad), r["res"][2])
    with pytest.raises(ValueError, match="accel_weight"):
        differentiable_smooth_packed_sequences(seq, kpt, r["layout"], view,
                                               accel_weight=torch.tensor(r["c"], requires_grad=True))


def test_writes_stay_inside_their_buffers():
    """Every output is a view with SENTINEL rows before and after it: the sentinels survive, and a zero-length stream's
    anchor row is 0."""
    seq, o = build_product(KEYS[1], device=0), build_oracle(KEYS[1])
    kp, lengths = W.ragged_streams(5, 3, 9, 53)
    lengths[2] = 0
    kp = kp[:int(lengths.sum())]
    r = _run(seq, o, kp, lengths, None, 54, _c(seq))
    Nf, S, n, dof = int(lengths.sum()), len(lengths), o.opt_dof, seq.optimizer.robot.dof

    def framed(shape, dtype=torch.float32):
        big = torch.full((SENTINEL * 2 + shape[0],) + tuple(shape[1:]), -7, dtype=dtype, device=_dev())
        return big, big[SENTINEL:SENTINEL + shape[0]]

    bo, vo = framed((Nf, dof))
    bs, vs = framed((Nf,), torch.int32)
    st = r["state"]
    seq.smooth_packed_sequences(_t(kp), r["layout"], st, qpos_init=_t(r["qinit"]), accel_weight=r["c"], out=vo,
                                status_out=vs)
    bk, vk = framed((Nf, 21, 3))
    bl, vl = framed((S, n))
    seq.smooth_packed_sequences_vjp(_t(kp), r["layout"], _t(r["q"]), st.last_qpos, st.projected, _t(r["gq"]),
                                    _t(r["grq"]), accel_weight=r["c"], grad_keypoints_out=vk, grad_last_qpos_out=vl)
    for big in (bo, bs, bk, bl):
        b = _np(big)
        assert (b[:SENTINEL] == -7).all() and (b[-SENTINEL:] == -7).all()
    np.testing.assert_array_equal(_np(vo), r["rq"])
    np.testing.assert_array_equal(_np(vs), r["status"])
    np.testing.assert_array_equal(_np(vk), r["res"][0])
    assert (_np(vl)[2] == 0).all()


def test_calls_are_asynchronous():
    seq, o = build_product(KEYS[1], device=0), build_oracle(KEYS[1])
    kp, lengths = W.ragged_streams(64, 20, 40, 55)
    r = _run(seq, o, kp, lengths, None, 56, _c(seq))
    st = r["state"]
    for call in (lambda: seq.smooth_packed_sequences(_t(kp), r["layout"], st, qpos_init=_t(r["qinit"]), accel_weight=r["c"]),
                 lambda: seq.smooth_packed_sequences_vjp(_t(kp), r["layout"], _t(r["q"]), st.last_qpos, st.projected,
                                                         _t(r["gq"]), _t(r["grq"]), accel_weight=r["c"])):
        torch.cuda.synchronize()
        torch.cuda._sleep(200_000_000)  # keep the stream busy: a synchronising call would wait for it
        e = torch.cuda.Event()
        call()
        e.record()
        assert not e.query()
        torch.cuda.synchronize()
