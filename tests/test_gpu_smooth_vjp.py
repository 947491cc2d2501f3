"""Backpropagation through the offline smoother on the GPU (`dexr_smooth_sequences_packed_vjp` through
SeqRetargeting.smooth_packed_sequences_vjp and objective.differentiable_smooth_packed_sequences): the float64 model of
tests/smooth_vjp_cases.py on ragged LEAP DexPilot, Allegro vector and Shadow position clips (tools/workloads.py
`ragged_streams`) and on structure cases with fixed, mimic and prismatic joints; the GPU against the host emulation; autograd
against the direct call bit for bit; stream bits independent of packing; writes inside their buffers; an asynchronous call."""
import sys
from pathlib import Path

import numpy as np
import pytest

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
# dry run (tests/tools/emu_gpu_smooth_vjp.py) shrinks them.
STREAMS, LO, HI = 24, 20, 60
CHECKED = 3
NEIGHBOURS = (48, 5, 30)  # clips and their length range of the layout checks
SENTINEL = 64  # rows of sentinels before and after every output block


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


def _run(seq, o, kp, lengths, fixed, seed):
    """The smoother from the causal tape of a fresh state (anchor moved off the middle), then its VJP of seeded cotangents."""
    layout = seq.pack_streams(lengths)
    st = seq.make_stream_state(len(lengths))
    rng = np.random.RandomState(seed)
    lim = o.joint_limits
    st.last_qpos.copy_(_t(np.clip(lim.mean(1) + 0.1 * rng.randn(len(lengths), o.opt_dof), lim[:, 0], lim[:, 1])
                          .astype(np.float32)))
    rq, q, status = seq.smooth_packed_sequences(_t(kp), layout, st, fixed_qpos=_t(fixed))
    Nf = int(np.sum(lengths))
    gq = rng.randn(Nf, o.opt_dof).astype(np.float32)
    grq = rng.randn(Nf, seq.optimizer.robot.dof).astype(np.float32)
    vst = torch.empty(Nf, dtype=torch.int32, device=_dev())
    g_kp, g_f, g_l = seq.smooth_packed_sequences_vjp(_t(kp), layout, q, st.last_qpos, st.projected, _t(gq), _t(grq),
                                                     fixed_qpos=_t(fixed), status_out=vst)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(kp), layout, seq.make_stream_state(len(lengths)).__class__(
        **{k: (None if getattr(st, k) is None else getattr(st, k).clone()) for k in st._FIELDS}), fixed_qpos=_t(fixed),
        tape=tape)
    return dict(kp=kp, fixed=fixed, layout=layout, state=st, q=_np(q), status=_np(status), gq=gq, grq=grq,
                flags=_np(tape.projected), res=(_np(g_kp), _np(g_f), _np(g_l), _np(vst)),
                offs=np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64))


def _models(seq, o, r, streams):
    nd = float(seq.optimizer.params().norm_delta)
    last = _np(r["state"].last_qpos)
    anch = SMC.clipped_anchor(o, last)
    out = [None] * (len(r["offs"]) - 1)
    for s in streams:
        a, b = int(r["offs"][s]), int(r["offs"][s + 1])
        fl = None if r["flags"] is None else r["flags"][a:b]
        fx = None if r["fixed"] is None else r["fixed"][a:b]
        m = SMC.Model(o, r["kp"][a:b], fx, fl, anch[s], nd)
        out[s] = SVC.model_stream(m, r["q"][a:b], r["kp"][a:b], fx, fl, last[s], r["gq"][a:b], r["grq"][a:b])
    return out


def _maxiter(r, s):
    return bool(r["status"][r["offs"][s]] & (1 << 24))


@pytest.mark.parametrize("key", KEYS)
def test_matches_the_model_on_ragged_clips(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(STREAMS, LO, HI, 21)
    fixed = _fixed(o, int(lengths.sum()), 1)
    r = _run(seq, o, kp, lengths, fixed, 22)
    st = r["res"][3]
    assert not (st & SVC.STATUS_NONFINITE).any()
    cand = [s for s in np.argsort(lengths, kind="stable") if not _maxiter(r, s) and not (st[r["offs"][s]] & SVC.STATUS_NOT_PD)]
    ratio, checked = SVC.compare(r["res"], _models(seq, o, r, cand[:CHECKED]), r["offs"])
    assert checked >= 1, key
    print(f"{key}: worst {ratio:.3f} of tau over {checked} clips")


@pytest.mark.parametrize("case", STRUCTURES)
def test_matches_the_model_on_structure_cases(case, tmp_path):
    seq, o = SC.build(SC.BY_ID[case], tmp_path)
    lengths = np.array([4, 7, 6], np.int64)
    kp, _ = W.ragged_streams(3, 7, 7, 23)
    kp = np.concatenate([kp[int(o_):int(o_) + int(n)] for o_, n in zip(np.arange(3) * 7, lengths)])
    fixed = _fixed(o, int(lengths.sum()), 2)
    r = _run(seq, o, kp, lengths, fixed, 24)
    ratio, checked = SVC.compare(r["res"], _models(seq, o, r, [s for s in range(3) if not _maxiter(r, s)]), r["offs"])
    assert checked >= 1, case
    if fixed is not None:
        assert np.abs(r["res"][1]).max() > 0
    print(f"{case}: worst {ratio:.3f} of tau over {checked} clips")


@pytest.mark.parametrize("key", KEYS[:2])
def test_gpu_matches_the_emulation(key):
    import emu_smooth_vjp_host as SVH

    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(3, 4, 8, 25)
    r = _run(seq, o, kp, lengths, None, 26)
    emu = SVH.smooth_vjp_packed(seq, kp, r["offs"], r["q"], last_qpos=_np(r["state"].last_qpos),
                                projected=_np(r["state"].projected), grad_qpos=r["gq"], grad_robot_qpos=r["grq"])
    np.testing.assert_array_equal(emu[3], r["res"][3])
    for s in range(len(lengths)):
        a, b = r["offs"][s], r["offs"][s + 1]
        assert SVC.stream_errors(r["res"][0][a:b], emu[0][a:b]) <= 1e-3, s
        assert SVC.stream_errors(r["res"][2][s], emu[2][s]) <= 1e-3, s


@pytest.mark.parametrize("key", KEYS[1:])
def test_autograd_is_the_direct_call(key):
    from dex_retargeting_b200.objective import differentiable_smooth_packed_sequences

    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(4, 10, 20, 27)
    fixed = _fixed(o, int(lengths.sum()), 3)
    r = _run(seq, o, kp, lengths, fixed, 28)
    kpt = _t(kp).requires_grad_(True)
    st = r["state"]
    last = st.last_qpos.clone().requires_grad_(True)
    view = st.__class__(last_qpos=last, filter_state=st.filter_state, filter_init=st.filter_init, projected=st.projected,
                        damping=st.damping)
    rq, q, status = differentiable_smooth_packed_sequences(seq, kpt, r["layout"], view, fixed_qpos=_t(fixed))
    np.testing.assert_array_equal(_np(q), r["q"])
    ((rq * _t(r["grq"])).sum() + (q * _t(r["gq"])).sum()).backward()
    np.testing.assert_array_equal(_np(kpt.grad), r["res"][0])
    np.testing.assert_array_equal(_np(last.grad), r["res"][2])
    with pytest.raises(ValueError, match="qpos_init"):
        differentiable_smooth_packed_sequences(seq, kpt, r["layout"], view, qpos_init=q.detach().clone().requires_grad_(True))


@pytest.mark.parametrize("key", KEYS)
def test_stream_bits_do_not_depend_on_packing(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    S, lo, hi = NEIGHBOURS
    kp, lengths = W.ragged_streams(S, lo, hi, 29)
    whole = _run(seq, o, kp, lengths, _fixed(o, int(lengths.sum()), 4), 30)
    offs = whole["offs"]
    for s in (0, S // 3, S - 1):
        a, b = offs[s], offs[s + 1]
        lay = seq.pack_streams(lengths[s:s + 1])
        fx = None if whole["fixed"] is None else whole["fixed"][a:b]
        g = seq.smooth_packed_sequences_vjp(_t(kp[a:b]), lay, _t(whole["q"][a:b]), whole["state"].last_qpos[s:s + 1],
                                            None if whole["state"].projected is None else whole["state"].projected[s:s + 1],
                                            _t(whole["gq"][a:b]), _t(whole["grq"][a:b]), fixed_qpos=_t(fx))
        np.testing.assert_array_equal(_np(g[0]), whole["res"][0][a:b])
        np.testing.assert_array_equal(_np(g[2])[0], whole["res"][2][s])


def test_writes_stay_inside_their_buffers():
    """Every output is a view with SENTINEL rows before and after it: the sentinels survive, and a zero-length stream's
    anchor row is 0."""
    seq, o = build_product(KEYS[1], device=0), build_oracle(KEYS[1])
    kp, lengths = W.ragged_streams(5, 3, 9, 31)
    lengths[2] = 0
    r = _run(seq, o, kp[:int(lengths.sum())], lengths, None, 32)
    Nf, S, n = int(lengths.sum()), len(lengths), o.opt_dof

    def framed(shape):
        big = torch.full((SENTINEL * 2 + shape[0],) + tuple(shape[1:]), -7.0, device=_dev())
        return big, big[SENTINEL:SENTINEL + shape[0]]

    bk, vk = framed((Nf, 21, 3))
    bl, vl = framed((S, n))
    st = r["state"]
    seq.smooth_packed_sequences_vjp(_t(r["kp"]), r["layout"], _t(r["q"]), st.last_qpos, st.projected, _t(r["gq"]),
                                    _t(r["grq"]), grad_keypoints_out=vk, grad_last_qpos_out=vl)
    for big in (bk, bl):
        b = _np(big)
        assert (b[:SENTINEL] == -7.0).all() and (b[-SENTINEL:] == -7.0).all()
    np.testing.assert_array_equal(_np(vk), r["res"][0])
    assert (_np(vl)[2] == 0).all()


def test_call_is_asynchronous():
    seq, o = build_product(KEYS[1], device=0), build_oracle(KEYS[1])
    kp, lengths = W.ragged_streams(64, 20, 40, 33)
    r = _run(seq, o, kp, lengths, None, 34)
    args = (_t(kp), r["layout"], _t(r["q"]), r["state"].last_qpos, r["state"].projected, _t(r["gq"]), _t(r["grq"]))
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)  # keep the stream busy: a synchronising call would wait for it
    e = torch.cuda.Event()
    seq.smooth_packed_sequences_vjp(*args)
    e.record()
    assert not e.query()
    torch.cuda.synchronize()
