"""Offline smoothing on the GPU (`dexr_smooth_sequences_packed` through SeqRetargeting.smooth_packed_sequences) on LEAP
DexPilot, Allegro vector and Shadow position ragged clips (tools/workloads.py `ragged_streams`): the float64 model's polish
(tests/smooth_cases.py) barely moves the answer and finds no lower F, the answer descends from its start, almost no clip
ends at max_iters, the default start is the causal tape, a one-frame clip is
the single-frame minimiser, dropped frames are interpolated, a stream's bits do not depend on its neighbours, the call is
asynchronous, and equal-length clips started from dexr_solve_sequences tapes give the packed tapes' answers."""
import sys
from pathlib import Path

import numpy as np
import pytest

import smooth_cases as SMC
from helpers import build_oracle, build_product

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
# clips of the ragged check (lengths uniform over [LO, HI]) and how many of them the float64 model checks.  The CPU dry run
# (tests/tools/emu_gpu_smooth.py) shrinks them.
STREAMS, LO, HI = 256, 20, 60
CHECKED = 3
MAXITER_FRACTION = 0.01  # clips allowed to end at max_iters
NEIGHBOURS = (64, 5, 30)  # clips and their length range of the layout check
RECT_SIZE = (32, 24)  # streams x frames of the equal-length check
STATUS_MISSING, STATUS_NONFINITE, STATUS_MAXITER = 1 << 27, 1 << 25, 1 << 24


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _fixed(o, Nf, seed):
    """Fixed joints inside their limits (the oracle's), or None."""
    nf = len(o.idx_pin2fixed)
    if not nf:
        return None
    lim = o.robot.joint_limits[o.idx_pin2fixed]
    return np.random.RandomState(seed).uniform(lim[:, 0], lim[:, 1], size=(Nf, nf)).astype(np.float32)


def _run(seq, kp, lengths, fixed=None, drop=None):
    """Causal taped solve from a fresh state, then the smoother from its tape.  `drop`: frames set to NaN before both."""
    kp = kp.copy()
    if drop is not None:
        kp[drop] = np.nan
    layout = seq.pack_streams(lengths)
    st = seq.make_stream_state(len(lengths))
    tape = seq.make_packed_sequence_tape(layout)
    st_run = seq.make_stream_state(len(lengths))
    seq.retarget_packed_sequences(_t(kp), layout, st_run, fixed_qpos=_t(fixed), tape=tape)
    rq, q, status = seq.smooth_packed_sequences(_t(kp), layout, st, fixed_qpos=_t(fixed), qpos_init=tape.qpos)
    return dict(kp=kp, layout=layout, state=st, tape_q=_np(tape.qpos), tape_p=_np(tape.projected), rq=_np(rq), q=_np(q),
                status=_np(status))


def _models(seq, o, r, fixed, streams):
    nd = float(seq.optimizer.params().norm_delta)
    offs = np.concatenate([[0], np.cumsum(r["layout"].lengths)])
    anch = SMC.clipped_anchor(o, _np(r["state"].last_qpos))
    out = []
    for s in streams:
        a, b = offs[s], offs[s + 1]
        m = SMC.Model(o, r["kp"][a:b], None if fixed is None else fixed[a:b],
                      None if r["tape_p"] is None else r["tape_p"][a:b], anch[s], nd)
        out.append((s, a, b, m))
    return out


@pytest.mark.parametrize("key", KEYS)
def test_minimiser_and_descent(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(STREAMS, LO, HI, 11)
    fixed = _fixed(o, int(lengths.sum()), 1)
    r = _run(seq, kp, lengths, fixed)
    assert np.isfinite(r["q"]).all() and not (r["status"] & STATUS_NONFINITE).any()
    offs = np.concatenate([[0], np.cumsum(lengths)])
    assert ((r["status"][offs[:-1]] & STATUS_MAXITER) != 0).mean() <= MAXITER_FRACTION, key
    rng = np.random.RandomState(0)
    for s, a, b, m in _models(seq, o, r, fixed, rng.choice(len(lengths), CHECKED, replace=False)):
        X = r["q"][a:b].astype(np.float64)
        f, f0 = m.value(X), m.value(r["tape_q"][a:b])
        assert f <= f0 * (1 + 1e-6), (key, s, f, f0)  # descent from the causal start
        Xp = m.polish(X)
        assert np.abs(Xp - X).max() <= SMC.PARITY, (key, s, np.abs(Xp - X).max())
        assert m.value(Xp) >= f - 1e-6 * abs(f), (key, s, f)


@pytest.mark.parametrize("key", KEYS[:2])
def test_default_start_is_the_causal_tape(key):
    """qpos_init None: the call runs the taped causal solve on a copy of the state and starts from its tape."""
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, lengths = W.ragged_streams(NEIGHBOURS[0], NEIGHBOURS[1], NEIGHBOURS[2], 15)
    r = _run(seq, kp, lengths)
    st = seq.make_stream_state(len(lengths))
    before = _np(st.last_qpos).copy()
    rq, q, status = seq.smooth_packed_sequences(_t(kp), r["layout"], st)
    np.testing.assert_array_equal(_np(q), r["q"])
    np.testing.assert_array_equal(_np(rq), r["rq"])
    np.testing.assert_array_equal(_np(status), r["status"])
    np.testing.assert_array_equal(_np(st.last_qpos), before)  # the state is read only


@pytest.mark.parametrize("key", KEYS)
def test_one_frame_clip_is_the_frame_minimiser(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, _ = W.ragged_streams(1, 8, 8, 5)
    lengths = np.ones(8, np.int64)
    fixed = _fixed(o, 8, 2)
    r = _run(seq, kp, lengths, fixed)
    for s, a, b, m in _models(seq, o, r, fixed, range(8)):
        X = r["q"][a:b].astype(np.float64)
        assert np.abs(m.polish(X) - X).max() <= SMC.PARITY, (key, s)


@pytest.mark.parametrize("key", KEYS)
def test_dropped_frames_are_interpolated(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    kp, _ = W.ragged_streams(1, 40, 40, 6)
    lengths = np.array([40], np.int64)
    drop = np.r_[0:3, 17:21, 36:40]  # leading, interior and trailing gaps
    fixed = _fixed(o, 40, 3)
    r = _run(seq, kp, lengths, fixed, drop=drop)
    miss = np.zeros(40, bool)
    miss[drop] = True
    np.testing.assert_array_equal((r["status"] & STATUS_MISSING) != 0, miss)
    q = r["q"].astype(np.float64)
    anchor = SMC.clipped_anchor(o, _np(r["state"].last_qpos))[0]
    np.testing.assert_allclose(q[17:21], SMC.interpolation(q[16], q[21], 4), atol=1e-5)
    np.testing.assert_allclose(q[36:40], SMC.interpolation(q[35], None, 4, has_next=False), atol=1e-5)
    np.testing.assert_allclose(q[0:3], SMC.interpolation(anchor, q[3], 3), atol=1e-5)


@pytest.mark.parametrize("key", KEYS)
def test_stream_bits_do_not_depend_on_neighbours(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    S, lo, hi = NEIGHBOURS
    kp, lengths = W.ragged_streams(S, lo, hi, 12)
    fixed = _fixed(o, int(lengths.sum()), 4)
    whole = _run(seq, kp, lengths, fixed)
    offs = np.concatenate([[0], np.cumsum(lengths)])
    for s in (0, S // 3, S - 1):
        a, b = offs[s], offs[s + 1]
        alone = _run(seq, kp[a:b], lengths[s:s + 1], None if fixed is None else fixed[a:b])
        np.testing.assert_array_equal(alone["q"], whole["q"][a:b])
        np.testing.assert_array_equal(alone["status"], whole["status"][a:b])


def test_call_is_asynchronous():
    seq = build_product(KEYS[1], device=0)
    kp, lengths = W.ragged_streams(64, 20, 40, 13)
    layout = seq.pack_streams(lengths)
    st = seq.make_stream_state(64)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(kp), layout, seq.make_stream_state(64), tape=tape)
    kpt = _t(kp)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)  # keep the stream busy: a synchronising call would wait for it
    e = torch.cuda.Event()
    seq.smooth_packed_sequences(kpt, layout, st, qpos_init=tape.qpos)
    e.record()
    assert not e.query()
    torch.cuda.synchronize()


@pytest.mark.parametrize("key", KEYS)
def test_rectangular_tapes_give_the_packed_answers(key):
    seq, o = build_product(key, device=0), build_oracle(key)
    S, T = RECT_SIZE
    kp, _ = W.ragged_streams(S, T, T, 14)
    lengths = np.full(S, T, np.int64)
    fixed = _fixed(o, S * T, 5)
    r = _run(seq, kp, lengths, fixed)
    st = seq.make_stream_state(S)
    tape = seq.make_sequence_tape(S, T)
    seq.retarget_sequences(_t(kp.reshape(S, T, 21, 3)), seq.make_stream_state(S),
                           fixed_qpos=None if fixed is None else _t(fixed.reshape(S, T, -1)), tape=tape)
    np.testing.assert_array_equal(_np(tape.qpos).reshape(S * T, -1), r["tape_q"])
    rq, q, status = seq.smooth_packed_sequences(_t(kp), r["layout"], st, fixed_qpos=_t(fixed),
                                                qpos_init=tape.qpos.reshape(S * T, -1))
    np.testing.assert_array_equal(_np(q), r["q"])
    np.testing.assert_array_equal(_np(status), r["status"])
