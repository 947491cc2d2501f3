"""Packed streams on the GPU (`dexr_solve_sequences_packed`, `dexr_solve_sequences_packed_vjp`,
SeqRetargeting.retarget_packed_sequences / retarget_packed_sequences_vjp, objective.differentiable_retarget_packed_sequences):
equal lengths bit for bit against the rectangular calls, ragged streams (lengths 0 and 1 included, two different lengths in
one warp) bit for bit against a call on each stream alone, the float64 oracle on the benchmark's ragged workloads, chained
chunks, the streams' positions in the batch, central differences and the argument checks."""
import ctypes as C
import os
import sys
from pathlib import Path

import numpy as np
import pytest

import seq_vjp_cases as SV
from helpers import build_oracle, build_product

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
# streams x steps of the equal-length check; streams of the ragged check (more than one wave of warps, so that two 16-lane
# streams of different lengths share a warp) and how many of them are re-solved alone.  The CPU dry run
# (tests/tools/emu_gpu_packed.py) shrinks them: the emulation solves a few frames per second.
EQUAL_SIZE = (96, 12)
RAGGED_STREAMS = 1200
RAGGED_CHECKED = 12
ORACLE_STREAMS, ORACLE_FRAMES = 3, 6


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _seq(key, override=None):
    return build_product(key, override, device=0)


def _state_copy(st):
    from dex_retargeting_b200.seq_retarget import StreamState

    return StreamState(**{k: None if getattr(st, k) is None else getattr(st, k).clone() for k in StreamState._FIELDS})


def _state_np(st):
    return {k: _np(getattr(st, k)) for k in ("last_qpos", "filter_state", "filter_init", "projected", "damping")}


def _assert_same(a, b, what=""):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    np.testing.assert_array_equal(np.asarray(a), np.asarray(b), err_msg=what)


def _ragged(S, seed):
    """Seeded lengths 0..6 with 0 and 1 present, keypoints from the recorded trajectory packed end to end."""
    rng = np.random.RandomState(seed)
    lengths = rng.randint(0, 7, size=S)
    lengths[:3] = [0, 1, 6]
    rng.shuffle(lengths)
    traj = W.ragged_streams(1, 300, 300, seed)[0]
    kp = np.concatenate([traj[:n] + (rng.randn(1, 21, 3) * 0.002).astype(np.float32) for n in lengths])
    kp[:, 0] = 0
    return np.ascontiguousarray(kp, np.float32), lengths


def _forward_and_backward(seq, kp, lengths, cot=None):
    """Recorded packed forward from fresh state, then the packed VJP with seeded cotangents (or `cot`).  Returns host
    arrays."""
    S, N_ = len(lengths), int(np.sum(lengths))
    layout = seq.pack_streams(lengths)
    st = seq.make_stream_state(S)
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    status = torch.empty((N_,), dtype=torch.int32, device=_dev())
    tape = seq.make_packed_sequence_tape(layout)
    out, _ = seq.retarget_packed_sequences(_t(kp), layout, st, status_out=status, tape=tape)
    opt = seq.optimizer
    rng = np.random.RandomState(5)
    g_out = _t(rng.randn(N_, opt.robot.dof).astype(np.float32))
    g_last = _t(rng.randn(S, opt.opt_dof).astype(np.float32))
    g_filter = _t(rng.randn(S, opt.robot.dof).astype(np.float32))
    if cot is not None:
        g_out, g_last, g_filter = (_t(c) for c in cot)
    vstatus = torch.empty((N_,), dtype=torch.int32, device=_dev())
    grads = seq.retarget_packed_sequences_vjp(_t(kp), layout, tape, last0, finit0, grad_robot_qpos=g_out,
                                              grad_last_qpos=g_last, grad_filter_state=g_filter, status_out=vstatus)
    return dict(out=_np(out), status=_np(status), state=_state_np(st), tape_qpos=_np(tape.qpos),
                tape_proj=_np(tape.projected), grads=[_np(g) for g in grads], vstatus=_np(vstatus),
                cot=(_np(g_out), _np(g_last), _np(g_filter)))


@pytest.mark.parametrize("key", KEYS)
def test_equal_lengths_match_the_rectangular_calls(key):
    """Every length T: forward, recorded forward and backward equal dexr_solve_sequences / _tape / _vjp bit for bit."""
    seq = _seq(key)
    S, T = EQUAL_SIZE
    kp = W.streams(S, T, seed=W.STREAM_SEED)
    p = _forward_and_backward(seq, kp.reshape(S * T, 21, 3), np.full(S, T))
    st = seq.make_stream_state(S)
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    st_plain = _state_copy(st)
    status = torch.empty((S, T), dtype=torch.int32, device=_dev())
    out_plain, _ = seq.retarget_sequences(_t(kp), st_plain)
    tape = seq.make_sequence_tape(S, T)
    out, _ = seq.retarget_sequences(_t(kp), st, status_out=status, tape=tape)
    _assert_same(_np(out_plain), _np(out))
    # the unrecorded packed forward too
    st_p = seq.make_stream_state(S)
    out_p, _ = seq.retarget_packed_sequences(_t(kp.reshape(S * T, 21, 3)), seq.pack_streams(np.full(S, T)), st_p)
    _assert_same(_np(out_p).reshape(S, T, -1), _np(out), "unrecorded packed forward")
    _assert_same(p["out"].reshape(S, T, -1), _np(out), "robot_qpos")
    _assert_same(p["status"].reshape(S, T), _np(status), "status")
    for k, v in _state_np(st).items():
        _assert_same(p["state"][k], v, k)
    _assert_same(p["tape_qpos"].reshape(S, T, -1), _np(tape.qpos), "tape.qpos")
    if tape.projected is not None:
        _assert_same(p["tape_proj"].reshape(S, T, -1), _np(tape.projected), "tape.projected")
    g_out, g_last, g_filter = p["cot"]
    vstatus = torch.empty((S, T), dtype=torch.int32, device=_dev())
    grads = seq.retarget_sequences_vjp(_t(kp), tape, last0, finit0, grad_robot_qpos=_t(g_out.reshape(S, T, -1)),
                                       grad_last_qpos=_t(g_last), grad_filter_state=_t(g_filter), status_out=vstatus)
    _assert_same(p["grads"][0].reshape(S, T, 21, 3), _np(grads[0]), "grad_keypoints")
    _assert_same(p["grads"][2], _np(grads[2]), "grad_last_qpos")
    _assert_same(p["grads"][3], _np(grads[3]), "grad_filter_state")
    _assert_same(p["vstatus"].reshape(S, T), _np(vstatus), "vjp status")


@pytest.mark.parametrize("key", KEYS)
def test_ragged_streams_match_each_stream_alone(key):
    """Lengths 0..6 over more streams than one wave of warps (16-lane streams of different lengths share a warp): every
    stream's outputs, final state, tape and gradients equal a rectangular call on that stream alone; a stream of length 0
    keeps its state and passes its cotangents through.  Both calls without duo mode (DEXR_SEQ_DUO=0), which would
    otherwise split a lone 16-lane stream over two half-warps."""
    seq = _seq(key)
    kp, lengths = _ragged(RAGGED_STREAMS, seed=61)
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    old = os.environ.get("DEXR_SEQ_DUO")
    os.environ["DEXR_SEQ_DUO"] = "0"
    try:
        p = _forward_and_backward(seq, kp, lengths)
        fresh = _state_np(seq.make_stream_state(1))
        g_out, g_last, g_filter = p["cot"]
        empty = [s for s in range(len(lengths)) if lengths[s] == 0][:2]
        checked = empty + [s for s in range(len(lengths)) if lengths[s] > 0][:RAGGED_CHECKED - len(empty)]
        for s in checked:
            a, b = int(offsets[s]), int(offsets[s + 1])
            if a == b:
                for k, v in fresh.items():
                    _assert_same(None if p["state"][k] is None else p["state"][k][s:s + 1], v, f"stream {s} {k}")
                _assert_same(p["grads"][2][s], g_last[s], "empty stream: grad_last_qpos passes through")
                _assert_same(p["grads"][3][s], g_filter[s], "empty stream: grad_filter_state passes through")
                continue
            st = seq.make_stream_state(1)
            last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
            status = torch.empty((1, b - a), dtype=torch.int32, device=_dev())
            tape = seq.make_sequence_tape(1, b - a)
            kp1 = _t(kp[None, a:b])
            out, _ = seq.retarget_sequences(kp1, st, status_out=status, tape=tape)
            _assert_same(p["out"][a:b], _np(out)[0], f"stream {s} robot_qpos")
            _assert_same(p["status"][a:b], _np(status)[0], f"stream {s} status")
            for k, v in _state_np(st).items():
                _assert_same(None if p["state"][k] is None else p["state"][k][s:s + 1], v, f"stream {s} {k}")
            _assert_same(p["tape_qpos"][a:b], _np(tape.qpos)[0], f"stream {s} tape")
            grads = seq.retarget_sequences_vjp(kp1, tape, last0, finit0, grad_robot_qpos=_t(g_out[None, a:b]),
                                               grad_last_qpos=_t(g_last[s:s + 1]), grad_filter_state=_t(g_filter[s:s + 1]))
            _assert_same(p["grads"][0][a:b], _np(grads[0])[0], f"stream {s} grad_keypoints")
            _assert_same(p["grads"][2][s], _np(grads[2])[0], f"stream {s} grad_last_qpos")
            _assert_same(p["grads"][3][s], _np(grads[3])[0], f"stream {s} grad_filter_state")
    finally:
        if old is None:
            os.environ.pop("DEXR_SEQ_DUO", None)
        else:
            os.environ["DEXR_SEQ_DUO"] = old


@pytest.mark.parametrize("key,S", [(W.LEAP_DEXPILOT_KEY, 2048), (W.METRIC_KEY, 2048), (W.SHADOW_POS_KEY, 512)])
def test_ragged_workloads_match_the_oracle(key, S):
    """The benchmark's workloads (tools/workloads.py `ragged_streams`) in one packed launch; the first frames of a few
    streams (a stream's prefix is a stream) against the float64 oracle: |dq| < 1e-4 rad, as tests/test_gpu_parity.py."""
    seq = _seq(key)
    o = build_oracle(key)
    kp, lengths = W.ragged_streams(S)
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    out, _ = seq.retarget_packed_sequences(_t(kp), seq.pack_streams(lengths))
    got = _np(out)
    assert np.isfinite(got).all()
    last0 = seq.joint_limits.mean(1).astype(np.float32)
    worst = 0.0
    for s in np.linspace(0, S - 1, ORACLE_STREAMS).astype(int):
        a = int(offsets[s])
        r = SV.oracle_stream(o, kp[a:a + ORACLE_FRAMES], None, last0, np.zeros(o.robot.dof), 0)
        worst = max(worst, float(np.abs(got[a:a + ORACLE_FRAMES] - r["robot_qpos"]).max()))
    assert worst < 1e-4, worst


@pytest.mark.parametrize("key", KEYS[:2])
def test_chained_chunks_equal_one_call(key):
    """packed(L1) then packed(L2) on the returned state equals packed(L1 + L2), forward and backward (autograd)."""
    from dex_retargeting_b200.objective import differentiable_retarget_packed_sequences

    seq = _seq(key)
    l1, l2 = np.array([3, 0, 2, 4, 1]), np.array([2, 3, 0, 1, 4])
    S = len(l1)
    lengths = l1 + l2
    traj = W.ragged_streams(S, 10, 10, seed=64)[0].reshape(S, 10, 21, 3)
    w = torch.randn((int(lengths.sum()), seq.optimizer.robot.dof), generator=torch.Generator().manual_seed(65)).to(_dev())

    def run(split):
        kp = _t(np.concatenate([traj[s, :lengths[s]] for s in range(S)])).requires_grad_(True)
        state = seq.make_stream_state(S)
        last = state.last_qpos.clone().requires_grad_(True)
        state.last_qpos = last
        # frame rows of each chunk in the packed order of the whole call
        offs = np.concatenate([[0], np.cumsum(lengths)])
        rows1 = np.concatenate([offs[s] + np.arange(l1[s]) for s in range(S)])
        rows2 = np.concatenate([offs[s] + l1[s] + np.arange(l2[s]) for s in range(S)])
        if split:
            o1, s1 = differentiable_retarget_packed_sequences(seq, kp[_t(rows1)], seq.pack_streams(l1), state)
            o2, s2 = differentiable_retarget_packed_sequences(seq, kp[_t(rows2)], seq.pack_streams(l2), s1)
            out = torch.empty((int(lengths.sum()), o1.shape[1]), device=_dev())
            out = out.index_put((_t(rows1),), o1).index_put((_t(rows2),), o2)
            fin = s2
        else:
            out, fin = differentiable_retarget_packed_sequences(seq, kp, seq.pack_streams(lengths), state)
        ((w * out).sum() + fin.last_qpos.sum()).backward()
        return out.detach(), fin.last_qpos.detach(), kp.grad, last.grad

    for x, y in zip(run(False), run(True)):
        assert torch.equal(x, y)


def test_results_do_not_depend_on_the_position_in_the_batch():
    """The same streams packed in another order (longest first, and a random permutation) give every stream the same bits
    (the cotangents follow their streams)."""
    key = KEYS[0]
    seq = _seq(key)
    kp, lengths = _ragged(9, seed=67)
    offs = np.concatenate([[0], np.cumsum(lengths)])
    a = _forward_and_backward(seq, kp, lengths)
    for perm in (np.argsort(-lengths, kind="stable"), np.random.RandomState(68).permutation(len(lengths))):
        rows = np.concatenate([offs[s] + np.arange(lengths[s]) for s in perm]).astype(int)
        g_out, g_last, g_filter = a["cot"]
        b = _forward_and_backward(seq, kp[rows], lengths[perm], cot=(g_out[rows], g_last[perm], g_filter[perm]))
        for k in ("out", "status", "tape_qpos", "tape_proj", "vstatus"):
            if a[k] is not None:
                _assert_same(a[k][rows], b[k], k)
        for k in a["state"]:
            if a["state"][k] is not None:
                _assert_same(a["state"][k][perm], b["state"][k], k)
        _assert_same(a["grads"][0][rows], b["grads"][0], "grad_keypoints")
        _assert_same(a["grads"][2][perm], b["grads"][2], "grad_last_qpos")
        _assert_same(a["grads"][3][perm], b["grads"][3], "grad_filter_state")


def test_differentiable_retarget_packed_sequences_against_central_differences():
    """Stream 1 of three (lengths 2, 4, 0): the autograd gradient against central differences of float64 oracle streams."""
    from dex_retargeting_b200.objective import differentiable_retarget_packed_sequences

    key = "teleop/allegro_hand_right"
    seq, o = _seq(key), build_oracle(key)
    kp4, _ = SV.stream_inputs(o, 2, 4, seed=69)
    lengths = np.array([2, 4, 0])
    kp_np = np.concatenate([kp4[1, :2], kp4[0]])
    rng = np.random.RandomState(70)
    last0 = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(3, o.opt_dof), o.joint_limits[:, 0],
                    o.joint_limits[:, 1]).astype(np.float32)
    y0 = rng.uniform(-0.3, 0.3, size=(3, o.robot.dof)).astype(np.float32)
    state = seq.make_stream_state(3)
    state.last_qpos.copy_(_t(last0))
    state.filter_state.copy_(_t(y0))
    state.filter_init.fill_(1)
    kp = _t(kp_np).requires_grad_(True)
    last = state.last_qpos.clone().requires_grad_(True)
    filt = state.filter_state.clone().requires_grad_(True)
    state.last_qpos, state.filter_state = last, filt
    out, _ = differentiable_retarget_packed_sequences(seq, kp, seq.pack_streams(lengths), state)
    w = _t(rng.randn(6, o.robot.dof).astype(np.float32))
    (w * out).sum().backward()
    g = _np(w)[2:6].astype(np.float64)

    def loss(kp_=kp_np[2:6], last_=last0[1], y_=y0[1]):
        r = SV.oracle_stream(o, kp_, None, last_, y_, 1)
        return float((g * r["robot_qpos"]).sum())

    h = 1e-3
    used = int(np.asarray(o.target_link_human_indices).reshape(-1)[-1])
    for name, at, grad in (("kp_", (0, used, 1), kp.grad[2:6]), ("kp_", (3, used, 0), kp.grad[2:6]),
                           ("last_", (2,), last.grad[1]), ("y_", (1,), filt.grad[1])):
        base = dict(kp_=kp_np[2:6], last_=last0[1], y_=y0[1])[name].astype(np.float64)
        plus, minus = base.copy(), base.copy()
        plus[at] += h
        minus[at] -= h
        fd = (loss(**{name: plus}) - loss(**{name: minus})) / (2 * h)
        an = float(grad[at])
        assert abs(an - fd) <= 5e-2 * max(abs(fd), 2e-2), (name, at, an, fd)
    assert float(last.grad[2].abs().max()) == 0.0 and float(filt.grad[2].abs().max()) == 0.0  # the empty stream


def test_argument_errors_are_rejected_with_a_message():
    from dex_retargeting_b200 import _native as N
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq = _seq(KEYS[0])
    lengths = np.array([2, 0, 3])
    layout = seq.pack_streams(lengths)
    kp = torch.zeros((5, 21, 3), device=_dev())
    state = seq.make_stream_state(3)
    tape = seq.make_packed_sequence_tape(layout)
    with pytest.raises(N.DexrError, match="flag tape"):
        seq.retarget_packed_sequences(kp, layout, state, tape=SequenceTape(qpos=tape.qpos, projected=None))
    with pytest.raises(N.DexrError, match="DexPilot needs the flag tape"):
        seq.retarget_packed_sequences_vjp(kp, layout, SequenceTape(qpos=tape.qpos, projected=None), state.last_qpos,
                                          state.filter_init)
    with pytest.raises(ValueError, match="keypoints"):
        seq.retarget_packed_sequences(torch.zeros((4, 21, 3), device=_dev()), layout, state)
    with pytest.raises(ValueError, match="tape.qpos"):
        seq.retarget_packed_sequences_vjp(kp, layout, SequenceTape(qpos=tape.qpos[:4].contiguous(), projected=tape.projected),
                                          state.last_qpos, state.filter_init)
    with pytest.raises(ValueError, match=">= 0"):
        seq.pack_streams([2, -1])
    eng = seq.optimizer.engine()
    p = seq.optimizer.params(clip_init=True, lp_alpha=seq.low_pass_alpha)
    io = N.DexrSequences()
    io.keypoints, io.last_qpos, io.robot_qpos_out = kp.data_ptr(), state.last_qpos.data_ptr(), kp.data_ptr()
    io.filter_state, io.filter_init = state.filter_state.data_ptr(), state.filter_init.data_ptr()
    rc = eng.lib.dexr_solve_sequences_packed(eng.handle, C.byref(p), C.byref(io), None, None, 3, 5, None)
    assert rc == -1 and b"offsets" in eng.lib.dexr_last_error()
    rc = eng.lib.dexr_solve_sequences_packed(eng.handle, C.byref(p), C.byref(io), None, C.c_void_p(layout.offsets.data_ptr()),
                                             -1, 5, None)
    assert rc == -1 and b"bad sizes" in eng.lib.dexr_last_error()
