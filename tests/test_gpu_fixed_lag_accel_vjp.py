"""Backpropagation through fixed-lag smoothing with an acceleration penalty on the GPU (`retarget_fixed_lag` with an
accelerated tape, `retarget_fixed_lag_accel_vjp`, `flush_fixed_lag_accel_vjp` and the autograd functions) on LEAP
DexPilot, Allegro vector and Shadow position streams and on structure cases with fixed, mimic and prismatic joints: the
float64 model of tests/fixed_lag_accel_vjp_cases.py at L in {0, 1, 4}; recording changes no bit; with L >= K - 1 and a flush
the backward is the device offline accel VJP of the whole clip bit for bit; chunks chained through the state cotangents give
the bits of one call; a stream's bits depend neither on S nor on its neighbours; the GPU agrees with the host emulation;
autograd through two chunks and a flush equals the direct calls; outputs written into sentinel-framed views stay inside
them; the call is asynchronous."""
import numpy as np
import pytest

import fixed_lag_accel_vjp_cases as FAV
import fixed_lag_vjp_cases as FLC
import seq_vjp_cases as SV
import structure_cases as SC
from helpers import build_oracle, build_product

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
STRUCTURES = ["fixed_dense16", "mimic_dense16", "mimic_fixed_dense32", "prismatic_arrow"]
SENTINEL = 16
C_OVER_W = 10.0
STREAMS = 256  # the batch of the batch-independence test (the CPU dry run shrinks it)
BATCH = 64     # the batch of the recording, full-lag, chunking and autograd tests (likewise)
CHECKED = 3    # streams checked against the model per case
STATE = ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len", "prev_qpos",
         "has_prev")


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _c(seq):
    return C_OVER_W * float(seq.optimizer.params().norm_delta)


def _state(seq, o, S, lag, seed, has_prev=1):
    """An accelerated state, empty window, seeded anchor and (has_prev = 1) pre-anchor inside the limits."""
    st = seq.make_fixed_lag_state(S, lag, accel_weight=_c(seq))
    rng = np.random.RandomState(seed)
    lo, hi = o.joint_limits[:, 0], o.joint_limits[:, 1]
    a = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), lo, hi).astype(np.float32)
    st.last_qpos.copy_(_t(a))
    if has_prev:
        st.prev_qpos.copy_(_t(np.clip(a + 0.05 * rng.randn(S, o.opt_dof), lo, hi).astype(np.float32)))
        st.has_prev.fill_(1)
    return st


def _setup(key, S, T, seed, lag, has_prev=1):
    seq, o = build_product(key, None, device=0), build_oracle(key, None)
    kp, fx = SV.stream_inputs(o, S, T, seed)
    return seq, o, _t(kp), _t(fx), _state(seq, o, S, lag, seed + 1, has_prev)


def _copy(st):
    from dex_retargeting_b200.objective import _fixed_lag_copy

    return _fixed_lag_copy(st)


def same_bits(a, b):
    """Equal with NaN where NaN (+0 == -0: an added zero cotangent may flip the sign of a zero)."""
    a, b = _np(a) if isinstance(a, torch.Tensor) else a, _np(b) if isinstance(b, torch.Tensor) else b
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def _sl(t, a, b):
    return None if t is None else t[:, a:b].contiguous()


def _cots(seq, S, K, L, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    n, dof = seq.optimizer.opt_dof, seq.optimizer.robot.dof
    r = (lambda *s: torch.randn(*s, generator=g).to(_dev()))
    return dict(grad_qpos=r(S, K, n), grad_robot_qpos=r(S, K, dof), flush_q=r(S, L, n), flush_r=r(S, L, dof),
                last=r(S, n), prev=r(S, n))


def _record(seq, kp, fx, st, L):
    s0 = _copy(st)
    tape = seq.make_fixed_lag_tape(kp.shape[0], kp.shape[1], L, accel_weight=st.accel_weight)
    out = seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    return s0, tape, out


@pytest.mark.parametrize("key", KEYS)
def test_recording_changes_no_bit(key):
    S, L, K = BATCH, 4, 12
    seq, o, kp, fx, st = _setup(key, S, K, 3, L)
    a, b = _copy(st), _copy(st)
    r0 = seq.retarget_fixed_lag(kp, a, fixed_qpos=fx)
    _, tape, r1 = _record(seq, kp, fx, b, L)
    for x, y in zip(r0, r1):
        assert same_bits(x, y) if x.dtype == torch.float32 else torch.equal(x, y)
    for k in STATE:
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None and y is None) or torch.equal(x, y), k
    assert same_bits(tape.qpos[:, -1, 1:], b.window_qpos[:, :L])


@pytest.mark.parametrize("key", KEYS)
def test_full_lag_is_the_offline_accel_vjp(key):
    """A fresh stream, L = K - 1, ticks then a flush: the device offline accel VJP of the whole clip, bit for bit."""
    S, K = BATCH, 6
    L = K - 1
    seq, o, kp, fx, st = _setup(key, S, K, 7, L, has_prev=0)
    st0, tape, _ = _record(seq, kp, fx, st, L)
    mid = _copy(st)
    seq.flush_fixed_lag(st)
    c = _cots(seq, S, K, L, 8)
    fl = seq.flush_fixed_lag_accel_vjp(mid, grad_qpos=c["flush_q"], grad_robot_qpos=c["flush_r"],
                                       grad_last_qpos_out=c["last"], grad_prev_qpos_out=c["prev"])
    got = seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=c["grad_qpos"],
                                           grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=fl[0],
                                           grad_window_keypoints_out=fl[1], grad_window_fixed_qpos_out=fl[2],
                                           grad_window_qpos_out=fl[3], grad_prev_qpos_out=fl[4])
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    cq = torch.cat([c["grad_qpos"][:, K - 1:K], c["flush_q"][:, :K - 1]], 1)
    cr = torch.cat([c["grad_robot_qpos"][:, K - 1:K], c["flush_r"][:, :K - 1]], 1)
    cq[:, -1] += c["last"]
    cq[:, -2] += c["prev"]
    layout = seq.pack_streams([K] * S)
    gk, gf, gl = seq.smooth_packed_sequences_vjp(
        kp.reshape(-1, 21, 3), layout, tape.qpos[:, K - 1].reshape(-1, n).contiguous(), st0.last_qpos, st0.projected,
        grad_qpos=cq.reshape(-1, n).contiguous(), grad_robot_qpos=cr.reshape(-1, dof).contiguous(),
        fixed_qpos=None if fx is None else fx.reshape(S * K, -1), accel_weight=st0.accel_weight)
    assert same_bits(got[0], gk.reshape(S, K, 21, 3))
    assert same_bits(got[2], gl)
    assert (got[7] == 0).all()
    if gf is not None:
        assert same_bits(got[1], gf.reshape(S, K, -1))


def _chunked(seq, kp, fx, st, cuts, c, L):
    """Forward in chunks then a flush-only call; backward chained through the state cotangents.  Returns (grad_keypoints
    [S,K], grad_fixed [S,K] or None, the first state's cotangents (last, window keypoints, window fixed, window qpos,
    prev))."""
    K = kp.shape[1]
    bounds = [0] + list(cuts) + [K]
    calls = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        s0, tape, _ = _record(seq, _sl(kp, a, b), _sl(fx, a, b), st, L)
        calls.append((a, b, s0, tape))
    mid = _copy(st)
    seq.flush_fixed_lag(st)
    carry = seq.flush_fixed_lag_accel_vjp(mid, grad_qpos=c["flush_q"], grad_robot_qpos=c["flush_r"],
                                          grad_last_qpos_out=c["last"], grad_prev_qpos_out=c["prev"])
    gks, gfs = [], []
    for a, b, s0, tape in reversed(calls):
        out = seq.retarget_fixed_lag_accel_vjp(
            _sl(kp, a, b), tape, s0, fixed_qpos=_sl(fx, a, b), grad_qpos=_sl(c["grad_qpos"], a, b),
            grad_robot_qpos=_sl(c["grad_robot_qpos"], a, b), grad_last_qpos_out=carry[0], grad_window_keypoints_out=carry[1],
            grad_window_fixed_qpos_out=carry[2], grad_window_qpos_out=carry[3], grad_prev_qpos_out=carry[4])
        gks.insert(0, out[0])
        gfs.insert(0, out[1])
        carry = out[2:6] + out[7:8]
    return torch.cat(gks, 1), (None if gfs[0] is None else torch.cat(gfs, 1)), carry


@pytest.mark.parametrize("key", KEYS)
def test_chunks_give_the_bits_of_one_call(key):
    """K ticks in one call equal the same ticks in three calls, then the flush-only call, bit for bit; the run starts with
    has_prev = 1 and a partly filled window, and one chunk starts right after the first commit."""
    S, L, K = BATCH, 4, 14
    seq, o, kp, fx, st = _setup(key, S, K + 2, 11, L)
    seq.retarget_fixed_lag(_sl(kp, 0, 2), st, fixed_qpos=_sl(fx, 0, 2))
    kp, fx = _sl(kp, 2, K + 2), _sl(fx, 2, K + 2)
    c = _cots(seq, S, K, L, 12)
    one = _chunked(seq, kp, fx, _copy(st), [], c, L)
    split = _chunked(seq, kp, fx, _copy(st), [3, 9], c, L)  # (tick 2 commits the first frame: 3 is right after it)
    assert same_bits(one[0], split[0])
    assert same_bits(one[1], split[1])
    for x, y in zip(one[2], split[2]):
        assert same_bits(x, y)
    assert torch.isfinite(one[0]).float().mean() > 0.9
    assert (one[2][4] != 0).any()


@pytest.mark.parametrize("key", KEYS[:2])
def test_stream_bits_do_not_depend_on_batch(key):
    S, L, K = STREAMS, 3, 10
    seq, o, kp, fx, st = _setup(key, S, K, 21, L)
    c = _cots(seq, S, K, L, 22)

    def run(sel):
        s = _copy(st)
        for k in STATE:
            if getattr(s, k) is not None:
                setattr(s, k, getattr(s, k)[sel].contiguous())
        kk, ff = kp[sel].contiguous(), None if fx is None else fx[sel].contiguous()
        s0, tape, _ = _record(seq, kk, ff, s, L)
        return seq.retarget_fixed_lag_accel_vjp(kk, tape, s0, fixed_qpos=ff, grad_qpos=c["grad_qpos"][sel].contiguous(),
                                                grad_robot_qpos=c["grad_robot_qpos"][sel].contiguous(),
                                                grad_prev_qpos_out=c["prev"][sel].contiguous())

    full = run(torch.arange(S, device=_dev()))
    for sel in ([S - 1], [S - 2, 0, S // 2]):
        part = run(torch.tensor(sel, device=_dev()))
        for i in (0, 2, 7):
            assert same_bits(part[i], full[i][sel]), i
        assert torch.equal(part[6], full[6][sel])


@pytest.mark.parametrize("key", KEYS[:2])
def test_gpu_matches_the_emulation(key):
    import emu_fixed_lag_accel_vjp_host as AV

    S, L, K = 3, 2, 6
    seq, o, kp, fx, st = _setup(key, S, K, 31, L)
    st0, tape, _ = _record(seq, kp, fx, st, L)
    c = _cots(seq, S, K, L, 32)
    got = seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=c["grad_qpos"],
                                           grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=c["last"],
                                           grad_prev_qpos_out=c["prev"])
    s0 = {k: _np(getattr(st0, k)) for k in STATE}
    s0.update(lag=L, accel_weight=float(st0.accel_weight))
    want = AV.fixed_lag_accel_vjp(seq, _np(kp), s0, _np(tape.qpos), _np(tape.projected), fixed_qpos=_np(fx),
                                  grad_qpos=_np(c["grad_qpos"]), grad_robot_qpos=_np(c["grad_robot_qpos"]),
                                  grad_last_qpos_out=_np(c["last"]), grad_prev_qpos_out=_np(c["prev"]))
    for g, w in ((got[0], want["grad_keypoints"]), (got[2], want["grad_last_qpos"]), (got[7], want["grad_prev_qpos"])):
        g = _np(g)
        scale = max(1.0, float(np.abs(w).max()))
        assert np.abs(g - w).max() <= 1e-3 * scale, np.abs(g - w).max()
    assert np.array_equal(_np(got[6]), want["status"])


@pytest.mark.parametrize("key", KEYS[1:2])
def test_autograd_equals_the_direct_calls(key):
    """Two chained chunks and a flush through differentiable_retarget_fixed_lag_accel / differentiable_flush_fixed_lag_accel:
    the gradients of a loss on every emitted and flushed row and on the final last_qpos and prev_qpos equal the direct VJP
    chain, in the keypoints, the anchor and the pre-anchor."""
    from dex_retargeting_b200.objective import (differentiable_flush_fixed_lag_accel,
                                                differentiable_retarget_fixed_lag_accel)

    S, L, K = BATCH, 3, 10
    seq, o, kp, fx, st = _setup(key, S, K, 41, L)
    c = _cots(seq, S, K, L, 42)
    kp_g = kp.clone().requires_grad_(True)
    last = st.last_qpos.clone().requires_grad_(True)
    prev = st.prev_qpos.clone().requires_grad_(True)
    before = _copy(st)
    s = _copy(st)
    s.last_qpos, s.prev_qpos = last, prev
    rq1, q1, _, s = differentiable_retarget_fixed_lag_accel(seq, kp_g[:, :4], s, fx if fx is None else fx[:, :4])
    assert s.accel_weight == st.accel_weight and s.prev_qpos.requires_grad
    rq2, q2, _, s = differentiable_retarget_fixed_lag_accel(seq, kp_g[:, 4:], s, fx if fx is None else fx[:, 4:])
    frq, fq, count, s = differentiable_flush_fixed_lag_accel(seq, s)
    q = torch.cat([q1, q2], 1)
    rq = torch.cat([rq1, rq2], 1)
    keep = ~torch.isnan(q[..., :1])
    fkeep = ~torch.isnan(fq[..., :1])
    loss = (torch.where(keep, q, 0) * c["grad_qpos"]).sum() + (torch.where(keep, rq, 0) * c["grad_robot_qpos"]).sum() \
        + (torch.where(fkeep, fq, 0) * c["flush_q"]).sum() + (torch.where(fkeep, frq, 0) * c["flush_r"]).sum() \
        + (s.last_qpos * c["last"]).sum() + (s.prev_qpos * c["prev"]).sum()
    loss.backward()
    gd = _chunked(seq, kp, fx, _copy(st), [4], c, L)
    assert torch.allclose(kp_g.grad, gd[0], rtol=1e-5, atol=1e-6), (kp_g.grad - gd[0]).abs().max()
    assert torch.allclose(last.grad, gd[2][0], rtol=1e-5, atol=1e-6)
    assert torch.allclose(prev.grad, gd[2][4], rtol=1e-5, atol=1e-6)
    for k in ("last_qpos", "prev_qpos", "has_prev", "window_keypoints", "window_qpos", "window_len"):
        assert torch.equal(getattr(st, k), getattr(before, k)), k
    with pytest.raises(ValueError, match="accel_weight"):
        bad = _copy(st)
        bad.accel_weight = torch.tensor(float(st.accel_weight), requires_grad=True)
        differentiable_retarget_fixed_lag_accel(seq, kp[:, :2], bad, fx if fx is None else fx[:, :2])


def test_tape_and_state_must_agree():
    from dex_retargeting_b200.objective import differentiable_retarget_fixed_lag_accel

    S, L, K = 4, 1, 3
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 45, L)
    with pytest.raises(ValueError, match="backward"):
        seq.retarget_fixed_lag(kp, _copy(st), fixed_qpos=fx, tape=seq.make_fixed_lag_tape(S, K, L))
    plain = seq.make_fixed_lag_state(S, L)
    with pytest.raises(ValueError, match="accel_weight"):
        seq.retarget_fixed_lag(kp, plain, fixed_qpos=fx, tape=seq.make_fixed_lag_tape(S, K, L, accel_weight=1.0))
    with pytest.raises(ValueError, match="accel_weight"):
        seq.retarget_fixed_lag_accel_vjp(kp, seq.make_fixed_lag_tape(S, K, L), plain)
    with pytest.raises(ValueError, match="accel_weight"):
        differentiable_retarget_fixed_lag_accel(seq, kp, plain, fx)


def test_backward_is_asynchronous():
    import time

    S, L, K = 256, 4, 20
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 51, L)
    st0, tape, _ = _record(seq, kp, fx, st, L)
    gq = torch.ones((S, K, o.opt_dof), device=_dev())
    seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=gq)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))  # ~1 s of GPU time ahead of the call on the stream
    t0 = time.perf_counter()
    out = seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=gq)
    host = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert host < 0.3, host
    assert torch.isfinite(out[0]).all()


def _model_check(seq, o, S, K, L, seed):
    """Recorded forward and backward of S streams (has_prev = 1, empty window), compared with the float64 model until
    CHECKED streams are (a stream the model skips -- near a DexPilot zone switch or singular -- is passed over); returns
    the streams checked."""
    kp_np, fx_np = SV.stream_inputs(o, S, K, seed)
    kp, fx = _t(kp_np), _t(fx_np)
    st = _state(seq, o, S, L, seed + 1)
    st0, tape, _ = _record(seq, kp, fx, st, L)
    rng = np.random.RandomState(seed + 2)
    gq = rng.randn(S, K, o.opt_dof).astype(np.float32)
    grq = rng.randn(S, K, seq.optimizer.robot.dof).astype(np.float32)
    gl, gp = rng.randn(S, o.opt_dof).astype(np.float32), rng.randn(S, o.opt_dof).astype(np.float32)
    g_kp, g_f, g_last, *_, status, g_prev = seq.retarget_fixed_lag_accel_vjp(
        kp, tape, st0, fixed_qpos=fx, grad_qpos=_t(gq), grad_robot_qpos=_t(grq), grad_last_qpos_out=_t(gl),
        grad_prev_qpos_out=_t(gp))
    status = _np(status)
    layout = seq.pack_streams([K] * S)
    ptape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(kp.reshape(-1, 21, 3), layout, seq.make_stream_state(S),
                                  fixed_qpos=None if fx is None else fx.reshape(S * K, -1), tape=ptape)
    fl = None if ptape.projected is None else _np(ptape.projected).reshape(S, K, -1)
    tq = _np(tape.qpos)
    w = float(seq.optimizer.params().norm_delta)
    a, p = _np(st0.last_qpos), _np(st0.prev_qpos)
    checked = 0
    for s in range(S):
        if checked >= CHECKED:
            break
        if (status[s] & ((1 << 26) | (1 << 25))).any():
            continue
        Xs = [tq[s, k, :FLC.window(k, L)[1]] for k in range(K)]
        md = FAV.model_chain(o, w, float(st0.accel_weight), kp_np[s].astype(np.float64),
                             None if fx_np is None else fx_np[s].astype(np.float64), None if fl is None else fl[s],
                             a[s].astype(np.float64), p[s].astype(np.float64), 1, Xs, L, gq[s], grq[s], gl[s], gp[s])
        if md["skip"] or md["not_pd"]:
            continue
        FAV.compare(_np(g_kp)[s], None if g_f is None else _np(g_f)[s], _np(g_last)[s], _np(g_prev)[s], md)
        checked += 1
    return checked


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("key", KEYS)
def test_matches_the_model(key, lag):
    seq, o = build_product(key, None, device=0), build_oracle(key, None)
    assert _model_check(seq, o, 8, 6, lag, 61 + lag) >= 1


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("case", STRUCTURES)
def test_matches_the_model_on_structure_cases(case, lag, tmp_path):
    seq, o = SC.build(SC.BY_ID[case], tmp_path)
    assert _model_check(seq, o, 8, 6, lag, 71 + lag) >= 1


def test_writes_stay_inside_their_buffers():
    """Every output is a view with SENTINEL rows before and after it: the sentinels survive, the values are those of the
    library's own buffers."""
    S, L, K = 5, 3, 9
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 81, L)
    st0, tape, _ = _record(seq, kp, fx, st, L)
    c = _cots(seq, S, K, L, 82)
    args = dict(fixed_qpos=fx, grad_qpos=c["grad_qpos"], grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=c["last"],
                grad_prev_qpos_out=c["prev"])
    want = seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, **args)
    n = o.opt_dof
    shapes = dict(grad_keypoints=(S, K, 21, 3), grad_last_qpos=(S, n), grad_window_keypoints=(S, L + 1, 21, 3),
                  grad_window_qpos=(S, L + 1, n), status_out=(S, K), grad_prev_qpos=(S, n))
    bigs, views = {}, {}
    for name, shape in shapes.items():
        dt = torch.int32 if name == "status_out" else torch.float32
        big = torch.full((SENTINEL * 2 + shape[0],) + tuple(shape[1:]), -7, dtype=dt, device=_dev())
        bigs[name], views[name] = big, big[SENTINEL:SENTINEL + shape[0]]
    got = seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, outputs=views, **args)
    for name, big in bigs.items():
        b = _np(big)
        assert (b[:SENTINEL] == -7).all() and (b[-SENTINEL:] == -7).all(), name
    for i in (0, 2, 3, 5, 6, 7):
        assert same_bits(got[i], want[i]) if got[i].dtype == torch.float32 else torch.equal(got[i], want[i])
    assert got[7].data_ptr() == views["grad_prev_qpos"].data_ptr()
