"""Backpropagation through fixed-lag smoothing on the GPU (`retarget_fixed_lag` with `tape=`, `retarget_fixed_lag_vjp`,
`flush_fixed_lag_vjp` and the autograd functions) on LEAP DexPilot, Allegro vector and Shadow position streams and on
structure cases with fixed, mimic and prismatic joints: the float64 model of tests/fixed_lag_vjp_cases.py; recording
changes no output bit; with L >= K - 1 and a flush the backward is the device smoother VJP of the whole clip bit for bit; a
run split into chunks chained through the state cotangents gives the bits of one call; a stream's bits do not depend on S;
the GPU agrees with the host emulation; autograd through two chunks and a flush equals the direct calls; the call is
asynchronous; outputs written into sentinel-framed views stay inside them."""
import numpy as np
import pytest

import fixed_lag_vjp_cases as FLC
import seq_vjp_cases as SV
import structure_cases as SC
from helpers import build_oracle, build_product

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
STRUCTURES = ["fixed_dense16", "mimic_dense16", "mimic_fixed_dense32", "prismatic_arrow"]
SENTINEL = 16
STATUS_PENDING = 1 << 28


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _setup(key, S, T, seed, lag):
    seq, o = build_product(key, None, device=0), build_oracle(key, None)
    kp, fx = SV.stream_inputs(o, S, T, seed)
    st = seq.make_fixed_lag_state(S, lag)
    rng = np.random.RandomState(seed + 1)
    a = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    st.last_qpos.copy_(_t(a.astype(np.float32)))
    return seq, o, _t(kp), _t(fx), st


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
                last=r(S, n))


@pytest.mark.parametrize("key", KEYS)
def test_recording_changes_no_bit(key):
    S, L, K = 64, 4, 12
    seq, o, kp, fx, st = _setup(key, S, K, 3, L)
    a, b = _copy(st), _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    r0 = seq.retarget_fixed_lag(kp, a, fixed_qpos=fx)
    r1 = seq.retarget_fixed_lag(kp, b, fixed_qpos=fx, tape=tape)
    for x, y in zip(r0, r1):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y)
    for k in ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len"):
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None and y is None) or torch.equal(x, y), k
    assert same_bits(tape.qpos[:, -1, 1:], b.window_qpos[:, :L])  # the last tick's window, shifted by its emission


@pytest.mark.parametrize("key", KEYS)
def test_full_lag_is_the_smoother_vjp(key):
    """Fresh state, L = K - 1, ticks then a flush: the device smoother VJP of the whole clip at the last window, bit for bit."""
    S, K = 48, 6
    L = K - 1
    seq, o, kp, fx, st = _setup(key, S, K, 7, L)
    st0 = _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    mid = _copy(st)
    seq.flush_fixed_lag(st)
    c = _cots(seq, S, K, L, 8)
    # one call = the ticks' VJP fed the flush's (the chunk identity makes it the same bits as ticks + flush in one call)
    fl = seq.flush_fixed_lag_vjp(mid, grad_qpos=c["flush_q"], grad_robot_qpos=c["flush_r"], grad_last_qpos_out=c["last"])
    got = seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=c["grad_qpos"],
                                     grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=fl[0],
                                     grad_window_keypoints_out=fl[1], grad_window_fixed_qpos_out=fl[2],
                                     grad_window_qpos_out=fl[3])
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    cq = torch.cat([c["grad_qpos"][:, K - 1:K], c["flush_q"][:, :K - 1]], 1)
    cr = torch.cat([c["grad_robot_qpos"][:, K - 1:K], c["flush_r"][:, :K - 1]], 1)
    cq[:, -1] += c["last"]
    layout = seq.pack_streams([K] * S)
    gk, gf, gl = seq.smooth_packed_sequences_vjp(
        kp.reshape(-1, 21, 3), layout, tape.qpos[:, K - 1].reshape(-1, n).contiguous(), st0.last_qpos, st0.projected,
        grad_qpos=cq.reshape(-1, n).contiguous(), grad_robot_qpos=cr.reshape(-1, dof).contiguous(),
        fixed_qpos=None if fx is None else fx.reshape(S * K, -1))
    assert same_bits(got[0], gk.reshape(S, K, 21, 3))
    assert same_bits(got[2], gl)
    if gf is not None:
        assert same_bits(got[1], gf.reshape(S, K, -1))


def _chunked(seq, kp, fx, st, cuts, c, L):
    """Forward in chunks then a flush-only call; backward chained through the state cotangents.  Returns (grad_keypoints
    [S,K], grad_fixed [S,K] or None, the first state's cotangents)."""
    K = kp.shape[1]
    bounds = [0] + list(cuts) + [K]
    calls = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        s0 = _copy(st)
        tape = seq.make_fixed_lag_tape(kp.shape[0], b - a, L)
        seq.retarget_fixed_lag(_sl(kp, a, b), st, fixed_qpos=_sl(fx, a, b), tape=tape)
        calls.append((a, b, s0, tape))
    mid = _copy(st)
    seq.flush_fixed_lag(st)
    carry = seq.flush_fixed_lag_vjp(mid, grad_qpos=c["flush_q"], grad_robot_qpos=c["flush_r"], grad_last_qpos_out=c["last"])
    gks, gfs = [], []
    for a, b, s0, tape in reversed(calls):
        out = seq.retarget_fixed_lag_vjp(_sl(kp, a, b), tape, s0, fixed_qpos=_sl(fx, a, b),
                                         grad_qpos=_sl(c["grad_qpos"], a, b), grad_robot_qpos=_sl(c["grad_robot_qpos"], a, b),
                                         grad_last_qpos_out=carry[0], grad_window_keypoints_out=carry[1],
                                         grad_window_fixed_qpos_out=carry[2], grad_window_qpos_out=carry[3])
        gks.insert(0, out[0])
        gfs.insert(0, out[1])
        carry = out[2:6]
    return torch.cat(gks, 1), (None if gfs[0] is None else torch.cat(gfs, 1)), carry


@pytest.mark.parametrize("key", KEYS)
def test_chunks_give_the_bits_of_one_call(key):
    """K ticks in one call equal the same ticks in three calls, each followed by the flush-only call, bit for bit; the run
    starts with a partly filled window."""
    S, L, K = 64, 4, 14
    seq, o, kp, fx, st = _setup(key, S, K + 2, 11, L)
    seq.retarget_fixed_lag(_sl(kp, 0, 2), st, fixed_qpos=_sl(fx, 0, 2))
    kp, fx = _sl(kp, 2, K + 2), _sl(fx, 2, K + 2)
    c = _cots(seq, S, K, L, 12)
    one = _chunked(seq, kp, fx, _copy(st), [], c, L)
    split = _chunked(seq, kp, fx, _copy(st), [5, 9], c, L)
    assert same_bits(one[0], split[0])
    assert same_bits(one[1], split[1])
    for x, y in zip(one[2], split[2]):
        assert same_bits(x, y)
    assert torch.isfinite(one[0]).float().mean() > 0.9


@pytest.mark.parametrize("key", KEYS[:2])
def test_stream_bits_do_not_depend_on_batch(key):
    S, L, K = 256, 3, 10
    seq, o, kp, fx, st = _setup(key, S, K, 21, L)
    c = _cots(seq, S, K, L, 22)

    def run(sel):
        s = _copy(st)
        for k in ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos", "window_qpos", "window_len"):
            if getattr(s, k) is not None:
                setattr(s, k, getattr(s, k)[sel].contiguous())
        s0 = _copy(s)
        tape = seq.make_fixed_lag_tape(len(sel), K, L)
        kk, ff = kp[sel].contiguous(), None if fx is None else fx[sel].contiguous()
        seq.retarget_fixed_lag(kk, s, fixed_qpos=ff, tape=tape)
        return seq.retarget_fixed_lag_vjp(kk, tape, s0, fixed_qpos=ff, grad_qpos=c["grad_qpos"][sel].contiguous(),
                                          grad_robot_qpos=c["grad_robot_qpos"][sel].contiguous())

    full = run(torch.arange(S, device=_dev()))
    for sel in ([7], [200, 3, 100]):
        part = run(torch.tensor(sel, device=_dev()))
        assert same_bits(part[0], full[0][sel])
        assert same_bits(part[2], full[2][sel])
        assert torch.equal(part[6], full[6][sel])


@pytest.mark.parametrize("key", KEYS[:2])
def test_gpu_matches_the_emulation(key):
    import emu_fixed_lag_vjp_host as FV

    S, L, K = 3, 2, 6
    seq, o, kp, fx, st = _setup(key, S, K, 31, L)
    st0 = _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    c = _cots(seq, S, K, L, 32)
    got = seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=c["grad_qpos"],
                                     grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=c["last"])
    s0 = {k: _np(getattr(st0, k)) for k in ("last_qpos", "projected", "window_keypoints", "window_fixed_qpos",
                                             "window_qpos", "window_len")}
    s0["lag"] = L
    want = FV.fixed_lag_vjp(seq, _np(kp), s0, _np(tape.qpos), _np(tape.projected), fixed_qpos=_np(fx),
                            grad_qpos=_np(c["grad_qpos"]), grad_robot_qpos=_np(c["grad_robot_qpos"]),
                            grad_last_qpos_out=_np(c["last"]))
    for g, w in ((got[0], want["grad_keypoints"]), (got[2], want["grad_last_qpos"])):
        g = _np(g)
        scale = max(1.0, float(np.abs(w).max()))
        assert np.abs(g - w).max() <= 1e-3 * scale, np.abs(g - w).max()
    assert np.array_equal(_np(got[6]), want["status"])


@pytest.mark.parametrize("key", KEYS[1:2])
def test_autograd_equals_the_direct_calls(key):
    """Two chained chunks and a flush through differentiable_retarget_fixed_lag / differentiable_flush_fixed_lag: the
    gradients of a loss on every emitted and flushed row equal the direct VJP chain."""
    from dex_retargeting_b200.objective import differentiable_flush_fixed_lag, differentiable_retarget_fixed_lag

    S, L, K = 32, 3, 10
    seq, o, kp, fx, st = _setup(key, S, K, 41, L)
    c = _cots(seq, S, K, L, 42)
    kp_g = kp.clone().requires_grad_(True)
    last = st.last_qpos.clone().requires_grad_(True)
    before = _copy(st)
    s = _copy(st)
    s.last_qpos = last
    rq1, q1, _, s = differentiable_retarget_fixed_lag(seq, kp_g[:, :4], s)
    rq2, q2, _, s = differentiable_retarget_fixed_lag(seq, kp_g[:, 4:], s)
    frq, fq, count, s = differentiable_flush_fixed_lag(seq, s)
    q = torch.cat([q1, q2], 1)
    rq = torch.cat([rq1, rq2], 1)
    keep = ~torch.isnan(q[..., :1])
    fkeep = ~torch.isnan(fq[..., :1])
    loss = (torch.where(keep, q, 0) * c["grad_qpos"]).sum() + (torch.where(keep, rq, 0) * c["grad_robot_qpos"]).sum() \
        + (torch.where(fkeep, fq, 0) * c["flush_q"]).sum() + (torch.where(fkeep, frq, 0) * c["flush_r"]).sum() \
        + (s.last_qpos * c["last"]).sum()
    loss.backward()
    # the direct chain; the PENDING and past-count rows' cotangents are ignored by the library
    gd = _chunked(seq, kp, fx, _copy(st), [4], c, L)
    assert torch.allclose(kp_g.grad, gd[0], rtol=1e-5, atol=1e-6), (kp_g.grad - gd[0]).abs().max()
    assert torch.allclose(last.grad, gd[2][0], rtol=1e-5, atol=1e-6)
    for k in ("last_qpos", "window_keypoints", "window_qpos", "window_len"):  # the caller's state is not modified
        assert torch.equal(getattr(st, k), getattr(before, k)), k


def test_backward_is_asynchronous():
    import time

    S, L, K = 256, 4, 20
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 51, L)
    st0 = _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    gq = torch.ones((S, K, o.opt_dof), device=_dev())
    seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=gq)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e9))  # ~1 s of GPU time ahead of the call on the stream
    t0 = time.perf_counter()
    out = seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=gq)
    host = time.perf_counter() - t0
    torch.cuda.synchronize()
    assert host < 0.3, host
    assert torch.isfinite(out[0]).all()


def _model_check(seq, o, S, K, L, seed):
    """Recorded forward and backward of S fresh streams, each compared with the float64 model; returns the streams checked."""
    kp_np, fx_np = SV.stream_inputs(o, S, K, seed)
    kp, fx = _t(kp_np), _t(fx_np)
    st = seq.make_fixed_lag_state(S, L)
    rng = np.random.RandomState(seed + 1)
    a = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    st.last_qpos.copy_(_t(a.astype(np.float32)))
    st0 = _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    gq = rng.randn(S, K, o.opt_dof).astype(np.float32)
    grq = rng.randn(S, K, seq.optimizer.robot.dof).astype(np.float32)
    g_kp, g_f, g_last, *_, status = seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fx, grad_qpos=_t(gq),
                                                                grad_robot_qpos=_t(grq))
    status = _np(status)
    # the DexPilot flags every frame uses: the causal walk from fresh flags
    layout = seq.pack_streams([K] * S)
    ptape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(kp.reshape(-1, 21, 3), layout, seq.make_stream_state(S),
                                  fixed_qpos=None if fx is None else fx.reshape(S * K, -1), tape=ptape)
    fl = None if ptape.projected is None else _np(ptape.projected).reshape(S, K, -1)
    tq = _np(tape.qpos)
    w = float(seq.optimizer.params().norm_delta)
    checked = 0
    for s in range(S):
        if (status[s] & ((1 << 26) | (1 << 25))).any():
            continue
        Xs = [tq[s, k, :FLC.window(k, L)[1]] for k in range(K)]
        md = FLC.model_chain(o, w, kp_np[s].astype(np.float64), None if fx_np is None else fx_np[s].astype(np.float64),
                             None if fl is None else fl[s], a[s], Xs, L, gq[s], grq[s])
        if md["skip"] or md["not_pd"]:
            continue
        FLC.compare(_np(g_kp)[s], None if g_f is None else _np(g_f)[s], _np(g_last)[s], md)
        checked += 1
    return checked


@pytest.mark.parametrize("key", KEYS)
def test_matches_the_model(key):
    seq, o = build_product(key, None, device=0), build_oracle(key, None)
    assert _model_check(seq, o, 3, 6, 2, 61) >= 1


@pytest.mark.parametrize("case", STRUCTURES)
def test_matches_the_model_on_structure_cases(case, tmp_path):
    seq, o = SC.build(SC.BY_ID[case], tmp_path)
    assert _model_check(seq, o, 2, 6, 2, 71) >= 1


def test_writes_stay_inside_their_buffers():
    """Every output is a view with SENTINEL rows before and after it: the sentinels survive, the values are those of the
    library's own buffers."""
    S, L, K = 5, 3, 9
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 81, L)
    st0 = _copy(st)
    tape = seq.make_fixed_lag_tape(S, K, L)
    seq.retarget_fixed_lag(kp, st, fixed_qpos=fx, tape=tape)
    c = _cots(seq, S, K, L, 82)
    args = dict(fixed_qpos=fx, grad_qpos=c["grad_qpos"], grad_robot_qpos=c["grad_robot_qpos"], grad_last_qpos_out=c["last"])
    want = seq.retarget_fixed_lag_vjp(kp, tape, st0, **args)
    n = o.opt_dof
    shapes = dict(grad_keypoints=(S, K, 21, 3), grad_last_qpos=(S, n), grad_window_keypoints=(S, L + 1, 21, 3),
                  grad_window_qpos=(S, L + 1, n), status_out=(S, K))
    bigs, views = {}, {}
    for name, shape in shapes.items():
        dt = torch.int32 if name == "status_out" else torch.float32
        big = torch.full((SENTINEL * 2 + shape[0],) + tuple(shape[1:]), -7, dtype=dt, device=_dev())
        bigs[name], views[name] = big, big[SENTINEL:SENTINEL + shape[0]]
    got = seq.retarget_fixed_lag_vjp(kp, tape, st0, outputs=views, **args)
    for name, big in bigs.items():
        b = _np(big)
        assert (b[:SENTINEL] == -7).all() and (b[-SENTINEL:] == -7).all(), name
    for i in (0, 2, 3, 5, 6):
        assert same_bits(got[i], want[i]) if got[i].dtype == torch.float32 else torch.equal(got[i], want[i])
    assert got[0].data_ptr() == views["grad_keypoints"].data_ptr()
