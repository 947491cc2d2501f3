"""Fixed-lag smoothing with an acceleration penalty on the GPU (`dexr_fixed_lag_step_accel` through
SeqRetargeting.retarget_fixed_lag / flush_fixed_lag on a state made with accel_weight) on LEAP DexPilot, Allegro vector and
Shadow position streams and on structure cases with fixed, mimic and prismatic joints: each window answer is the float64
minimiser of tests/fixed_lag_accel_cases.py at L = 0, 1, 4; a
fresh stream with L >= T - 1 and a flush is `smooth_packed_sequences(..., accel_weight=c)` bit for bit; a run split over
calls through state_dict round trips, or a stream run alone, gives the same bits; the GPU agrees with the host emulation;
outputs and state written into sentinel-framed views stay inside them; the call is asynchronous; the backward entry points
refuse accelerated states."""
import numpy as np
import pytest

import fixed_lag_accel_cases as FAC
import seq_vjp_cases as SV
import structure_cases as SC
from helpers import build_oracle, build_product

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
STRUCTURES = ["fixed_dense16", "mimic_dense16", "mimic_fixed_dense32", "prismatic_arrow"]
# streams per call and how many of them the float64 model checks.  The CPU dry run (tests/tools/emu_gpu_fixed_lag_accel.py)
# shrinks them.
STREAMS = 256
CHECKED = 3  # streams the float64 model checks
SENTINEL = 64
C_OVER_W = 10.0
STATUS_MAXITER, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 24, 1 << 25, 1 << 27, 1 << 28


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _setup(key, S, T, seed, lag=0, pinch=False, tmp_path=None):
    """A packaged config (key) or a structure case (tmp_path given), its inputs and a fresh accelerated state."""
    if tmp_path is None:
        seq, o = build_product(key, None, device=0), build_oracle(key, None)
    else:
        seq, o = SC.build(SC.BY_ID[key], tmp_path)
    kp, fx = SV.stream_inputs(o, S, T, seed, pinch=pinch)
    st = seq.make_fixed_lag_state(S, lag, accel_weight=C_OVER_W * _nd(seq))
    rng = np.random.RandomState(seed + 1)
    a = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    st.last_qpos.copy_(_t(a.astype(np.float32)))
    return seq, o, kp, fx, st


def _causal_flags(seq, kp, fx=None):
    S, T = kp.shape[:2]
    layout = seq.pack_streams([T] * S)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(kp.reshape(-1, 21, 3)), layout, seq.make_stream_state(S), tape=tape,
                                  fixed_qpos=None if fx is None else _t(fx.reshape(S * T, -1)))
    return None if tape.projected is None else _np(tape.projected).reshape(S, T, -1)


def _snap(st):
    return {f: None if getattr(st, f) is None else _np(getattr(st, f)).copy() for f in st._FIELDS}


def _window_model(seq, o, st, kp, fx, lag, case):
    """Tick by tick, the window the state holds after each tick is the float64 minimiser of its window problem (fixed
    joints passed through), the pre-anchor triple included once a frame has been committed."""
    K = kp.shape[1]
    c = float(st.accel_weight)
    flags = _causal_flags(seq, kp, fx)
    checked = 0
    for k in range(K):
        snap = _snap(st)
        _, q, status = seq.retarget_fixed_lag(_t(kp[:, k:k + 1]), st,
                                              fixed_qpos=None if fx is None else _t(fx[:, k:k + 1]))
        q, status = _np(q), _np(status)
        wq = _np(st.window_qpos)
        for s in range(CHECKED):
            h = int(snap["window_len"][s])
            m_ = h + 1
            X = np.concatenate([q[s, :1], wq[s, :lag]]) if h == lag else wq[s, :m_]
            if status[s, 0] & (STATUS_MAXITER | STATUS_NONFINITE):
                continue
            wk = np.concatenate([snap["window_keypoints"][s, :h], kp[s, k:k + 1]])
            wf = None if fx is None else np.concatenate([snap["window_fixed_qpos"][s, :h], fx[s, k:k + 1]])
            pre = FAC.clipped(o, snap["prev_qpos"][s]) if snap["has_prev"][s] else None
            m = FAC.Model(o, wk, wf, None if flags is None else flags[s, k + 1 - m_:k + 1],
                          FAC.clipped(o, snap["last_qpos"][s]), _nd(seq), c, pre)
            X = X.astype(np.float64)
            assert np.abs(m.polish(X) - X).max() <= FAC.PARITY, (case, k, s)
            checked += 1
    assert checked >= CHECKED * K // 2
    assert (_np(st.has_prev) == 1).all()


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("key", KEYS)
def test_each_window_is_the_model_minimiser(key, lag):
    seq, o, kp, fx, st = _setup(key, STREAMS, lag + 3, 211 + lag, lag=lag, pinch=True)
    _window_model(seq, o, st, kp, fx, lag, key)


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("case", STRUCTURES)
def test_structure_windows_are_the_model_minimiser(case, lag, tmp_path):
    """As above on robots with fixed joints (fixed_qpos passed through every tick), mimic joints (the pre-anchor's +2c on
    the diagonal of a mimic source) and prismatic joints, at 16 and 32 lanes."""
    seq, o, kp, fx, st = _setup(case, STREAMS, lag + 3, 221 + lag, lag=lag, tmp_path=tmp_path)
    assert fx is not None or "fixed" not in case
    _window_model(seq, o, st, kp, fx, lag, case)


@pytest.mark.parametrize("key", KEYS)
def test_full_lag_and_flush_is_the_offline_accel_smoother(key):
    T, lag = 6, 5
    seq, o, kp, fx, st = _setup(key, STREAMS, T, 231, lag=lag, pinch=True)
    kp[:, 2] = np.nan
    a0 = _np(st.last_qpos).copy()
    seq.retarget_fixed_lag(_t(kp[:, :T - 1]), st)
    # the last tick's solve is the whole clip, started from the window it holds plus the appended frame
    w = _np(st.window_qpos)
    wq = np.concatenate([w[:, :T - 1], w[:, T - 2:T - 1]], axis=1).reshape(-1, w.shape[-1])
    _, q, status = seq.retarget_fixed_lag(_t(kp[:, T - 1:]), st)
    _, fq, count = seq.flush_fixed_lag(st)
    q, status, fq, count = _np(q), _np(status), _np(fq), _np(count)
    assert (count == T - 1).all()
    X = np.concatenate([q[:, -1:], fq[:, :T - 1]], axis=1)
    layout = seq.pack_streams([T] * STREAMS)
    ss = seq.make_stream_state(STREAMS)
    ss.last_qpos.copy_(_t(a0))
    _, ref, rst = seq.smooth_packed_sequences(_t(kp.reshape(-1, 21, 3)), layout, ss, qpos_init=_t(wq),
                                              accel_weight=float(st.accel_weight))
    np.testing.assert_array_equal(X.reshape(-1, X.shape[-1]), _np(ref))
    np.testing.assert_array_equal(status[:, -1], _np(rst).reshape(STREAMS, T)[:, 0])
    np.testing.assert_array_equal(_np(st.prev_qpos), X[:, -2])
    np.testing.assert_array_equal(_np(st.last_qpos), X[:, -1])


@pytest.mark.parametrize("key", KEYS[:2])
def test_splitting_and_neighbours_are_invisible(key):
    """One call against three calls through state_dict round trips and a flush-only call; a middle stream alone."""
    from dex_retargeting_b200.seq_retarget import FixedLagState

    K, lag = 7, 2
    seq, o, kp, fx, st0 = _setup(key, STREAMS, K, 241, lag=lag)
    mid = STREAMS // 2
    kp[mid, 3] = np.nan
    d0 = st0.state_dict()
    assert {"accel_weight", "prev_qpos", "has_prev"} <= set(d0)
    st = FixedLagState.from_state_dict(d0, device=_dev())
    _, q1, s1 = seq.retarget_fixed_lag(_t(kp), st)
    _, f1, c1 = seq.flush_fixed_lag(st)
    sp = FixedLagState.from_state_dict(d0, device=_dev())
    parts = []
    for a, b in ((0, 2), (2, 5), (5, 7)):
        _, q, s = seq.retarget_fixed_lag(_t(kp[:, a:b]), sp)
        parts.append((_np(q), _np(s)))
        sp = FixedLagState.from_state_dict(sp.state_dict(), device=_dev())
    _, f2, c2 = seq.flush_fixed_lag(sp)
    np.testing.assert_array_equal(np.concatenate([p[0] for p in parts], 1), _np(q1))
    np.testing.assert_array_equal(np.concatenate([p[1] for p in parts], 1), _np(s1))
    np.testing.assert_array_equal(_np(f2), _np(f1))
    for k, v in st.state_dict().items():
        if isinstance(v, torch.Tensor):
            np.testing.assert_array_equal(_np(sp.state_dict()[k]), _np(v), err_msg=k)
    alone = FixedLagState.from_state_dict({k: (v[mid:mid + 1] if isinstance(v, torch.Tensor) else v) for k, v in d0.items()},
                                          device=_dev())
    _, qa, sa = seq.retarget_fixed_lag(_t(kp[mid:mid + 1]), alone)
    np.testing.assert_array_equal(_np(qa), _np(q1)[mid:mid + 1])
    np.testing.assert_array_equal(_np(sa), _np(s1)[mid:mid + 1])


@pytest.mark.parametrize("key", KEYS)
def test_gpu_matches_the_emulation(key):
    import emu_fixed_lag_accel_host as FA

    K, lag, S = 5, 2, 4
    seq, o, kp, fx, st = _setup(key, S, K, 251, lag=lag, pinch=True)
    es = FA.fresh_state(seq, S, lag, float(st.accel_weight))
    es["last_qpos"][...] = _np(st.last_qpos)
    _, q, status = seq.retarget_fixed_lag(_t(kp), st)
    _, fq, count = seq.flush_fixed_lag(st)
    r = FA.fixed_lag_step(seq, kp, es, flush=True)
    for got, want in ((q, r["qpos"]), (fq, r["flush_qpos"]), (count, r["flush_count"])):
        got = _np(got)
        assert got.shape == want.shape
        assert np.allclose(got, want, atol=2e-5, equal_nan=True), np.nanmax(np.abs(got - want))
    # the status flags agree; the iteration counts in the low bits may differ by the GPU's last-bit arithmetic
    flags = ~np.int32(0x7fffff)
    np.testing.assert_array_equal(_np(status) & flags, r["status"] & flags)
    for k in ("last_qpos", "prev_qpos", "has_prev", "window_len"):
        assert np.allclose(_np(getattr(st, k)), es[k], atol=2e-5), k


def test_writes_stay_inside_their_buffers():
    """Outputs and every state array, the new ones included, as views inside sentinel-framed buffers."""
    from dex_retargeting_b200.seq_retarget import FixedLagState

    K, lag, S = 4, 1, 32
    seq, o, kp, fx, st = _setup(KEYS[0], S, K, 261, lag=lag, pinch=True)

    def framed(t):
        buf = torch.full((t.numel() + 2 * SENTINEL,), -7, dtype=t.dtype, device=t.device) if t.dtype != torch.uint8 else \
            torch.full((t.numel() + 2 * SENTINEL,), 0xAB, dtype=t.dtype, device=t.device)
        v = buf[SENTINEL:SENTINEL + t.numel()].view(t.shape)
        v.copy_(t)
        return buf, v

    bufs = {}
    fields = {}
    for f in st._FIELDS:
        t = getattr(st, f)
        if t is not None:
            bufs[f] = framed(t)
            fields[f] = bufs[f][1]
    fs = FixedLagState(lag=lag, accel_weight=st.accel_weight, **{f: fields.get(f) for f in st._FIELDS})
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    ob = {k: framed(torch.empty(shape, dtype=dt, device=_dev())) for k, shape, dt in
          (("out", (S, K, dof), torch.float32), ("qpos", (S, K, n), torch.float32), ("status", (S, K), torch.int32),
           ("fout", (S, lag, dof), torch.float32), ("fq", (S, lag, n), torch.float32), ("count", (S,), torch.int32))}
    seq.retarget_fixed_lag(_t(kp), fs, out=ob["out"][1], qpos_out=ob["qpos"][1], status_out=ob["status"][1])
    seq.flush_fixed_lag(fs, out=ob["fout"][1], qpos_out=ob["fq"][1], count_out=ob["count"][1])
    torch.cuda.synchronize()
    for name, (buf, _) in list(bufs.items()) + list(ob.items()):
        head, tail = _np(buf[:SENTINEL]), _np(buf[-SENTINEL:])
        want = 0xAB if buf.dtype == torch.uint8 else -7
        assert (head == want).all() and (tail == want).all(), name
    assert (_np(fs.has_prev) == 1).all()


def test_calls_are_asynchronous():
    seq, o, kp, fx, st = _setup(KEYS[1], STREAMS, 8, 271, lag=4)
    kpt = _t(kp)
    seq.retarget_fixed_lag(kpt, st)  # (warm-up: module load)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        seq.retarget_fixed_lag(kpt, st, stream=side)
        seq.flush_fixed_lag(st, stream=side)
        assert not side.query()
    side.synchronize()


def test_backward_refuses_accelerated_states():
    from dex_retargeting_b200.objective import differentiable_flush_fixed_lag, differentiable_retarget_fixed_lag

    K, lag, S = 3, 1, 4
    seq, o, kp, fx, st = _setup(KEYS[1], S, K, 281, lag=lag)
    st0 = seq.make_fixed_lag_state(S, lag, accel_weight=float(st.accel_weight))
    with pytest.raises(ValueError, match="backward"):
        seq.retarget_fixed_lag(_t(kp), st, tape=seq.make_fixed_lag_tape(S, K, lag))
    with pytest.raises(ValueError, match="backward"):
        seq.retarget_fixed_lag_vjp(_t(kp), seq.make_fixed_lag_tape(S, K, lag), st0)
    with pytest.raises(ValueError, match="backward"):
        seq.flush_fixed_lag_vjp(st0)
    with pytest.raises(ValueError, match="backward"):
        differentiable_retarget_fixed_lag(seq, _t(kp).requires_grad_(), st0)
    with pytest.raises(ValueError, match="backward"):
        differentiable_flush_fixed_lag(seq, st0)
    # a c = 0 state is today's: no new fields, the same checkpoint keys
    plain = seq.make_fixed_lag_state(S, lag, accel_weight=0.0)
    assert plain.prev_qpos is None and plain.has_prev is None
    assert set(plain.state_dict()) == set(seq.make_fixed_lag_state(S, lag).state_dict())
    with pytest.raises(ValueError, match="accel_weight"):
        seq.make_fixed_lag_state(S, lag, accel_weight=-1.0)
