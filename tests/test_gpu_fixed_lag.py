"""Fixed-lag smoothing on the GPU (`dexr_fixed_lag_step` through SeqRetargeting.retarget_fixed_lag / flush_fixed_lag) on
LEAP DexPilot, Allegro vector and Shadow position streams: every tick is the device smoother (`smooth_packed_sequences`)
on the window rebuilt from the state, bit for bit; L = 0 is the causal minimiser and L >= T - 1 with a flush the offline
one (the float64 model of tests/smooth_cases.py); committed DexPilot flags follow the causal tape; a run split over calls
through a state_dict round trip, or a stream run alone, gives the same bits; the GPU agrees with the host emulation;
outputs and state written into sentinel-framed views stay inside them; the call is asynchronous."""
import numpy as np
import pytest

import seq_vjp_cases as SV
import smooth_cases as SMC
from helpers import build_oracle, build_product

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
STREAMS = 256
CHECKED = 3  # streams the float64 model checks
SENTINEL = 64
STATUS_MAXITER, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 24, 1 << 25, 1 << 27, 1 << 28


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _setup(key, S, T, seed, lag=0, pinch=False):
    seq, o = build_product(key, None, device=0), build_oracle(key, None)
    kp, fx = SV.stream_inputs(o, S, T, seed, pinch=pinch)
    st = seq.make_fixed_lag_state(S, lag)
    rng = np.random.RandomState(seed + 1)
    a = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    st.last_qpos.copy_(_t(a.astype(np.float32)))
    return seq, o, kp, fx, st


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _causal_flags(seq, kp):
    """DexPilot flags after every frame of the causal taped packed solve from fresh flags: [S,T,len_proj] or None."""
    S, T = kp.shape[:2]
    layout = seq.pack_streams([T] * S)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(kp.reshape(-1, 21, 3)), layout, seq.make_stream_state(S), tape=tape)
    return None if tape.projected is None else _np(tape.projected).reshape(S, T, -1)


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("key", KEYS)
def test_each_tick_is_the_device_smoother(key, lag):
    seq, o, kp, fx, st = _setup(key, STREAMS, lag + 2, 11 + lag, lag=lag, pinch=True)
    S = STREAMS
    for k in range(lag + 2):
        snap = {f: None if getattr(st, f) is None else _np(getattr(st, f)).copy() for f in st._FIELDS}
        rq, q, status = seq.retarget_fixed_lag(_t(kp[:, k:k + 1]), st)
        h = snap["window_len"]
        lengths = [int(x) + 1 for x in h]
        wk = np.concatenate([np.concatenate([snap["window_keypoints"][s, :h[s]], kp[s, k:k + 1]]) for s in range(S)])
        wq0 = snap["window_qpos"]
        a0 = snap["last_qpos"]
        wq = np.concatenate([np.concatenate([wq0[s, :h[s]], wq0[s, h[s] - 1:h[s]] if h[s] else a0[s:s + 1]]) for s in range(S)])
        layout = seq.pack_streams(lengths)
        ss = seq.make_stream_state(S)
        ss.last_qpos.copy_(_t(snap["last_qpos"]))
        if ss.projected is not None:
            ss.projected.copy_(_t(snap["projected"]))
        rrq, rq_ref, rst = seq.smooth_packed_sequences(_t(wk), layout, ss, qpos_init=_t(wq))
        rrq, rq_ref, rst = _np(rrq), _np(rq_ref), _np(rst)
        q, rq, status = _np(q), _np(rq), _np(status)
        offs = np.concatenate([[0], np.cumsum(lengths)])
        wnew = _np(st.window_qpos)
        held = min(k + 1, lag)  # frames held after this tick: the last `held` inputs, in order
        np.testing.assert_array_equal(_np(st.window_len), np.full(S, held, np.int32))
        np.testing.assert_array_equal(_np(st.window_keypoints)[:, :held], kp[:, k + 1 - held:k + 1])
        for s in range(S):
            a, b = offs[s], offs[s + 1]
            if h[s] == lag:
                np.testing.assert_array_equal(q[s, 0], rq_ref[a])
                np.testing.assert_array_equal(rq[s, 0], rrq[a])
                assert status[s, 0] == rst[a]
                np.testing.assert_array_equal(wnew[s, :lag], rq_ref[a + 1:b])
            else:
                assert status[s, 0] == STATUS_PENDING and np.isnan(q[s, 0]).all()
                np.testing.assert_array_equal(wnew[s, :b - a], rq_ref[a:b])


@pytest.mark.parametrize("key", KEYS)
def test_lag_zero_is_the_causal_minimiser(key):
    T = 5
    seq, o, kp, fx, st = _setup(key, STREAMS, T, 21, pinch=True)
    a0 = _np(st.last_qpos).copy()
    _, q, status = seq.retarget_fixed_lag(_t(kp), st)
    q, status = _np(q), _np(status)
    assert not (status & (STATUS_PENDING | STATUS_NONFINITE)).any()
    flags = _causal_flags(seq, kp)
    for s in range(CHECKED):
        prev = a0[s]
        for t in range(T):
            m = SMC.Model(o, kp[s, t:t + 1], None, None if flags is None else flags[s, t:t + 1], SMC.clipped_anchor(o, prev),
                          _nd(seq))
            X = q[s, t:t + 1].astype(np.float64)
            assert np.abs(m.polish(X) - X).max() <= SMC.PARITY, (s, t)
            prev = q[s, t]


@pytest.mark.parametrize("key", KEYS)
def test_full_lag_and_flush_is_the_offline_smoother(key):
    T, lag = 6, 5
    seq, o, kp, fx, st = _setup(key, STREAMS, T, 31, pinch=True)
    st = seq.make_fixed_lag_state(STREAMS, lag)
    a0 = _np(st.last_qpos).copy()
    _, q, status = seq.retarget_fixed_lag(_t(kp), st)
    _, fq, count = seq.flush_fixed_lag(st)
    q, status, fq, count = _np(q), _np(status), _np(fq), _np(count)
    assert ((status[:, :lag] == STATUS_PENDING).all() and (count == lag).all())
    assert (_np(st.window_len) == 0).all()
    flags = _causal_flags(seq, kp)
    checked = 0
    for s in range(STREAMS):
        if status[s, lag] & STATUS_MAXITER:
            continue
        X = np.concatenate([q[s, lag:], fq[s]]).astype(np.float64)
        m = SMC.Model(o, kp[s], None, None if flags is None else flags[s], SMC.clipped_anchor(o, a0[s]), _nd(seq))
        assert np.abs(m.polish(X) - X).max() <= SMC.PARITY, s
        checked += 1
        if checked == CHECKED:
            break
    assert checked == CHECKED
    if flags is not None:
        np.testing.assert_array_equal(_np(st.projected), flags[:, -1])


def test_committed_flags_follow_the_causal_tape():
    T, lag = 6, 1
    seq, o, kp, fx, st = _setup(KEYS[0], STREAMS, T, 41, lag=lag, pinch=True)
    flags = _causal_flags(seq, kp)
    assert flags.any() and not flags.all()
    for k in range(T):
        seq.retarget_fixed_lag(_t(kp[:, k:k + 1]), st)
        if k >= lag:
            np.testing.assert_array_equal(_np(st.projected), flags[:, k - lag])


@pytest.mark.parametrize("key", KEYS)
def test_splitting_and_neighbours_change_no_bit(key):
    T, lag = 8, 3
    seq, o, kp, fx, st = _setup(key, STREAMS, T, 51, lag=lag)
    j = min(7, STREAMS - 1)  # the stream with a dropped frame, also run alone
    kp[j, 4] = np.nan
    d0 = st.state_dict()
    rq1, q1, s1 = (_np(x) for x in seq.retarget_fixed_lag(_t(kp), st))
    f1 = [_np(x) for x in seq.flush_fixed_lag(st)]
    from dex_retargeting_b200.seq_retarget import FixedLagState

    st2 = FixedLagState.from_state_dict(d0, device=_dev())
    parts = []
    for a, b in ((0, 3), (3, 8)):
        parts.append([_np(x) for x in seq.retarget_fixed_lag(_t(kp[:, a:b]), st2)])
        st2 = FixedLagState.from_state_dict(st2.state_dict(), device=_dev())
    f2 = [_np(x) for x in seq.flush_fixed_lag(st2)]
    for i, ref in enumerate((rq1, q1, s1)):
        np.testing.assert_array_equal(np.concatenate([p[i] for p in parts], axis=1), ref)
    for x, y in zip(f1, f2):
        np.testing.assert_array_equal(x, y)
    assert (s1[j] & STATUS_MISSING).any()
    # stream j alone
    one = FixedLagState.from_state_dict({k: (v if not hasattr(v, "shape") else v[j:j + 1]) for k, v in d0.items()},
                                        device=_dev())
    rqj, qj, sj = (_np(x) for x in seq.retarget_fixed_lag(_t(kp[j:j + 1]), one))
    np.testing.assert_array_equal(qj[0], q1[j])
    np.testing.assert_array_equal(sj[0], s1[j])


@pytest.mark.parametrize("key", KEYS[:2])
def test_gpu_matches_the_emulation(key):
    """The same seeded streams through the device and the host emulation: status words exactly, outputs and state to
    within the device's last bits, the window keypoints and counts exactly."""
    import emu_fixed_lag_host as FL

    T, lag = 5, 2
    seq, o, kp, fx, st = _setup(key, 4, T, 61, lag=lag)
    kp[1, 2] = np.nan
    es = FL.fresh_state(seq, 4, lag)
    es["last_qpos"][...] = _np(st.last_qpos)
    rq, q, status = (_np(x) for x in seq.retarget_fixed_lag(_t(kp), st))
    r = FL.fixed_lag_step(seq, kp, es)
    np.testing.assert_array_equal(status, r["status"])
    np.testing.assert_allclose(q, r["qpos"], atol=1e-4)
    np.testing.assert_allclose(rq, r["robot_qpos"], atol=1e-4)
    np.testing.assert_allclose(_np(st.last_qpos), es["last_qpos"], atol=1e-4)
    np.testing.assert_allclose(_np(st.window_qpos)[:, :lag], es["window_qpos"][:, :lag], atol=1e-4)
    np.testing.assert_array_equal(_np(st.window_keypoints)[:, :lag], es["window_keypoints"][:, :lag])
    np.testing.assert_array_equal(_np(st.window_len), es["window_len"])
    if st.projected is not None:
        np.testing.assert_array_equal(_np(st.projected), es["projected"])


@pytest.mark.parametrize("case", ["teleop/leap_hand_right_dexpilot", "mimic_fixed_dense32"])
def test_writes_stay_inside_their_buffers(case, tmp_path):
    """Every output and every state array is a view with SENTINEL rows before and after it, through ticks that fill and
    shift the window and a flush, on a DexPilot robot (flags) and one with fixed joints: the sentinels survive."""
    import structure_cases as SC

    S, K, lag = 8, 5, 2
    if "/" in case:
        seq, o = build_product(case, None, device=0), build_oracle(case, None)
    else:
        seq, o = SC.build(SC.BY_ID[case], tmp_path)
    kp, fx = SV.stream_inputs(o, S, K, 71, pinch=True)
    st = seq.make_fixed_lag_state(S, lag)

    def framed(t):
        fill = 0xAB if t.dtype == torch.uint8 else -7
        big = torch.full((SENTINEL * 2 + t.shape[0],) + tuple(t.shape[1:]), fill, dtype=t.dtype, device=_dev())
        v = big[SENTINEL:SENTINEL + t.shape[0]]
        v.copy_(t)
        return (big, fill), v

    bigs = []
    for f in st._FIELDS:
        if getattr(st, f) is not None:
            big, v = framed(getattr(st, f))
            bigs.append(big)
            setattr(st, f, v)
    assert (st.projected is not None) == ("dexpilot" in case) and (st.window_fixed_qpos is not None) == ("fixed" in case)
    n, dof = seq.optimizer.opt_dof, seq.optimizer.robot.dof

    def out(shape, dtype=torch.float32):
        big, v = framed(torch.zeros(shape, dtype=dtype, device=_dev()))
        bigs.append(big)
        return v

    seq.retarget_fixed_lag(_t(kp), st, fixed_qpos=_t(fx), out=out((S, K, dof)), qpos_out=out((S, K, n)),
                           status_out=out((S, K), torch.int32))
    fo, fq, fc = out((S, lag, dof)), out((S, lag, n)), out((S,), torch.int32)
    seq.flush_fixed_lag(st, out=fo, qpos_out=fq, count_out=fc)
    torch.cuda.synchronize()
    assert (_np(fc) == lag).all()
    for b, fill in bigs:
        assert (b[:SENTINEL] == fill).all() and (b[-SENTINEL:] == fill).all()


def test_call_is_asynchronous():
    seq, o, kp, fx, st = _setup(KEYS[1], 64, 4, 81)
    x = _t(kp)
    torch.cuda.synchronize()
    s = torch.cuda.current_stream()
    torch.cuda._sleep(200_000_000)  # keep the stream busy: a synchronising call would wait for it
    e = torch.cuda.Event()
    seq.retarget_fixed_lag(x, st)
    e.record(s)
    assert not e.query()
    torch.cuda.synchronize()
