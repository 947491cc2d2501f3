"""Backpropagation through acceleration-penalised fixed-lag smoothing (`dexr_fixed_lag_step_accel_vjp`) through the host
emulation of the kernels' own code (tests/emu runs fixed_lag_tick<G, true, true> and the fixed_lag_vjp_* helpers with ACC
and smooth_vjp_packed_stream<G, true, true> of dexr_kernels.cuh on the fiber warp): the float64 model of
tests/fixed_lag_accel_vjp_cases.py, itself checked against central differences of the chain re-polished in float64 tick by
tick; recording changes no bit; a fresh stream with L >= K - 1 and a flush is the offline accel VJP bit for bit; chunks
chained through the state cotangents give the bits of one call; one window's anchor and pre-anchor cotangents; a NOT_PD
window lets the later window's pre-anchor cotangent through; missing frames; a non-finite prev_qpos; causality; the
argument checks, the workspace size, the struct sizes, the register budget and a dry run of
tests/test_gpu_fixed_lag_accel_vjp.py."""
import ctypes as C
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_fixed_lag_accel_host as FA
import emu_fixed_lag_accel_vjp_host as AV
import emu_smooth_accel_host as SA
import fixed_lag_accel_vjp_cases as FAV
import fixed_lag_vjp_cases as FLC
import seq_vjp_cases as SV
import structure_cases as SC
from emu_eval_host import EmulationError
from test_fixed_lag_emulation import CASES as ALL_CASES, _setup
from test_fixed_lag_vjp_emulation import _flags, _nd, same_bits

ROOT = Path(__file__).resolve().parent.parent
STATUS_NOT_PD, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 26, 1 << 25, 1 << 27, 1 << 28
CASES = [c for c in ALL_CASES if c[0] in ("leap_dexpilot", "allegro_vector", "mimic_dense16", "mimic_fixed_dense32")]
IDS = [c[0] for c in CASES]
C_OVER_W = 10.0


def _state(seq, o, S, lag, seed, c, has_prev=0):
    """An accelerated state with an empty window, a seeded anchor and (has_prev = 1) pre-anchor inside the limits."""
    st = FA.fresh_state(seq, S, lag, c)
    rng = np.random.RandomState(seed)
    lo, hi = o.joint_limits[:, 0], o.joint_limits[:, 1]
    st["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), lo, hi)
    if has_prev:
        st["prev_qpos"][...] = np.clip(st["last_qpos"] + 0.05 * rng.randn(S, o.opt_dof), lo, hi)
        st["has_prev"][...] = 1
    return st


def _copy(st):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}


def _cot(rng, shape):
    return rng.randn(*shape).astype(np.float32)


def _run(seq, kp, fx, st, flush=False):
    st0 = _copy(st)
    return st0, AV.fixed_lag_step_accel_tape(seq, kp, st, fixed_qpos=fx, flush=flush)


def _vjp(seq, kp, fx, st0, r, flushed=False, **g):
    return AV.fixed_lag_accel_vjp(seq, kp, st0, r["tape_qpos"], r["tape_projected"], fixed_qpos=fx, flushed=flushed, **g)


def _windows(r, s, L):
    return [r["tape_qpos"][s, k, :FLC.window(k, L)[1]] for k in range(r["tape_qpos"].shape[1])]


def _model(seq, o, kp, fx, fl, st0, r, L, gq, grq, s, Xs=None, glast=None, gprev=None):
    return FAV.model_chain(o, _nd(seq), st0["accel_weight"], kp[s].astype(np.float64),
                           None if fx is None else fx[s].astype(np.float64), None if fl is None else fl[s],
                           st0["last_qpos"][s].astype(np.float64), st0["prev_qpos"][s].astype(np.float64),
                           int(st0["has_prev"][s]), _windows(r, s, L) if Xs is None else Xs, L, gq[s], grq[s],
                           None if glast is None else glast[s], None if gprev is None else gprev[s])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_recording_changes_no_bit(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    S, L, K = 2, 2, 5
    kp, fx = SV.stream_inputs(o, S, K, 5)
    a = _state(seq, o, S, L, 6, C_OVER_W * _nd(seq), has_prev=1)
    b = _copy(a)
    r = FA.fixed_lag_step(seq, kp, a, fixed_qpos=fx, flush=True)
    t = AV.fixed_lag_step_accel_tape(seq, kp, b, fixed_qpos=fx, flush=True)
    for k in r:
        assert same_bits(r[k], t[k]), k
    for k in FA.STATE:
        if a.get(k) is not None:
            assert np.array_equal(a[k], b[k]), k
    assert same_bits(t["tape_qpos"][:, -1, 1:L + 1], t["flush_qpos"][:, :L])


@pytest.mark.parametrize("K,L", [(5, 4), (5, 6), (2, 1), (1, 1)], ids=["K5-L4", "K5-L6", "K2-L1", "K1-L1"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_full_lag_is_the_offline_accel_vjp(case, K, L, tmp_path):
    """A fresh stream, L >= K - 1, ticks then a flush in one call: dexr_smooth_sequences_packed_accel_vjp of the whole clip
    at the last window, bit for bit (no window sees a pre-anchor).  The final prev_qpos is the second-to-last flushed row,
    or, with K = 2 and L = 1, the frame the last tick emitted (slot 0 of the last window), or, with K = 1 and L = 1, the
    incoming anchor (grad_prev_qpos_out is then added to grad_last_qpos)."""
    seq, o = _setup(case, tmp_path)
    S = 2
    c = C_OVER_W * _nd(seq)
    kp, fx = SV.stream_inputs(o, S, K, 11)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 12, c), flush=True)
    rng = np.random.RandomState(13)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    gq, gr = _cot(rng, (S, K, n)), _cot(rng, (S, K, dof))
    gfq, gfr = _cot(rng, (S, L, n)), _cot(rng, (S, L, dof))
    glast, gprev = _cot(rng, (S, n)), _cot(rng, (S, n))
    got = _vjp(seq, kp, fx, st0, r, flushed=True, grad_qpos=gq, grad_robot_qpos=gr, grad_flush_qpos=gfq,
               grad_flush_robot_qpos=gfr, grad_last_qpos_out=glast, grad_prev_qpos_out=gprev)
    e = 1 if L == K - 1 else 0
    cq = np.concatenate([gq[:, K - 1:K] if e else np.zeros((S, 0, n), np.float32), gfq[:, :K - e]], 1)
    cr = np.concatenate([gr[:, K - 1:K] if e else np.zeros((S, 0, dof), np.float32), gfr[:, :K - e]], 1)
    cq[:, -1] += glast
    if K > 1:
        cq[:, -2] += gprev
    X = r["tape_qpos"][:, K - 1, :K]
    gk, gf, gl, status = SA.smooth_vjp_packed(seq, kp.reshape(S * K, 21, 3), np.arange(S + 1) * K, X.reshape(S * K, n), c,
                                              last_qpos=st0["last_qpos"], projected=st0["projected"],
                                              fixed_qpos=None if fx is None else fx.reshape(S * K, -1),
                                              grad_qpos=cq.reshape(S * K, n), grad_robot_qpos=cr.reshape(S * K, dof))
    assert same_bits(got["grad_keypoints"], gk.reshape(S, K, 21, 3))
    if fx is not None:
        assert same_bits(got["grad_fixed_qpos"], gf.reshape(S, K, -1))
    assert same_bits(got["grad_last_qpos"], gl if K > 1 else gprev + gl)
    assert (got["grad_prev_qpos"] == 0).all()
    assert not np.isnan(got["grad_keypoints"]).any()


def _chain(seq, kp, fx, st, cuts, g):
    """The run of `kp` split at `cuts` then a flush-only call, each chunk's VJP fed the next one's state cotangents;
    returns the per-frame keypoint and fixed gradients [S,K] and the first state's cotangents."""
    K = kp.shape[1]
    bounds = [0] + list(cuts) + [K]
    calls = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        calls.append((a, b, *_run(seq, kp[:, a:b], None if fx is None else fx[:, a:b], st)))
    st0 = _copy(st)
    AV.fixed_lag_step_accel_tape(seq, None, st, flush=True)
    carry = AV.fixed_lag_accel_vjp(seq, None, st0, None, None, flushed=True, grad_flush_qpos=g["grad_flush_qpos"],
                                   grad_flush_robot_qpos=g["grad_flush_robot_qpos"],
                                   grad_last_qpos_out=g["grad_last_qpos_out"], grad_prev_qpos_out=g["grad_prev_qpos_out"])
    gks, gfs = [], []
    for a, b, st0, r in reversed(calls):
        out = _vjp(seq, kp[:, a:b], None if fx is None else fx[:, a:b], st0, r, grad_qpos=g["grad_qpos"][:, a:b],
                   grad_robot_qpos=g["grad_robot_qpos"][:, a:b], grad_last_qpos_out=carry["grad_last_qpos"],
                   grad_prev_qpos_out=carry["grad_prev_qpos"], grad_window_qpos_out=carry["grad_window_qpos"],
                   grad_window_keypoints_out=carry["grad_window_keypoints"],
                   grad_window_fixed_qpos_out=carry["grad_window_fixed_qpos"])
        gks.insert(0, out["grad_keypoints"])
        gfs.insert(0, out["grad_fixed_qpos"])
        carry = out
    return np.concatenate(gks, 1), np.concatenate(gfs, 1), carry


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_chunks_give_the_bits_of_one_call(case, tmp_path):
    """K ticks then a flush in one call equal three chunks and a flush-only call, bit for bit.  The run starts with
    has_prev = 1 and a partly filled window (2 of L = 3 held); tick 1 commits the first frame, so the chunk starting at
    tick 2 begins right after it (c_k = 1 there in the one call)."""
    seq, o = _setup(case, tmp_path)
    S, L, K = 2, 3, 8
    kp, fx = SV.stream_inputs(o, S, K + 2, 21)
    pre = _state(seq, o, S, L, 22, C_OVER_W * _nd(seq), has_prev=1)
    FA.fixed_lag_step(seq, kp[:, :2], pre, fixed_qpos=None if fx is None else fx[:, :2])
    assert (pre["window_len"] == 2).all() and (pre["has_prev"] == 1).all()
    kp, fx = kp[:, 2:], None if fx is None else fx[:, 2:]
    rng = np.random.RandomState(23)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    g = dict(grad_qpos=_cot(rng, (S, K, n)), grad_robot_qpos=_cot(rng, (S, K, dof)), grad_flush_qpos=_cot(rng, (S, L, n)),
             grad_flush_robot_qpos=_cot(rng, (S, L, dof)), grad_last_qpos_out=_cot(rng, (S, n)),
             grad_prev_qpos_out=_cot(rng, (S, n)))
    st0, r = _run(seq, kp, fx, _copy(pre), flush=True)
    want = _vjp(seq, kp, fx, st0, r, flushed=True, **g)
    gk, gf, first = _chain(seq, kp, fx, _copy(pre), [2, 5], g)
    assert same_bits(gk, want["grad_keypoints"])
    assert same_bits(gf, want["grad_fixed_qpos"])
    for k in ("grad_last_qpos", "grad_prev_qpos", "grad_window_keypoints", "grad_window_fixed_qpos", "grad_window_qpos"):
        assert same_bits(first[k], want[k]), k
    assert not np.isnan(want["grad_keypoints"]).any()
    assert (want["grad_prev_qpos"] != 0).any() and (want["grad_window_keypoints"][:, :2] != 0).any()


@pytest.mark.parametrize("clipped", [False, True], ids=["p_inside", "p_clipped"])
def test_pre_window_cotangents_match_the_model(clipped, tmp_path):
    """One emitting window with a pre-anchor (L = 2, K = 3, has_prev = 1): its keypoint, anchor and pre-anchor cotangents
    against the model; with p outside the clip range the pre-anchor's cotangent is exactly 0."""
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 2, 2, 3
    kp, fx = SV.stream_inputs(o, S, K, 31)
    st = _state(seq, o, S, L, 32, C_OVER_W * _nd(seq), has_prev=1)
    if clipped:
        st["prev_qpos"][:, ::2] = o.joint_limits[::2, 1] + 0.3
    st0, r = _run(seq, kp, fx, st)
    rng = np.random.RandomState(33)
    gq, grq = _cot(rng, (S, K, o.opt_dof)), _cot(rng, (S, K, seq.optimizer.robot.dof))
    got = _vjp(seq, kp, fx, st0, r, grad_qpos=gq, grad_robot_qpos=grq)
    assert got["status"][0, K - 1] == 0
    for s in range(S):
        md = _model(seq, o, kp, fx, None, st0, r, L, gq, grq, s)
        FAV.compare(got["grad_keypoints"][s], got["grad_fixed_qpos"][s], got["grad_last_qpos"][s], got["grad_prev_qpos"][s],
                    md)
    if clipped:
        assert (got["grad_prev_qpos"][:, ::2] == 0).all() and (got["grad_prev_qpos"][:, 1::2] != 0).any()
    else:
        assert (got["grad_prev_qpos"] != 0).all()


def test_not_pd_window_lets_the_later_pre_anchor_cotangent_through(tmp_path):
    """Window k - 1 made NOT_PD (its tape point replaced by one far from any minimum) contributes zero, but window k's
    pre-anchor cotangent skips over it: a loss on tick k's row alone still reaches frame k - 3, which only window k - 2
    holds (L = 1)."""
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K, k = 1, 1, 7, 5
    kp, fx = SV.stream_inputs(o, S, K, 91)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 92, C_OVER_W * _nd(seq), has_prev=1))
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    gq[0, k] = 1.0
    rng = np.random.RandomState(93)
    lo, hi = o.joint_limits[:, 0], o.joint_limits[:, 1]
    for _ in range(50):
        bad = dict(r)
        bad["tape_qpos"] = r["tape_qpos"].copy()
        bad["tape_qpos"][0, k - 1, :L + 1] = lo + (hi - lo) * rng.rand(L + 1, o.opt_dof)
        out = _vjp(seq, kp, fx, st0, bad, grad_qpos=gq)
        if out["status"][0, k - 1] & STATUS_NOT_PD:
            break
    else:
        pytest.fail("no NOT_PD window found")
    assert not out["status"][0, k] & STATUS_NOT_PD
    reach = np.abs(out["grad_keypoints"][0]).reshape(K, -1).max(1)
    assert reach[k - 3] > 0, reach  # (frame k - 3 is in windows k - 3 and k - 2 only)
    assert (reach[k + 1:] == 0).all()
    assert np.isfinite(out["grad_keypoints"]).all()


def test_missing_frame_carries_the_chain(tmp_path):
    seq, o = _setup(CASES[3], tmp_path)
    S, L, K = 1, 2, 7
    kp, fx = SV.stream_inputs(o, S, K, 101)
    kp[0, 3] = np.nan
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 102, C_OVER_W * _nd(seq), has_prev=1))
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    grq = np.zeros((S, K, seq.optimizer.robot.dof), np.float32)
    gq[0, K - 1] = np.random.RandomState(103).randn(o.opt_dof)
    out = _vjp(seq, kp, fx, st0, r, grad_qpos=gq, grad_robot_qpos=grq)
    assert out["status"][0, 5] & STATUS_MISSING
    assert (out["grad_keypoints"][0, 3] == 0).all() and np.isfinite(out["grad_keypoints"]).all()
    assert all(np.abs(out["grad_keypoints"][0, t]).max() > 0 for t in (1, 2, 4))
    md = _model(seq, o, kp, fx, _flags(seq, np.nan_to_num(kp), fx), st0, r, L, gq, grq, 0)
    FAV.compare(out["grad_keypoints"][0], out["grad_fixed_qpos"][0], out["grad_last_qpos"][0], out["grad_prev_qpos"][0], md)


def test_non_finite_prev_qpos_is_nan_and_confined(tmp_path):
    """A NaN prev_qpos with has_prev = 1: the first emitting window is non-finite, so its cotangents, the anchor's and the
    pre-anchor's are NaN; the other stream's bits are those of a run without the NaN."""
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 2, 1, 5
    kp, fx = SV.stream_inputs(o, S, K, 41)
    st = _state(seq, o, S, L, 42, C_OVER_W * _nd(seq), has_prev=1)
    g = dict(grad_qpos=np.ones((S, K, o.opt_dof), np.float32), grad_prev_qpos_out=np.ones((S, o.opt_dof), np.float32))
    st0, r = _run(seq, kp, fx, _copy(st))
    clean = _vjp(seq, kp, fx, st0, r, **g)
    st["prev_qpos"][1, 0] = np.nan
    st0, r = _run(seq, kp, fx, st)
    out = _vjp(seq, kp, fx, st0, r, **g)
    assert out["status"][1, L] & STATUS_NONFINITE
    assert np.isnan(out["grad_prev_qpos"][1]).all() and np.isnan(out["grad_last_qpos"][1]).all()
    assert np.isnan(out["grad_keypoints"][1, :L + 1]).all()
    for k in ("grad_keypoints", "grad_last_qpos", "grad_prev_qpos", "status"):
        assert same_bits(out[k][0], clean[k][0]), k


@pytest.mark.parametrize("lag", [1, 3])
def test_cotangent_reaches_at_most_lag_frames_ahead(lag, tmp_path):
    seq, o = _setup(CASES[1], tmp_path)
    S, K = 1, 8
    kp, fx = SV.stream_inputs(o, S, K, 51)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, lag, 52, C_OVER_W * _nd(seq), has_prev=1))
    k = lag + 2
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    gq[0, k] = 1.0
    out = _vjp(seq, kp, fx, st0, r, grad_qpos=gq)
    reach = np.abs(out["grad_keypoints"][0]).reshape(K, -1).max(1)
    assert (reach[k + 1:] == 0).all(), reach
    assert reach[k] > 0 and reach[k - lag] > 0 and reach[0] > 0, reach
    assert (out["status"][0, :lag] == STATUS_PENDING).all()


def test_argument_checks_workspace_and_sizes(tmp_path):
    from dex_retargeting_b200 import _native as N

    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 2, 2, 3
    kp, fx = SV.stream_inputs(o, S, K, 61)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 62, C_OVER_W * _nd(seq)))
    lib = AV.load()
    assert lib.emu_fixed_lag_accel_vjp_sizeof() == C.sizeof(N.DexrFixedLagAccelVjp)
    assert lib.emu_fixed_lag_vjp_sizeof() == C.sizeof(N.DexrFixedLagVjp)
    import emu_fixed_lag_vjp_host as FV

    ws = AV.workspace_bytes(seq, S, L)
    assert ws >= FV.workspace_bytes(seq, S, L) + S * 4 * (2 + o.opt_dof)  # (plus the accel smoother's E_t per frame)
    assert AV.workspace_bytes(seq, 0, L) == 0
    for null, msg in (("prev_qpos", "prev_qpos"), ("has_prev", "has_prev"), ("tape.qpos", "tape.qpos"),
                      ("grad_keypoints", "grad_keypoints"), ("last_qpos", "last_qpos"), ("workspace", "workspace")):
        with pytest.raises(EmulationError, match=msg):
            _vjp(seq, kp, fx, st0, r, null=(null,))
    for c in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(EmulationError, match="accel_weight"):
            _vjp(seq, kp, fx, st0, r, accel_weight=c)
    for nb in (FV.workspace_bytes(seq, S, L), ws - 4):
        with pytest.raises(EmulationError, match="dexr_fixed_lag_accel_vjp_workspace_bytes"):
            _vjp(seq, kp, fx, st0, r, workspace_bytes=nb)
    # every output but grad_keypoints may be NULL
    _vjp(seq, kp, fx, st0, r, null=("grad_fixed_qpos", "grad_last_qpos", "grad_prev_qpos", "grad_window_keypoints",
                                    "grad_window_fixed_qpos", "grad_window_qpos", "status_out"))


SPILL_BUDGET = {"dexr_fixed_lag_accel_vjp_kernel": {16: 4, 32: 0}, "dexr_fixed_lag_accel_tape_kernel": {16: 36, 32: 0}}


def test_register_budget(tmp_path):
    """`-Xptxas -v`: the new kernels at 32 lanes spill nothing; at 16 lanes no more than the accel smoother VJP (4 bytes)
    and the accel fixed-lag forward (36 bytes) they are built from."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    for name, budget in SPILL_BUDGET.items():
        got = {k: v for k, v in stores.items() if name in k}
        assert len(got) == 2, (name, sorted(stores))
        for G, b in budget.items():
            v = [x for k, x in got.items() if f"ILi{G}E" in k]
            assert v and v[0] <= b, (name, G, got)


@pytest.mark.parametrize("hp,c_over_w", [(0, 1.0), (1, 1.0), (1, C_OVER_W)], ids=["fresh-c1", "prev-c1", "prev-c10"])
@pytest.mark.parametrize("lag", [0, 1, 3])
@pytest.mark.parametrize("name", ["allegro_vector", "mimic_fixed_dense16"])
def test_model_matches_central_differences_of_the_chain(name, lag, hp, c_over_w, tmp_path):
    """<theta_bar, delta> of the model equals the central difference of the loss (emitted rows, final last_qpos and
    prev_qpos) of the accelerated chain re-polished in float64 tick by tick, 7 ticks, in keypoints, fixed joints, the
    anchor and the pre-anchor."""
    if name in SC.BY_ID:
        seq, o = SC.build(SC.BY_ID[name], tmp_path)
    else:
        seq, o = _setup((name, ("teleop/allegro_hand_right", None)), tmp_path)
    S, K = 1, 7
    w = _nd(seq)
    c = c_over_w * w
    kp, fx = SV.stream_inputs(o, S, K, 71 + lag)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, lag, 72, c, has_prev=hp))
    fl = _flags(seq, kp, fx)
    rng = np.random.RandomState(73)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    gq, grq = _cot(rng, (K, n)), _cot(rng, (K, dof))
    glast, gprev = rng.randn(n), rng.randn(n)
    k0, f0 = kp[0].astype(np.float64), None if fx is None else fx[0].astype(np.float64)
    fl0 = None if fl is None else fl[0]
    a0, p0 = st0["last_qpos"][0].astype(np.float64), st0["prev_qpos"][0].astype(np.float64)
    Xs = FAV.polished_chain(o, w, c, k0, f0, fl0, a0, p0, hp, lag, _windows(r, 0, lag))
    md = FAV.model_chain(o, w, c, k0, f0, fl0, a0, p0, hp, Xs, lag, gq, grq, glast, gprev)
    assert not md["not_pd"]
    lim = o.joint_limits
    used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
    dk = np.zeros_like(k0)
    dk[:, used] = rng.randn(K, len(used), 3)
    df = None if f0 is None else rng.randn(*f0.shape)
    da = rng.randn(n) * ((a0 > lim[:, 0]) & (a0 < lim[:, 1]))
    dp = rng.randn(n) * ((p0 > lim[:, 0]) & (p0 < lim[:, 1]))
    h = 1e-5
    vals = []
    for sg in (1, -1):
        f_ = None if f0 is None else f0 + sg * h * df
        X = FAV.polished_chain(o, w, c, k0 + sg * h * dk, f_, fl0, a0 + sg * h * da, p0 + sg * h * dp, hp, lag, Xs)
        vals.append(FAV.chain_loss(o, X, f_, lag, gq, grq, a0 + sg * h * da, p0 + sg * h * dp, glast, gprev))
    fd = (vals[0] - vals[1]) / (2 * h)
    pred = float((md["keypoints"] * dk).sum() + (0 if df is None else (md["fixed"] * df).sum()) + (md["last"] * da).sum()
                 + (md["prev"] * dp).sum())
    # (5e-3, not the velocity-only 2e-3: at c = 10 w some windows hold a joint at its bound with a multiplier near 3e-4,
    # which the step comes close to crossing, and a smaller step drowns in the re-polished windows' float64 noise)
    assert abs(fd - pred) <= 5e-3 * max(abs(fd), 1e-3), (fd, pred)
    if hp:
        assert np.abs(md["prev"]).max() > 0


@pytest.mark.parametrize("case", ALL_CASES, ids=[c[0] for c in ALL_CASES])
def test_emulation_matches_the_model(case, tmp_path):
    name = case[0]
    seq, o = _setup(case, tmp_path)
    S, L, K = 2, 2, 6
    kp, fx = SV.stream_inputs(o, S, K, 81)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 82, C_OVER_W * _nd(seq), has_prev=1))
    fl = _flags(seq, kp, fx)
    rng = np.random.RandomState(83)
    gq, grq = _cot(rng, (S, K, o.opt_dof)), _cot(rng, (S, K, seq.optimizer.robot.dof))
    glast, gprev = _cot(rng, (S, o.opt_dof)), _cot(rng, (S, o.opt_dof))
    got = _vjp(seq, kp, fx, st0, r, grad_qpos=gq, grad_robot_qpos=grq, grad_last_qpos_out=glast, grad_prev_qpos_out=gprev)
    assert not (got["status"] & (STATUS_NOT_PD | STATUS_NONFINITE)).any(), got["status"]
    checked = 0
    for s in range(S):
        md = _model(seq, o, kp, fx, fl, st0, r, L, gq, grq, s, glast=glast, gprev=gprev)
        if md["skip"]:
            continue
        FAV.compare(got["grad_keypoints"][s], got["grad_fixed_qpos"][s], got["grad_last_qpos"][s], got["grad_prev_qpos"][s],
                    md)
        checked += 1
    assert checked >= 1, name


def test_gpu_fixed_lag_accel_vjp_file_passes_against_the_emulation():
    """tests/test_gpu_fixed_lag_accel_vjp.py dry-run on the CPU (tests/tools/emu_gpu_fixed_lag_accel_vjp.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_fixed_lag_accel_vjp.py")],
                         capture_output=True, text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
