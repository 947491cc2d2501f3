"""Backpropagation through fixed-lag smoothing (`dexr_fixed_lag_step_vjp`) through the host emulation of the kernel's own
driver (tests/emu runs fixed_lag_tick<G, true> and the fixed_lag_vjp_* helpers of dexr_kernels.cuh on the fiber warp):
the float64 model of tests/fixed_lag_vjp_cases.py, itself checked against central differences of the fixed-lag chain
re-polished in float64 tick by tick, on the packaged LEAP DexPilot, Allegro and Shadow configs and on structure cases with
fixed, mimic and prismatic joints at 16 and 32 lanes; L = 0 against the causal sequence VJP; with L >= K - 1 and a flush
it is the smoother's VJP of the whole clip bit for bit; a run split into chunks chained through the state cotangents gives
the bits of one call; recording changes no output bit; a cotangent reaches no frame more than L ticks after its own; a
NOT_PD window cuts the anchor chain, a missing frame carries it, a non-finite stream is NaN back to its start; the argument
checks, the workspace size, guard words around every written buffer and the register budget."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_fixed_lag_host as FL
import emu_fixed_lag_vjp_host as FV
import emu_packed_host as P
import emu_seq_vjp_host as SQ
import emu_smooth_vjp_host as SVJ
import fixed_lag_vjp_cases as FLC
import smooth_vjp_cases as SVC
import seq_vjp_cases as SV
import structure_cases as SC
from emu_eval_host import EmulationError
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1
STATUS_NOT_PD, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 26, 1 << 25, 1 << 27, 1 << 28
# the case list of tests/test_smooth_vjp_emulation.py: the packaged configs, then fixed, mimic and prismatic joints at 16
# and 32 lanes
MODEL_CASES = [
    ("leap_dexpilot", ("teleop/leap_hand_right_dexpilot", None)),
    ("allegro_vector", ("teleop/allegro_hand_right", None)),
    ("shadow_position", ("offline/shadow_hand_right", None)),
    ("fixed_dense16", "fixed_dense16"),
    ("mimic_dense16", "mimic_dense16"),
    ("mimic_fixed_dense32", "mimic_fixed_dense32"),
    ("prismatic_arrow", "prismatic_arrow"),
]

CASES = [
    ("leap_dexpilot", ("teleop/leap_hand_right_dexpilot", None)),
    ("allegro_vector", ("teleop/allegro_hand_right", None)),
    ("mimic_fixed_dense32", "mimic_fixed_dense32"),  # mimic and fixed joints, 32 lanes
    ("mimic_dense16", "mimic_dense16"),
]
IDS = [c[0] for c in CASES]


def _setup(case, tmp_path):
    name, spec = case
    if isinstance(spec, str):
        return SC.build(SC.BY_ID[spec], tmp_path)
    return build_product(*spec), build_oracle(*spec)


def _state(seq, o, S, lag, seed):
    st = FL.fresh_state(seq, S, lag)
    rng = np.random.RandomState(seed)
    st["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0],
                                   o.joint_limits[:, 1])
    return st


def same_bits(a, b):
    """Equal values with NaN where NaN (+0 and -0 compare equal: an added zero cotangent may flip the sign of a zero)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def _cot(rng, shape):
    return rng.randn(*shape).astype(np.float32)


def _run(seq, kp, fx, st, flush=False, w=-1.0):
    """A recorded forward on `st` (updated in place); returns (state before, outputs with the tape)."""
    st0 = FL.copy_state(st)
    r = FV.fixed_lag_step_tape(seq, kp, st, fixed_qpos=fx, flush=flush, smooth_weight=w)
    return st0, r


def _vjp(seq, kp, fx, st0, r, flushed=False, w=-1.0, **g):
    return FV.fixed_lag_vjp(seq, kp, st0, r["tape_qpos"], r["tape_projected"], fixed_qpos=fx, flushed=flushed,
                            smooth_weight=w, **g)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_recording_changes_no_bit(case, tmp_path):
    seq, o = _setup(case, tmp_path)
    S, L, K = 2, 2, 5
    kp, fx = SV.stream_inputs(o, S, K, 5)
    a, b = _state(seq, o, S, L, 6), _state(seq, o, S, L, 6)
    r = FL.fixed_lag_step(seq, kp, a, fixed_qpos=fx, flush=True)
    t = FV.fixed_lag_step_tape(seq, kp, b, fixed_qpos=fx, flush=True)
    for k in r:
        assert same_bits(r[k], t[k]), k
    for k in FL.STATE:
        if a.get(k) is not None:
            assert np.array_equal(a[k], b[k]), k
    # the tape: each tick's window minimiser (the last tick's window is the one the flush emits)
    assert same_bits(t["tape_qpos"][:, -1, 1:L + 1], t["flush_qpos"][:, :L])


@pytest.mark.parametrize("lag_extra", [0, 2])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_full_lag_is_the_smoother_vjp(case, lag_extra, tmp_path):
    """Fresh state, L >= K - 1, ticks then a flush: the smoother's VJP of the whole clip at the last window, bit for bit."""
    seq, o = _setup(case, tmp_path)
    S, K = 2, 5
    L = K - 1 + lag_extra
    kp, fx = SV.stream_inputs(o, S, K, 11)
    st = _state(seq, o, S, L, 12)
    st0, r = _run(seq, kp, fx, st, flush=True)
    rng = np.random.RandomState(13)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    gq, gr = _cot(rng, (S, K, n)), _cot(rng, (S, K, dof))
    gfq, gfr = _cot(rng, (S, L, n)), _cot(rng, (S, L, dof))
    glast = _cot(rng, (S, n))
    got = _vjp(seq, kp, fx, st0, r, flushed=True, grad_qpos=gq, grad_robot_qpos=gr, grad_flush_qpos=gfq,
               grad_flush_robot_qpos=gfr, grad_last_qpos_out=glast)
    # the clip's cotangents: the emitted row (only when L = K - 1), then the flushed rows; the last one takes glast
    e = 1 if L == K - 1 else 0
    cq = np.concatenate([gq[:, K - 1:K] if e else np.zeros((S, 0, n), np.float32), gfq[:, :K - e]], 1)
    cr = np.concatenate([gr[:, K - 1:K] if e else np.zeros((S, 0, dof), np.float32), gfr[:, :K - e]], 1)
    cq[:, -1] += glast
    X = r["tape_qpos"][:, K - 1, :K]
    pj = st0["projected"]
    gk, gf, gl, status = SVJ.smooth_vjp_packed(seq, kp.reshape(S * K, 21, 3), np.arange(S + 1) * K, X.reshape(S * K, n),
                                               last_qpos=st0["last_qpos"], projected=pj,
                                               fixed_qpos=None if fx is None else fx.reshape(S * K, -1),
                                               grad_qpos=cq.reshape(S * K, n), grad_robot_qpos=cr.reshape(S * K, dof))
    assert same_bits(got["grad_keypoints"], gk.reshape(S, K, 21, 3))
    if fx is not None:
        assert same_bits(got["grad_fixed_qpos"], gf.reshape(S, K, -1))
    assert same_bits(got["grad_last_qpos"], gl)
    assert not np.isnan(got["grad_keypoints"]).any()


def _chain(seq, o, kp, fx, st, cuts, g, flush_call):
    """The run of `kp` split at `cuts` (a flush-only call at the end when flush_call), each chunk's VJP fed the next one's
    state cotangents; returns the per-frame keypoint gradients [S,K], fixed [S,K] and the first state's cotangents."""
    K = kp.shape[1]
    bounds = [0] + list(cuts) + [K]
    calls = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        calls.append((a, b, *_run(seq, kp[:, a:b], None if fx is None else fx[:, a:b], st)))
    if flush_call:
        st0 = FL.copy_state(st)
        fr = FV.fixed_lag_step_tape(seq, None, st, flush=True)
        carry = FV.fixed_lag_vjp(seq, None, st0, None, None, flushed=True, grad_flush_qpos=g["grad_flush_qpos"],
                                 grad_flush_robot_qpos=g["grad_flush_robot_qpos"], grad_last_qpos_out=g["grad_last_qpos_out"])
    else:
        carry = dict(grad_last_qpos=g["grad_last_qpos_out"], grad_window_keypoints=None, grad_window_fixed_qpos=None,
                     grad_window_qpos=None)
    gks, gfs = [], []
    for a, b, st0, r in reversed(calls):
        out = _vjp(seq, kp[:, a:b], None if fx is None else fx[:, a:b], st0, r, grad_qpos=g["grad_qpos"][:, a:b],
                   grad_robot_qpos=g["grad_robot_qpos"][:, a:b], grad_last_qpos_out=carry["grad_last_qpos"],
                   grad_window_qpos_out=carry["grad_window_qpos"], grad_window_keypoints_out=carry["grad_window_keypoints"],
                   grad_window_fixed_qpos_out=carry["grad_window_fixed_qpos"])
        gks.insert(0, out["grad_keypoints"])
        gfs.insert(0, out["grad_fixed_qpos"])
        carry = out
    return np.concatenate(gks, 1), np.concatenate(gfs, 1), carry


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_chunks_give_the_bits_of_one_call(case, tmp_path):
    """K ticks then a flush in one call equal the same ticks split into three calls, the flush a call of its own, bit for
    bit; the run starts with a partly filled window."""
    seq, o = _setup(case, tmp_path)
    S, L, K = 2, 3, 8
    kp, fx = SV.stream_inputs(o, S, K + 2, 21)
    pre = _state(seq, o, S, L, 22)
    FL.fixed_lag_step(seq, kp[:, :2], pre, fixed_qpos=None if fx is None else fx[:, :2])  # 2 frames held
    kp, fx = kp[:, 2:], None if fx is None else fx[:, 2:]
    rng = np.random.RandomState(23)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    g = dict(grad_qpos=_cot(rng, (S, K, n)), grad_robot_qpos=_cot(rng, (S, K, dof)), grad_flush_qpos=_cot(rng, (S, L, n)),
             grad_flush_robot_qpos=_cot(rng, (S, L, dof)), grad_last_qpos_out=_cot(rng, (S, n)))
    one = FL.copy_state(pre)
    st0, r = _run(seq, kp, fx, one, flush=True)
    want = _vjp(seq, kp, fx, st0, r, flushed=True, **g)
    gk, gf, first = _chain(seq, o, kp, fx, FL.copy_state(pre), [3, 5], g, flush_call=True)
    assert same_bits(gk, want["grad_keypoints"])
    assert same_bits(gf, want["grad_fixed_qpos"])
    for k in ("grad_last_qpos", "grad_window_keypoints", "grad_window_fixed_qpos", "grad_window_qpos"):
        assert same_bits(first[k], want[k]), k
    assert not np.isnan(want["grad_keypoints"]).any()
    assert (want["grad_window_keypoints"][:, :2] != 0).any()  # the held frames are reached


@pytest.mark.parametrize("lag", [1, 3])
def test_cotangent_reaches_at_most_lag_frames_ahead(lag, tmp_path):
    """A cotangent on the frame emitted at tick k (frame k - L) reaches the keypoints of frames up to k and no later."""
    seq, o = _setup(CASES[1], tmp_path)
    S, K = 1, 8
    kp, fx = SV.stream_inputs(o, S, K, 31)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, lag, 32))
    k = lag + 2
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    gq[0, k] = 1.0
    out = _vjp(seq, kp, fx, st0, r, grad_qpos=gq)
    reach = np.abs(out["grad_keypoints"][0]).reshape(K, -1).max(1)
    assert (reach[k + 1:] == 0).all(), reach
    assert reach[k] > 0 and reach[k - lag] > 0, reach
    assert out["status"][0, k] == 0 and (out["status"][0, :lag] == STATUS_PENDING).all()


def test_non_finite_stream_is_nan_to_its_start_and_alone(tmp_path):
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 2, 2, 6
    kp, fx = SV.stream_inputs(o, S, K, 41)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 42))
    gq = np.ones((S, K, o.opt_dof), np.float32)
    clean = _vjp(seq, kp, fx, st0, r, grad_qpos=gq)
    gq[0, K - 1, 0] = np.inf
    out = _vjp(seq, kp, fx, st0, r, grad_qpos=gq)
    assert np.isnan(out["grad_keypoints"][0]).all() and np.isnan(out["grad_last_qpos"][0]).all()
    assert out["status"][0, K - 1] & STATUS_NONFINITE
    assert same_bits(out["grad_keypoints"][1], clean["grad_keypoints"][1])


def test_argument_checks_and_workspace(tmp_path):
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 2, 2, 3
    kp, fx = SV.stream_inputs(o, S, K, 51)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 52))
    assert FV.workspace_bytes(seq, S, L) >= S * (L + 1) * 4 * (o.opt_dof * 3 + 63 * 2)
    assert FV.workspace_bytes(seq, 0, L) == 0
    for null, msg in (("tape.qpos", "tape.qpos"), ("grad_keypoints", "grad_keypoints"), ("last_qpos", "last_qpos"),
                      ("workspace", "workspace")):
        with pytest.raises(EmulationError, match=msg):
            _vjp(seq, kp, fx, st0, r, null=(null,))
    with pytest.raises(EmulationError, match="workspace"):
        FV.fixed_lag_vjp(seq, kp, st0, r["tape_qpos"], fixed_qpos=fx, workspace_bytes=FV.workspace_bytes(seq, S, L) - 4)
    with pytest.raises(EmulationError, match="lag"):
        FV.fixed_lag_vjp(seq, kp, st0, r["tape_qpos"], fixed_qpos=fx, lag=5000)
    with pytest.raises(EmulationError, match="smooth_weight"):
        _vjp(seq, kp, fx, st0, r, w=float("inf"))
    # every output but grad_keypoints may be NULL
    _vjp(seq, kp, fx, st0, r, null=("grad_fixed_qpos", "grad_last_qpos", "grad_window_keypoints",
                                    "grad_window_fixed_qpos", "grad_window_qpos", "status_out"))


def test_register_budget_no_spills():
    """Both instantiations of dexr_fixed_lag_vjp_kernel and of the recording dexr_fixed_lag_tape_kernel, and the
    fixed-lag forward, compile without spills."""
    nvcc = Path("/usr/local/cuda/bin/nvcc")
    if not nvcc.exists():
        pytest.skip("nvcc not available")
    res = subprocess.run([str(nvcc), "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                          "-cubin", "-o", "/dev/null", str(ROOT / "dex_retargeting_b200" / "csrc" / "dexr.cu")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function properties for" in line and any(k in line for k in ("dexr_fixed_lag_vjp_kernel", "dexr_fixed_lag_kernel",
                                                                            "dexr_fixed_lag_tape_kernel")):
            seen += 1
            assert " 0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], (line, lines[i + 1])
    assert seen == 6


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _flags(seq, kp, fx):
    """The DexPilot flags every frame uses, [S,K,len_proj] (the causal walk from fresh flags), or None."""
    S, K = kp.shape[:2]
    st = SQ.fresh_state(seq, S)
    _, _, _, tape = P.solve_packed(seq, kp.reshape(-1, 21, 3), P.offsets_of([K] * S), state=st,
                                   fixed_qpos=None if fx is None else fx.reshape(S * K, -1), record=True)
    return None if tape["projected"] is None else tape["projected"].reshape(S, K, -1)


def _windows(r, s, L):
    K = r["tape_qpos"].shape[1]
    return [r["tape_qpos"][s, k, :FLC.window(k, L)[1]] for k in range(K)]


def _model(seq, o, kp, fx, fl, st0, r, L, gq, grq, s):
    return FLC.model_chain(o, _nd(seq), kp[s].astype(np.float64), None if fx is None else fx[s].astype(np.float64),
                           None if fl is None else fl[s], st0["last_qpos"][s].astype(np.float64), _windows(r, s, L), L,
                           gq[s], grq[s])


@pytest.mark.parametrize("lag", [1, 3])
@pytest.mark.parametrize("name", ["allegro_vector", "mimic_fixed_dense16"])
def test_model_matches_central_differences_of_the_chain(name, lag, tmp_path):
    """<theta_bar, delta> of the model equals the central difference of the loss on the emitted rows of the fixed-lag chain
    re-polished in float64 tick by tick (each window anchored at the previous re-polished commit), 7 ticks."""
    seq, o = SC.build(SC.BY_ID[name], tmp_path) if name in SC.BY_ID else _setup((name, ("teleop/allegro_hand_right", None)),
                                                                                  tmp_path)
    S, K = 1, 7
    kp, fx = SV.stream_inputs(o, S, K, 61 + lag)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, lag, 62))
    fl = _flags(seq, kp, fx)
    rng = np.random.RandomState(63)
    n, dof = o.opt_dof, seq.optimizer.robot.dof
    gq, grq = _cot(rng, (K, n)), _cot(rng, (K, dof))
    w = _nd(seq)
    k0, f0 = kp[0].astype(np.float64), None if fx is None else fx[0].astype(np.float64)
    fl0 = None if fl is None else fl[0]
    a0 = st0["last_qpos"][0].astype(np.float64)
    Xs = FLC.polished_chain(o, w, k0, f0, fl0, a0, lag, _windows(r, 0, lag))
    md = FLC.model_chain(o, w, k0, f0, fl0, a0, Xs, lag, gq, grq)
    assert not md["not_pd"]
    lim = o.joint_limits
    used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
    dk = np.zeros_like(k0)
    dk[:, used] = rng.randn(K, len(used), 3)
    df = None if f0 is None else rng.randn(*f0.shape)
    da = rng.randn(n) * ((a0 > lim[:, 0]) & (a0 < lim[:, 1]))
    h = 1e-5
    vals = []
    for sg in (1, -1):
        f_ = None if f0 is None else f0 + sg * h * df
        X = FLC.polished_chain(o, w, k0 + sg * h * dk, f_, fl0, a0 + sg * h * da, lag, Xs)
        vals.append(FLC.emitted_loss(o, X, f_, lag, gq, grq))
    fd = (vals[0] - vals[1]) / (2 * h)
    pred = float((md["keypoints"] * dk).sum() + (0 if df is None else (md["fixed"] * df).sum()) + (md["last"] * da).sum())
    assert abs(fd - pred) <= 2e-3 * max(abs(fd), 1e-3), (fd, pred)
    # the chain is exercised: frames committed before the last window are reached through the anchor
    assert np.abs(md["keypoints"][0]).max() > 0 and np.abs(md["last"]).max() > 0


@pytest.mark.parametrize("name", [c[0] for c in MODEL_CASES])
def test_emulation_matches_the_model(name, tmp_path):
    seq, o = _setup(dict(MODEL_CASES)[name] and (name, dict(MODEL_CASES)[name]), tmp_path)
    S, L, K = 2, 2, 6
    kp, fx = SV.stream_inputs(o, S, K, 71)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 72))
    fl = _flags(seq, kp, fx)
    rng = np.random.RandomState(73)
    gq, grq = _cot(rng, (S, K, o.opt_dof)), _cot(rng, (S, K, seq.optimizer.robot.dof))
    got = _vjp(seq, kp, fx, st0, r, grad_qpos=gq, grad_robot_qpos=grq)
    assert not (got["status"] & (STATUS_NOT_PD | STATUS_NONFINITE)).any(), got["status"]
    checked = 0
    for s in range(S):
        md = _model(seq, o, kp, fx, fl, st0, r, L, gq, grq, s)
        if md["skip"]:
            continue
        FLC.compare(got["grad_keypoints"][s], got["grad_fixed_qpos"][s], got["grad_last_qpos"][s], md)
        checked += 1
    assert checked >= 1, name
    if fx is not None:
        assert np.abs(got["grad_fixed_qpos"]).max() > 0


@pytest.mark.parametrize("name", ["allegro_vector", "mimic_fixed_dense32"])
def test_lag_zero_is_the_causal_vjp(name, tmp_path):
    """L = 0, w = norm_delta: each tick is the causal frame problem, so at the same points the backward is
    dexr_solve_sequences_vjp's without the low-pass filter (within smooth_vjp_cases' tolerance)."""
    import copy

    seq, o = _setup(dict(MODEL_CASES)[name] and (name, dict(MODEL_CASES)[name]), tmp_path)
    S, K = 2, 6
    kp, fx = SV.stream_inputs(o, S, K, 81)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, 0, 82))
    grq = _cot(np.random.RandomState(83), (S, K, seq.optimizer.robot.dof))
    got = _vjp(seq, kp, fx, st0, r, grad_robot_qpos=grq)
    nofilter = copy.copy(seq)
    nofilter.filter = None
    want = SQ.solve_sequences_vjp(nofilter, kp, r["tape_qpos"][:, :, 0], st0["last_qpos"], grad_robot_qpos=grq,
                                  fixed_qpos=fx)
    assert (want[4] & (STATUS_NOT_PD | STATUS_NONFINITE) == 0).all()
    for s in range(S):
        e = SVC.stream_errors(got["grad_keypoints"][s], want[0][s])
        e = max(e, SVC.stream_errors(got["grad_last_qpos"][s], want[2][s]))
        if fx is not None:
            e = max(e, SVC.stream_errors(got["grad_fixed_qpos"][s], want[1][s]))
        assert e <= SVC.TAU, (s, e)


def test_not_pd_window_cuts_the_chain(tmp_path):
    """A window whose stacked free Hessian is indefinite (its tape point replaced by one far from any minimum) contributes
    zero and passes no anchor cotangent on: a loss on its emitted row alone reaches nothing, with STATUS_NOT_PD."""
    seq, o = _setup(CASES[1], tmp_path)
    S, L, K = 1, 2, 7
    kp, fx = SV.stream_inputs(o, S, K, 91)
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 92))
    k = 5
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    gq[0, k] = 1.0
    clean = _vjp(seq, kp, fx, st0, r, grad_qpos=gq)
    assert clean["status"][0, k] == 0 and np.abs(clean["grad_keypoints"][0, :FLC.window(k, L)[0]]).max() > 0
    rng = np.random.RandomState(93)
    lo, hi = o.joint_limits[:, 0], o.joint_limits[:, 1]
    for _ in range(50):  # points with an indefinite window Hessian
        bad = dict(r)
        bad["tape_qpos"] = r["tape_qpos"].copy()
        bad["tape_qpos"][0, k, :L + 1] = lo + (hi - lo) * rng.rand(L + 1, o.opt_dof)
        out = _vjp(seq, kp, fx, st0, bad, grad_qpos=gq)
        if out["status"][0, k] & STATUS_NOT_PD:
            break
    else:
        pytest.fail("no NOT_PD window found")
    assert (out["grad_keypoints"] == 0).all() and (out["grad_last_qpos"] == 0).all()
    assert not (out["status"][0, :k] & STATUS_NOT_PD).any()


def test_missing_frame_carries_the_chain(tmp_path):
    """A dropped detection (NaN keypoints) inside the chain gets zero cotangents; the anchor chain runs through it to the
    frames before, and the result matches the model."""
    seq, o = _setup(CASES[2], tmp_path)
    S, L, K = 1, 2, 8
    kp, fx = SV.stream_inputs(o, S, K, 101)
    kp[0, 3] = np.nan
    st0, r = _run(seq, kp, fx, _state(seq, o, S, L, 102))
    gq = np.zeros((S, K, o.opt_dof), np.float32)
    grq = np.zeros((S, K, seq.optimizer.robot.dof), np.float32)
    gq[0, K - 1] = np.random.RandomState(103).randn(o.opt_dof)
    out = _vjp(seq, kp, fx, st0, r, grad_qpos=gq, grad_robot_qpos=grq)
    assert out["status"][0, 5] & STATUS_MISSING  # the tick that emitted frame 3
    assert (out["grad_keypoints"][0, 3] == 0).all() and (out["grad_fixed_qpos"][0, 3] == 0).all()
    assert np.isfinite(out["grad_keypoints"]).all()
    assert all(np.abs(out["grad_keypoints"][0, t]).max() > 0 for t in (0, 1, 2, 4, 5))
    md = _model(seq, o, kp, fx, _flags(seq, np.nan_to_num(kp), fx), st0, r, L, gq, grq, 0)
    FLC.compare(out["grad_keypoints"][0], out["grad_fixed_qpos"][0], out["grad_last_qpos"][0], md)
