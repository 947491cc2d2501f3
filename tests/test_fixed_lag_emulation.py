"""Fixed-lag smoothing of live streams (`dexr_fixed_lag_step`) through the host emulation of the kernel's own driver
(tests/emu runs fixed_lag_tick of dexr_kernels.cuh on the fiber warp) on the packaged LEAP DexPilot, Allegro vector and
Shadow position configs and on fixed-joint, mimic and prismatic robots of tests/structure_cases.py at 16 and 32 lanes: each
tick is the offline smoother (emu_smooth_host) on the window rebuilt from the state, bit for bit; L = 0 is the causal
minimiser and L >= T - 1 with a flush the offline one (the float64 model of tests/smooth_cases.py); the committed DexPilot
flags are the causal tape's; dropped frames are interpolated; splitting a run over calls or batching streams changes no bit;
the argument checks, the workspace size, guard words around every written buffer (state included), the register budget
and a dry run of tests/test_gpu_fixed_lag.py."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_fixed_lag_host as FL
import emu_packed_host as P
import emu_smooth_host as SM
import seq_vjp_cases as SV
import smooth_cases as SMC
import structure_cases as SC
from emu_eval_host import EmulationError
from emu_seq_vjp_host import fresh_state as fresh_stream_state
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID
STATUS_MAXITER, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 24, 1 << 25, 1 << 27, 1 << 28

# (name, how to build it): the packaged configs, then fixed joints, mimic and prismatic joints at 16 and 32 lanes
CASES = [
    ("leap_dexpilot", ("teleop/leap_hand_right_dexpilot", None)),
    ("allegro_vector", ("teleop/allegro_hand_right", None)),
    ("shadow_position", ("offline/shadow_hand_right", None)),
    ("mimic_dense16", "mimic_dense16"),              # mimic and prismatic joints, 16 lanes
    ("mimic_fixed_dense32", "mimic_fixed_dense32"),  # mimic and fixed joints, 32 lanes
    ("fixed_dense16", "fixed_dense16"),
    ("prismatic_arrow", "prismatic_arrow"),          # prismatic joints, 32 lanes
]
IDS = [c[0] for c in CASES]


def _setup(case, tmp_path):
    name, spec = case
    if isinstance(spec, str):
        return SC.build(SC.BY_ID[spec], tmp_path)
    return build_product(*spec), build_oracle(*spec)


def _state(seq, o, S, lag, seed):
    """A fresh state with a seeded warm start inside the joint limits."""
    st = FL.fresh_state(seq, S, lag)
    rng = np.random.RandomState(seed)
    st["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0],
                                   o.joint_limits[:, 1])
    return st


def _nd(seq):
    return float(seq.optimizer.params().norm_delta)


def _window_solve(seq, snap, kp, fx, s, w=-1.0):
    """dexr_smooth_sequences_packed on stream s's window rebuilt from the state `snap` before a tick and its new frame."""
    h = int(snap["window_len"][s])
    wk = np.concatenate([snap["window_keypoints"][s, :h], kp[s:s + 1]])
    start = snap["window_qpos"][s, h - 1:h] if h else snap["last_qpos"][s:s + 1]
    wq = np.concatenate([snap["window_qpos"][s, :h], start])
    wf = None if fx is None else np.concatenate([snap["window_fixed_qpos"][s, :h], fx[s:s + 1]])
    pj = None if snap["projected"] is None else snap["projected"][s:s + 1]
    q, rq, status, _ = SM.smooth_packed(seq, wk, [0, h + 1], wq, last_qpos=snap["last_qpos"][s:s + 1], projected=pj,
                                        fixed_qpos=wf, smooth_weight=w)
    return h, q, rq, status


def _check_tick(seq, snap, st, r, kp, fx, w=-1.0):
    """One tick (kp [S,1,21,3]) against the smoother on every stream's window: the emitted frame (or NaN and PENDING), the
    new window_qpos, the status word, the committed anchor, all bit for bit."""
    L = st["lag"]
    for s in range(kp.shape[0]):
        h, q, rq, status = _window_solve(seq, snap, kp[:, 0], None if fx is None else fx[:, 0], s, w)
        if h == L:
            np.testing.assert_array_equal(r["qpos"][s, 0], q[0])
            np.testing.assert_array_equal(r["robot_qpos"][s, 0], rq[0])
            assert r["status"][s, 0] == status[0], (s, r["status"][s, 0], status[0])
            np.testing.assert_array_equal(st["window_qpos"][s, :L], q[1:])
            np.testing.assert_array_equal(st["last_qpos"][s], q[0])
            assert st["window_len"][s] == L
        else:
            assert r["status"][s, 0] == STATUS_PENDING
            assert np.isnan(r["qpos"][s, 0]).all() and np.isnan(r["robot_qpos"][s, 0]).all()
            np.testing.assert_array_equal(st["window_qpos"][s, :h + 1], q)
            np.testing.assert_array_equal(st["last_qpos"][s], snap["last_qpos"][s])
            assert st["window_len"][s] == h + 1
    return status


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_each_tick_is_the_smoother(case, lag, tmp_path):
    """Snapshot, one tick, the smoother on the rebuilt window: the same bits, before and after the window fills."""
    seq, o = _setup(case, tmp_path)
    S, K = 2, lag + 2
    kp, fx = SV.stream_inputs(o, S, K, 31 + lag)
    st = _state(seq, o, S, lag, 32)
    w = -1.0 if lag != 1 else 2.0 * _nd(seq)  # a smoothing weight other than norm_delta on the L = 1 runs
    for k in range(K):
        snap = FL.copy_state(st)
        kk, ff = kp[:, k:k + 1], None if fx is None else fx[:, k:k + 1]
        r = FL.fixed_lag_step(seq, kk, st, fixed_qpos=ff, smooth_weight=w)
        _check_tick(seq, snap, st, r, kk, ff, w)
        held = min(k + 1, lag)  # the window holds the last `held` inputs, in order (the shift included)
        np.testing.assert_array_equal(st["window_keypoints"][:, :held], kp[:, k + 1 - held:k + 1])
        if fx is not None:
            np.testing.assert_array_equal(st["window_fixed_qpos"][:, :held], fx[:, k + 1 - held:k + 1])


@pytest.mark.parametrize("case", CASES[:3] + CASES[4:5], ids=IDS[:3] + IDS[4:5])
def test_lag_zero_is_the_causal_minimiser(case, tmp_path):
    """L = 0: every tick emits its frame, the float64 minimiser of L_t(x) + w |x - clip(x_{t-1})|^2 with the flags of the
    causal walk."""
    seq, o = _setup(case, tmp_path)
    T = 5
    kp, fx = SV.stream_inputs(o, 1, T, 41, pinch=True)
    st = _state(seq, o, 1, 0, 42)
    a0 = st["last_qpos"][0].copy()
    r = FL.fixed_lag_step(seq, kp, st, fixed_qpos=fx)
    assert not (r["status"] & (STATUS_PENDING | STATUS_MAXITER | STATUS_NONFINITE)).any(), r["status"]
    flags = _causal_flags(seq, kp[0], None if fx is None else fx[0])
    prev = a0
    for t in range(T):
        m = SMC.Model(o, kp[0, t:t + 1], None if fx is None else fx[0, t:t + 1], None if flags is None else flags[t:t + 1],
                      SMC.clipped_anchor(o, prev), _nd(seq))
        X = r["qpos"][0, t:t + 1].astype(np.float64)
        assert np.abs(m.polish(X) - X).max() <= SMC.PARITY, t
        prev = r["qpos"][0, t]
    np.testing.assert_array_equal(st["last_qpos"][0], r["qpos"][0, -1])


def _causal_flags(seq, kp, fx):
    """The DexPilot flags after every frame of the causal taped packed solve from fresh flags (None for other losses)."""
    st = fresh_stream_state(seq, 1)
    _, _, _, tape = P.solve_packed(seq, kp, P.offsets_of([len(kp)]), state=st, fixed_qpos=fx, record=True)
    return tape["projected"]


@pytest.mark.parametrize("case,T,lag", [(CASES[0], 5, 4), (CASES[1], 5, 6), (CASES[2], 4, 3), (CASES[3], 5, 4),
                                        (CASES[4], 4, 5)], ids=["leap_dexpilot-T5-L4", "allegro_vector-T5-L6",
                                                                "shadow_position-T4-L3", "mimic_dense16-T5-L4",
                                                                "mimic_fixed_dense32-T4-L5"])
def test_full_lag_and_flush_is_the_offline_smoother(case, T, lag, tmp_path):
    """L >= T - 1, then a flush: T frames emitted in all, the float64 smoother minimiser of the whole clip from the same
    anchor."""
    seq, o = _setup(case, tmp_path)
    kp, fx = SV.stream_inputs(o, 1, T, 51, pinch=True)
    st = _state(seq, o, 1, lag, 52)
    a0 = st["last_qpos"].copy()
    r = FL.fixed_lag_step(seq, kp, st, fixed_qpos=fx, flush=True)
    live = (r["status"][0] & STATUS_PENDING) == 0
    assert live.sum() == T - lag if lag == T - 1 else not live.any()
    n = int(r["flush_count"][0])
    assert live.sum() + n == T
    assert np.isnan(r["flush_qpos"][0, n:]).all() and np.isnan(r["flush_robot_qpos"][0, n:]).all()
    X = np.concatenate([r["qpos"][0, live], r["flush_qpos"][0, :n]]).astype(np.float64)
    assert not (r["status"][0, live] & STATUS_MAXITER).any()
    flags = _causal_flags(seq, kp[0], None if fx is None else fx[0])
    m = SMC.Model(o, kp[0], None if fx is None else fx[0], flags, SMC.clipped_anchor(o, a0[0]), _nd(seq))
    assert np.abs(m.polish(X) - X).max() <= SMC.PARITY
    # the flush commits the last frame and empties the window
    np.testing.assert_array_equal(st["last_qpos"][0], X[-1].astype(np.float32))
    assert st["window_len"][0] == 0
    if flags is not None:
        np.testing.assert_array_equal(st["projected"][0], flags[-1])


def test_committed_dexpilot_flags_are_the_causal_tapes(tmp_path):
    """A pinch switches the flags on and off again: after every commit the state's flags are the causal tape's for the
    committed frame."""
    seq, o = _setup(CASES[0], tmp_path)
    T, L = 6, 1
    kp, fx = SV.stream_inputs(o, 1, T, 61, pinch=True)
    flags = _causal_flags(seq, kp[0], None)
    assert flags.any() and not flags.all()
    st = _state(seq, o, 1, L, 62)
    seen = set()
    for k in range(T):
        FL.fixed_lag_step(seq, kp[:, k:k + 1], st)
        if k >= L:
            np.testing.assert_array_equal(st["projected"][0], flags[k - L], err_msg=f"tick {k}")
            seen.add(bool(flags[k - L].any()))
    assert seen == {True, False}
    FL.fixed_lag_step(seq, None, st, flush=True)
    np.testing.assert_array_equal(st["projected"][0], flags[T - 1])


@pytest.mark.parametrize("case", CASES[:2] + CASES[4:5], ids=IDS[:2] + IDS[4:5])
def test_missing_frames_are_interpolated(case, tmp_path):
    """Frames 5 and 6 dropped, L = 4: once frame 9 arrives the gap is the linear interpolation between the committed frame
    4 and the window's frame 7; the emitted gap frames carry MISSING, the others not."""
    seq, o = _setup(case, tmp_path)
    T, L = 12, 4
    kp, fx = SV.stream_inputs(o, 1, T, 71)
    kp[0, 5:7] = np.nan
    st = _state(seq, o, 1, L, 72)
    r = FL.fixed_lag_step(seq, kp[:, :10], st, fixed_qpos=None if fx is None else fx[:, :10])
    q4, q5 = r["qpos"][0, 8].astype(np.float64), r["qpos"][0, 9].astype(np.float64)
    x6, x7 = st["window_qpos"][0, 0].astype(np.float64), st["window_qpos"][0, 1].astype(np.float64)
    np.testing.assert_allclose(np.stack([q5, x6]), SMC.interpolation(SMC.clipped_anchor(o, q4), x7, 2), atol=1e-5)
    r2 = FL.fixed_lag_step(seq, kp[:, 10:], st, fixed_qpos=None if fx is None else fx[:, 10:], flush=True)
    status = np.concatenate([r["status"][0], r2["status"][0]])
    miss = (status & STATUS_MISSING) != 0
    np.testing.assert_array_equal(miss[L:], np.isin(np.arange(T - L), [5, 6]))
    assert not miss[:L].any() and (status[:L] == STATUS_PENDING).all()


@pytest.mark.parametrize("case", CASES[:2] + CASES[4:5], ids=IDS[:2] + IDS[4:5])
def test_splitting_is_invisible(case, tmp_path):
    """K ticks in one call, the same ticks over three calls (the state round-tripped through copies in between), and each
    stream alone or in another order: the same bits, flush included."""
    seq, o = _setup(case, tmp_path)
    S, K, L = 3, 6, 2
    kp, fx = SV.stream_inputs(o, S, K, 81)
    kp[1, 3] = np.nan
    st0 = _state(seq, o, S, L, 82)
    st = FL.copy_state(st0)
    one = FL.fixed_lag_step(seq, kp, st, fixed_qpos=fx, flush=True)
    sp = FL.copy_state(st0)
    parts = []
    for a, b in ((0, 1), (1, 4), (4, 6)):
        sp = FL.copy_state(sp)
        parts.append(FL.fixed_lag_step(seq, kp[:, a:b], sp, fixed_qpos=None if fx is None else fx[:, a:b]))
    fl = FL.fixed_lag_step(seq, None, sp, flush=True)
    for k in ("qpos", "robot_qpos", "status"):
        np.testing.assert_array_equal(np.concatenate([p[k] for p in parts], axis=1), one[k])
    for k in ("flush_qpos", "flush_robot_qpos", "flush_count"):
        np.testing.assert_array_equal(fl[k], one[k])
    for k in FL.STATE:
        if st[k] is not None:
            np.testing.assert_array_equal(sp[k], st[k], err_msg=k)
    order = [2, 0, 1]
    sr = {k: (v[order] if isinstance(v, np.ndarray) else v) for k, v in st0.items()}
    rev = FL.fixed_lag_step(seq, kp[order], sr, fixed_qpos=None if fx is None else fx[order], flush=True)
    for k in ("qpos", "status", "flush_qpos", "flush_count"):
        np.testing.assert_array_equal(rev[k], one[k][order])
    s1 = {k: (v[1:2] if isinstance(v, np.ndarray) else v) for k, v in st0.items()}
    alone = FL.fixed_lag_step(seq, kp[1:2], s1, fixed_qpos=None if fx is None else fx[1:2], flush=True)
    for k in ("qpos", "robot_qpos", "status", "flush_qpos", "flush_count"):
        np.testing.assert_array_equal(alone[k], one[k][1:2])


def test_nonfinite_state_is_flagged_until_reset(tmp_path):
    seq, o = _setup(CASES[1], tmp_path)
    S, K, L = 2, 4, 1
    kp, fx = SV.stream_inputs(o, S, K, 91)
    st0 = _state(seq, o, S, L, 92)
    st = FL.copy_state(st0)
    ref = FL.fixed_lag_step(seq, kp, st)
    st = FL.copy_state(st0)
    st["last_qpos"][1, 0] = np.nan
    r = FL.fixed_lag_step(seq, kp, st)
    assert (r["status"][1, :L] == STATUS_PENDING).all() and (r["status"][1, L:] == STATUS_NONFINITE).all()
    np.testing.assert_array_equal(r["qpos"][0], ref["qpos"][0])
    np.testing.assert_array_equal(r["status"][0], ref["status"][0])


def test_argument_checks(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    kp, _ = SV.stream_inputs(o, 2, 2, 101)

    def err(null=(), **kw):
        st = _state(seq, o, 2, 1, 102)
        before = FL.copy_state(st)
        with pytest.raises(EmulationError) as e:
            FL.fixed_lag_step(seq, kp, st, null=null, **kw)
        assert e.value.code == N_INVALID
        for k in FL.STATE:  # a refused call writes nothing
            if st[k] is not None:
                np.testing.assert_array_equal(st[k], before[k])
        return e.value.msg

    for name in ("last_qpos", "window_keypoints", "window_qpos", "window_len"):
        assert "required" in err(null=(name,)), name
    assert "required" in err(null=("keypoints",))
    assert "required" in err(null=("qpos_out",))
    assert "projected" in err(null=("projected",))
    assert "lag" in err(lag=-1)
    assert "lag" in err(lag=4096)
    assert "INT32_MAX" in err(num_streams=2 ** 31 // 2, lag=1)
    assert "sizes" in err(num_streams=-1)
    assert "sizes" in err(num_ticks=-1)
    assert "smooth_weight" in err(smooth_weight=float("nan"))
    assert "workspace" in err(workspace_bytes=FL.workspace_bytes(seq, 2, 1) - 1)
    assert "workspace" in err(null=("workspace",))
    prm = seq.optimizer.params(raw_hand=None)
    prm.preprocess = 1
    assert "preprocess" in err(params=prm)
    # a flush-only call needs neither keypoints nor qpos_out
    st = _state(seq, o, 2, 1, 103)
    assert FL.fixed_lag_step(seq, None, st, flush=True, null=("keypoints", "qpos_out"))["flush_count"].tolist() == [0, 0]


def test_fixed_joints_are_required(tmp_path):
    seq, o = _setup(CASES[5], tmp_path)
    kp, fx = SV.stream_inputs(o, 1, 1, 111)
    assert fx is not None
    for null in (("fixed_qpos",), ("window_fixed_qpos",)):
        with pytest.raises(EmulationError, match="fixed"):
            FL.fixed_lag_step(seq, kp, _state(seq, o, 1, 1, 112), fixed_qpos=fx, null=null)


@pytest.mark.parametrize("case", [CASES[1], CASES[2]], ids=[IDS[1], IDS[2]])
def test_workspace_size(case, tmp_path):
    """S (L+1) frames of the smoother's workspace, (G^2 + 5 G) floats each, then S (L+1) status words; the library agrees
    on a null robot."""
    seq, o = _setup(case, tmp_path)
    G = 16 if seq.optimizer.build_table().dof <= 16 else 32
    assert FL.workspace_bytes(seq, 3, 4) == 3 * 5 * (G * G + 5 * G) * 4 + 3 * 5 * 4
    assert FL.workspace_bytes(seq, 3, 0) == 3 * (G * G + 5 * G) * 4 + 3 * 4
    assert FL.workspace_bytes(seq, 0, 4) == 0
    from dex_retargeting_b200 import _native as N

    assert N.load().dexr_fixed_lag_workspace_bytes(None, 3, 4) == 0


def test_fixed_lag_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v`: both dexr_fixed_lag_kernel instantiations spill nothing at the smoother's launch bounds."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    fl = {k: v for k, v in stores.items() if "dexr_fixed_lag_kernel" in k}
    assert len(fl) == 2, sorted(stores)
    assert all(v == 0 for v in fl.values()), fl


def test_gpu_fixed_lag_file_passes_against_the_emulation():
    """tests/test_gpu_fixed_lag.py dry-run on the CPU (tests/tools/emu_gpu_fixed_lag.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_fixed_lag.py")], capture_output=True,
                         text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
