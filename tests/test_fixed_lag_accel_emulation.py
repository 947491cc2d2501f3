"""Fixed-lag smoothing with an acceleration penalty (`dexr_fixed_lag_step_accel`) through the host emulation of the kernel's
own driver (tests/emu runs fixed_lag_tick<G, false, true> and fixed_lag_flush<G, true> of dexr_kernels.cuh on the fiber
warp), on the case list of tests/test_fixed_lag_emulation.py: each tick, before and after commits, is
smooth_packed_stream<G, true, true> on the window rebuilt from the state, bit for bit, and the float64 minimiser of
tests/fixed_lag_accel_cases.py; a fresh stream with L >= T - 1 and a flush is the offline accel smoother bit for bit; L = 0
is the causal constant-velocity minimiser; splitting a run or batching streams changes no bit; a non-finite pre-anchor is
isolated; the pre-anchor is clipped at use; the penalty does not grow the second differences; the argument checks, the
workspace size, the register budget and a dry run of tests/test_gpu_fixed_lag_accel.py."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_fixed_lag_accel_host as FA
import emu_smooth_accel_host as SA
import fixed_lag_accel_cases as FAC
import seq_vjp_cases as SV
from emu_eval_host import EmulationError
from test_fixed_lag_emulation import CASES, IDS, _causal_flags, _nd, _setup

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID
STATUS_MAXITER, STATUS_NONFINITE, STATUS_MISSING, STATUS_PENDING = 1 << 24, 1 << 25, 1 << 27, 1 << 28
C_OVER_W = 10.0  # c = 10 w, the weight DESIGN.md 3.16 recommends


def _state(seq, o, S, lag, seed, c):
    """A fresh accelerated state with a seeded warm start inside the joint limits."""
    st = FA.fresh_state(seq, S, lag, c)
    rng = np.random.RandomState(seed)
    st["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0],
                                   o.joint_limits[:, 1])
    return st


def _copy(st):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}


def _window(snap, kp, fx, s):
    """Stream s's window rebuilt from the state `snap` before a tick and its new frame: (h, keypoints, qpos_init, fixed)."""
    h = int(snap["window_len"][s])
    wk = np.concatenate([snap["window_keypoints"][s, :h], kp[s:s + 1]])
    start = snap["window_qpos"][s, h - 1:h] if h else snap["last_qpos"][s:s + 1]
    wq = np.concatenate([snap["window_qpos"][s, :h], start])
    wf = None if fx is None else np.concatenate([snap["window_fixed_qpos"][s, :h], fx[s:s + 1]])
    return h, wk, wq, wf


def _check_tick(seq, snap, st, r, kp, fx, w=-1.0):
    """One tick against smooth_packed_stream<G, true, true> on every stream's rebuilt window, bit for bit: the emitted row
    (or NaN and PENDING), the status, the new window, the anchor, prev_qpos and has_prev.  Returns each stream's window
    answer and window frames' count."""
    L, c = st["lag"], st["accel_weight"]
    out = []
    for s in range(kp.shape[0]):
        h, wk, wq, wf = _window(snap, kp[:, 0], None if fx is None else fx[:, 0], s)
        pj = None if snap["projected"] is None else snap["projected"][s:s + 1]
        q, rq, status, _ = FA.smooth_pre_anchor(seq, wk, [0, h + 1], wq, c, snap["last_qpos"][s:s + 1],
                                                snap["prev_qpos"][s:s + 1], snap["has_prev"][s:s + 1], projected=pj,
                                                fixed_qpos=wf, smooth_weight=w)
        if h == L:
            np.testing.assert_array_equal(r["qpos"][s, 0], q[0])
            np.testing.assert_array_equal(r["robot_qpos"][s, 0], rq[0])
            assert r["status"][s, 0] == status[0], (s, r["status"][s, 0], status[0])
            np.testing.assert_array_equal(st["window_qpos"][s, :L], q[1:])
            np.testing.assert_array_equal(st["last_qpos"][s], q[0])
            np.testing.assert_array_equal(st["prev_qpos"][s], snap["last_qpos"][s])
            assert st["has_prev"][s] == 1 and st["window_len"][s] == L
        else:
            assert r["status"][s, 0] == STATUS_PENDING
            assert np.isnan(r["qpos"][s, 0]).all() and np.isnan(r["robot_qpos"][s, 0]).all()
            np.testing.assert_array_equal(st["window_qpos"][s, :h + 1], q)
            for k in ("last_qpos", "prev_qpos", "has_prev"):
                np.testing.assert_array_equal(st[k][s], snap[k][s])
            assert st["window_len"][s] == h + 1
        out.append((q, status, wk, wf))
    return out


@pytest.mark.parametrize("lag", [0, 1, 4])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_each_tick_is_the_window_solve(case, lag, tmp_path):
    """Snapshot, one tick, the pre-anchor smoother on the rebuilt window: the same bits, before the window fills, on the
    first commit (has_prev = 0) and after commits (has_prev = 1); each window answer is the float64 minimiser."""
    seq, o = _setup(case, tmp_path)
    S, K = 2, lag + 3
    kp, fx = SV.stream_inputs(o, S, K, 131 + lag)
    c = C_OVER_W * _nd(seq)
    st = _state(seq, o, S, lag, 132, c)
    w = -1.0 if lag != 1 else 2.0 * _nd(seq)  # a smoothing weight other than norm_delta on the L = 1 runs
    flags = [_causal_flags(seq, kp[s], None if fx is None else fx[s]) for s in range(S)]
    checked = 0
    for k in range(K):
        snap = _copy(st)
        kk, ff = kp[:, k:k + 1], None if fx is None else fx[:, k:k + 1]
        r = FA.fixed_lag_step(seq, kk, st, fixed_qpos=ff, smooth_weight=w)
        for s, (q, status, wk, wf) in enumerate(_check_tick(seq, snap, st, r, kk, ff, w)):
            if status[0] & (STATUS_MAXITER | STATUS_NONFINITE):
                continue
            m_ = len(q)
            fl = None if flags[s] is None else flags[s][k + 1 - m_:k + 1]
            pre = FAC.clipped(o, snap["prev_qpos"][s]) if snap["has_prev"][s] else None
            m = FAC.Model(o, wk, wf, fl, FAC.clipped(o, snap["last_qpos"][s]), _nd(seq) if w < 0 else w, c, pre)
            X = q.astype(np.float64)
            assert np.abs(m.polish(X) - X).max() <= FAC.PARITY, (k, s)
            checked += 1
    assert checked >= S * K // 2
    assert (st["has_prev"] == 1).all()


@pytest.mark.parametrize("case", CASES[1:2] + CASES[4:5], ids=IDS[1:2] + IDS[4:5])
def test_pre_anchor_is_clipped_at_use(case, tmp_path):
    """A warm start outside the clip range, L = 1: the first commit stores it raw as prev_qpos, and the next window's
    triple uses clip(p) -- that window is the float64 minimiser with the clipped pre-anchor, and not with the raw one."""
    seq, o = _setup(case, tmp_path)
    S, K, L = 2, 4, 1
    kp, fx = SV.stream_inputs(o, S, K, 195)
    c = C_OVER_W * _nd(seq)
    st = _state(seq, o, S, L, 196, c)
    st["last_qpos"][:, ::2] = o.joint_limits[::2, 1] + 0.3  # outside the clip range
    raw = st["last_qpos"].copy()
    sl = (lambda a, i, j: None if a is None else a[:, i:j])
    FA.fixed_lag_step(seq, kp[:, :2], st, fixed_qpos=sl(fx, 0, 2))  # fills the window, commits the first frame
    np.testing.assert_array_equal(st["prev_qpos"], raw)  # (stored raw)
    assert (st["has_prev"] == 1).all()
    snap = _copy(st)
    r = FA.fixed_lag_step(seq, kp[:, 2:3], st, fixed_qpos=sl(fx, 2, 3))
    flags = [_causal_flags(seq, kp[s], None if fx is None else fx[s]) for s in range(S)]
    for s in range(S):
        assert not r["status"][s, 0] & (STATUS_MAXITER | STATUS_NONFINITE)
        X = np.concatenate([r["qpos"][s, :1], st["window_qpos"][s, :L]]).astype(np.float64)
        wk = np.concatenate([snap["window_keypoints"][s, :1], kp[s, 2:3]])
        wf = None if fx is None else np.concatenate([snap["window_fixed_qpos"][s, :1], fx[s, 2:3]])
        fl = None if flags[s] is None else flags[s][1:3]
        a = FAC.clipped(o, snap["last_qpos"][s])
        m = FAC.Model(o, wk, wf, fl, a, _nd(seq), c, FAC.clipped(o, raw[s]))
        assert np.abs(m.polish(X) - X).max() <= FAC.PARITY, s
        m_raw = FAC.Model(o, wk, wf, fl, a, _nd(seq), c, raw[s].astype(np.float64))
        assert np.abs(m_raw.polish(X) - X).max() > 10 * FAC.PARITY, s


@pytest.mark.parametrize("case", CASES[:3] + CASES[4:5], ids=IDS[:3] + IDS[4:5])
def test_lag_zero_is_the_constant_velocity_minimiser(case, tmp_path):
    """L = 0: every tick emits the float64 minimiser of L_t(x) + w |x - clip(a)|^2 + c |x - 2 clip(a) + clip(p)|^2 (no c
    term on the first frame of a fresh stream), with the flags of the causal walk."""
    seq, o = _setup(case, tmp_path)
    T = 5
    kp, fx = SV.stream_inputs(o, 1, T, 141, pinch=True)
    c = C_OVER_W * _nd(seq)
    st = _state(seq, o, 1, 0, 142, c)
    hist = [st["last_qpos"][0].copy()]
    r = FA.fixed_lag_step(seq, kp, st, fixed_qpos=fx)
    assert not (r["status"] & (STATUS_PENDING | STATUS_MAXITER | STATUS_NONFINITE)).any(), r["status"]
    flags = _causal_flags(seq, kp[0], None if fx is None else fx[0])
    for t in range(T):
        pre = FAC.clipped(o, hist[-2]) if t >= 1 else None
        m = FAC.Model(o, kp[0, t:t + 1], None if fx is None else fx[0, t:t + 1], None if flags is None else flags[t:t + 1],
                      FAC.clipped(o, hist[-1]), _nd(seq), c, pre)
        X = r["qpos"][0, t:t + 1].astype(np.float64)
        assert np.abs(m.polish(X) - X).max() <= FAC.PARITY, t
        hist.append(r["qpos"][0, t])
    np.testing.assert_array_equal(st["last_qpos"][0], r["qpos"][0, -1])
    np.testing.assert_array_equal(st["prev_qpos"][0], r["qpos"][0, -2])


@pytest.mark.parametrize("case,T,lag", [(CASES[0], 5, 4), (CASES[1], 5, 6), (CASES[2], 4, 3), (CASES[3], 5, 4),
                                        (CASES[4], 4, 5)], ids=["leap_dexpilot-T5-L4", "allegro_vector-T5-L6",
                                                                "shadow_position-T4-L3", "mimic_dense16-T5-L4",
                                                                "mimic_fixed_dense32-T4-L5"])
def test_full_lag_and_flush_is_the_offline_accel_smoother(case, T, lag, tmp_path):
    """A fresh stream, L >= T - 1, then a flush: T frames, bit for bit the offline accel smoother of the whole clip from
    the same anchor -- with DexPilot flags, a warm start outside the clip range and a dropped frame; the flush leaves
    prev_qpos at the second-to-last frame."""
    seq, o = _setup(case, tmp_path)
    kp, fx = SV.stream_inputs(o, 1, T, 151, pinch=True)
    kp[0, 1] = np.nan
    c = C_OVER_W * _nd(seq)
    st = _state(seq, o, 1, lag, 152, c)
    st["last_qpos"][0, ::2] = o.joint_limits[::2, 1] + 0.3  # outside the clip range: clipped at use
    a0 = st["last_qpos"].copy()
    pj = None if st["projected"] is None else st["projected"].copy()
    sl = (lambda a, i, j: None if a is None else a[:, i:j])
    r0 = FA.fixed_lag_step(seq, kp[:, :T - 1], st, fixed_qpos=sl(fx, 0, T - 1))
    assert (r0["status"] == STATUS_PENDING).all()
    # the last tick's solve is the whole clip, started from the window it holds plus the appended frame
    wq = np.concatenate([st["window_qpos"][0, :T - 1], st["window_qpos"][0, T - 2:T - 1]])
    r = FA.fixed_lag_step(seq, kp[:, T - 1:], st, fixed_qpos=sl(fx, T - 1, T), flush=True)
    live = (r["status"][0] & STATUS_PENDING) == 0
    n = int(r["flush_count"][0])
    assert live.sum() + n == T
    X = np.concatenate([r["qpos"][0, live], r["flush_qpos"][0, :n]])
    q, _, ref_status, _ = SA.smooth_packed(seq, kp[0], [0, T], wq, c, last_qpos=a0, projected=pj,
                                           fixed_qpos=None if fx is None else fx[0])
    np.testing.assert_array_equal(X, q)
    if live.any():
        assert r["status"][0, 0] == ref_status[0]
    np.testing.assert_array_equal(st["last_qpos"][0], q[-1])
    np.testing.assert_array_equal(st["prev_qpos"][0], q[-2])
    assert st["has_prev"][0] == 1 and st["window_len"][0] == 0


@pytest.mark.parametrize("case", CASES[:2] + CASES[4:5], ids=IDS[:2] + IDS[4:5])
def test_splitting_is_invisible(case, tmp_path):
    """K ticks in one call, the same ticks over three calls and a flush-only call, and each stream alone or in another
    order: the same bits, the pre-anchor state included; a dropped frame on one stream."""
    seq, o = _setup(case, tmp_path)
    S, K, L = 3, 6, 2
    kp, fx = SV.stream_inputs(o, S, K, 161)
    kp[1, 3] = np.nan
    st0 = _state(seq, o, S, L, 162, C_OVER_W * _nd(seq))
    cp = _copy
    st = cp(st0)
    one = FA.fixed_lag_step(seq, kp, st, fixed_qpos=fx, flush=True)
    sp = cp(st0)
    parts = []
    for a, b in ((0, 1), (1, 4), (4, 6)):
        sp = cp(sp)
        parts.append(FA.fixed_lag_step(seq, kp[:, a:b], sp, fixed_qpos=None if fx is None else fx[:, a:b]))
    fl = FA.fixed_lag_step(seq, None, sp, flush=True)
    for k in ("qpos", "robot_qpos", "status"):
        np.testing.assert_array_equal(np.concatenate([p[k] for p in parts], axis=1), one[k])
    for k in ("flush_qpos", "flush_robot_qpos", "flush_count"):
        np.testing.assert_array_equal(fl[k], one[k])
    for k in FA.STATE:
        if st[k] is not None:
            np.testing.assert_array_equal(sp[k], st[k], err_msg=k)
    order = [2, 0, 1]
    sr = {k: (v[order] if isinstance(v, np.ndarray) else v) for k, v in st0.items()}
    rev = FA.fixed_lag_step(seq, kp[order], sr, fixed_qpos=None if fx is None else fx[order], flush=True)
    for k in ("qpos", "status", "flush_qpos", "flush_count"):
        np.testing.assert_array_equal(rev[k], one[k][order])
    s1 = {k: (v[1:2] if isinstance(v, np.ndarray) else v) for k, v in st0.items()}
    alone = FA.fixed_lag_step(seq, kp[1:2], s1, fixed_qpos=None if fx is None else fx[1:2], flush=True)
    for k in ("qpos", "robot_qpos", "status", "flush_qpos", "flush_count"):
        np.testing.assert_array_equal(alone[k], one[k][1:2])


def test_nonfinite_pre_anchor_is_isolated(tmp_path):
    """A NaN prev_qpos with has_prev = 1 makes its stream's next window solve NONFINITE (the smoother's non-finite start:
    the warm start is emitted and committed, which moves the pre-anchor on); the other stream is untouched; with has_prev
    = 0 the same NaN is never read."""
    seq, o = _setup(CASES[1], tmp_path)
    S, K, L = 2, 4, 1
    kp, fx = SV.stream_inputs(o, S, K, 171)
    st0 = _state(seq, o, S, L, 172, C_OVER_W * _nd(seq))
    cp = _copy
    ref = FA.fixed_lag_step(seq, kp, cp(st0))
    st = cp(st0)
    st["prev_qpos"][1, 0] = np.nan
    same = FA.fixed_lag_step(seq, kp, st)
    for k in ("qpos", "status"):
        np.testing.assert_array_equal(same[k], ref[k])
    st = cp(st0)
    st["prev_qpos"][1, 0] = np.nan
    st["has_prev"][1] = 7  # (any non-zero value reads as 1)
    r = FA.fixed_lag_step(seq, kp, st)
    # the first window solve that sees the pre-anchor is a non-finite start; its commit moves the pre-anchor on
    assert (r["status"][1, :L] == STATUS_PENDING).all() and r["status"][1, L] == STATUS_NONFINITE
    np.testing.assert_array_equal(r["qpos"][1, L], st0["last_qpos"][1])  # (the warm start as given)
    assert not (r["status"][1, L + 1:] & STATUS_NONFINITE).any()
    assert np.isfinite(st["prev_qpos"]).all()
    np.testing.assert_array_equal(r["qpos"][0], ref["qpos"][0])
    np.testing.assert_array_equal(r["status"][0], ref["status"][0])


@pytest.mark.parametrize("case", CASES[1:2], ids=IDS[1:2])
def test_penalty_does_not_grow_second_differences(case, tmp_path):
    """One window with a pre-anchor, the float64 minimiser at c = 0, w, 10 w, 100 w (each polished from the last): the sum
    of squared second differences (the pre-anchor triple included) does not grow with c."""
    seq, o = _setup(case, tmp_path)
    T = 5
    kp, fx = SV.stream_inputs(o, 1, T, 181)
    flags = _causal_flags(seq, kp[0], None if fx is None else fx[0])
    rng = np.random.RandomState(182)
    a = FAC.clipped(o, o.joint_limits.mean(1) + 0.1 * rng.randn(o.opt_dof))
    p = FAC.clipped(o, a - 0.05 * rng.randn(o.opt_dof))
    w = _nd(seq)
    X = np.repeat(a[None], T, 0)
    acc = []
    for cw in (0.0, 1.0, 10.0, 100.0):
        m = FAC.Model(o, kp[0], None if fx is None else fx[0], flags, a, w, cw * w, p)
        X = m.polish(X, iters=60)
        acc.append(FAC.Model(o, kp[0], None if fx is None else fx[0], flags, a, w, 1.0, p).accel_value(X))
    assert all(acc[i + 1] <= acc[i] * (1 + 1e-6) + 1e-12 for i in range(3)), acc
    assert acc[-1] < acc[0]


def test_argument_checks(tmp_path):
    seq, o = _setup(CASES[0], tmp_path)
    kp, _ = SV.stream_inputs(o, 2, 2, 191)
    c = C_OVER_W * _nd(seq)

    def err(null=(), **kw):
        st = _state(seq, o, 2, 1, 192, c)
        before = _copy(st)
        with pytest.raises(EmulationError) as e:
            FA.fixed_lag_step(seq, kp, st, null=null, **kw)
        assert e.value.code == N_INVALID
        for k in FA.STATE:  # a refused call writes nothing
            if st[k] is not None:
                np.testing.assert_array_equal(st[k], before[k])
        return e.value.msg

    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert "accel_weight" in err(accel_weight=bad), bad
    assert "required" in err(null=("prev_qpos",))
    assert "required" in err(null=("has_prev",))
    assert "dexr_fixed_lag_accel_workspace_bytes" in err(workspace_bytes=FA.workspace_bytes(seq, 2, 1) - 1)
    # dexr_fixed_lag_step's own checks
    assert "lag" in err(lag=-1)
    assert "required" in err(null=("window_qpos",))
    assert "smooth_weight" in err(smooth_weight=float("nan"))
    prm = seq.optimizer.params(raw_hand=None)
    prm.preprocess = 1
    assert "preprocess" in err(params=prm)
    # no streams: nothing is read
    st = _state(seq, o, 2, 1, 193, c)
    FA.fixed_lag_step(seq, kp, st, num_streams=0, null=("prev_qpos", "has_prev"))


@pytest.mark.parametrize("case", [CASES[1], CASES[2]], ids=[IDS[1], IDS[2]])
def test_workspace_size(case, tmp_path):
    """S (L+1) frames of the accel smoother's workspace, (2 G^2 + 5 G) floats each, then S (L+1) status words; the library
    agrees on a null robot."""
    seq, o = _setup(case, tmp_path)
    G = 16 if seq.optimizer.build_table().dof <= 16 else 32
    assert FA.workspace_bytes(seq, 3, 4) == 3 * 5 * (2 * G * G + 5 * G) * 4 + 3 * 5 * 4
    assert FA.workspace_bytes(seq, 3, 0) == 3 * (2 * G * G + 5 * G) * 4 + 3 * 4
    assert FA.workspace_bytes(seq, 0, 4) == 0
    from dex_retargeting_b200 import _native as N

    assert N.load().dexr_fixed_lag_accel_workspace_bytes(None, 3, 4) == 0


# spill stores (bytes) -Xptxas -v reports for dexr_fixed_lag_accel_kernel<16> / <32> (DESIGN.md 3.17)
SPILL_BUDGET = {16: 36, 32: 0}


def test_fixed_lag_accel_kernel_register_budget(tmp_path):
    """`-Xptxas -v`: dexr_fixed_lag_accel_kernel<32> spills nothing and <16> no more than it reaches today."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    fl = {k: v for k, v in stores.items() if "dexr_fixed_lag_accel_kernel" in k}
    assert len(fl) == 2, sorted(stores)
    for G, budget in SPILL_BUDGET.items():
        got = [v for k, v in fl.items() if f"ILi{G}E" in k]
        assert got and got[0] <= budget, (G, fl)


def test_gpu_fixed_lag_accel_file_passes_against_the_emulation():
    """tests/test_gpu_fixed_lag_accel.py dry-run on the CPU (tests/tools/emu_gpu_fixed_lag_accel.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_fixed_lag_accel.py")], capture_output=True,
                         text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
