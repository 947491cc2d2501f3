"""Backpropagation through the offline smoother (`dexr_smooth_sequences_packed_vjp`) through the host emulation of the
kernel's own driver (tests/emu runs smooth_vjp_packed_stream of dexr_kernels.cuh on the fiber warp): the float64 model of
tests/smooth_vjp_cases.py, itself checked against central differences of the re-polished minimiser, on the packaged LEAP
DexPilot, Allegro and Shadow configs and on structure cases with fixed, mimic and prismatic joints at 16 and 32 lanes;
missing frames, NOT_PD and non-finite streams, zero-length and malformed ranges, stream independence, non-causality, the
argument checks, the register budget and a dry run of tests/test_gpu_smooth_vjp.py.  Every output buffer lies between
guard words (tests/emu_smooth_vjp_host.py)."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_packed_host as P
import emu_smooth_host as SM
import emu_smooth_vjp_host as SVH
import seq_vjp_cases as SV
import smooth_cases as SMC
import smooth_vjp_cases as SVC
import structure_cases as SC
from emu_eval_host import EmulationError
from emu_seq_vjp_host import fresh_state
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID

# (name, how to build it)
CASES = [
    ("leap_dexpilot", ("teleop/leap_hand_right_dexpilot", None)),
    ("allegro_vector", ("teleop/allegro_hand_right", None)),
    ("shadow_position", ("offline/shadow_hand_right", None)),
    ("fixed_dense16", "fixed_dense16"),
    ("mimic_dense16", "mimic_dense16"),
    ("mimic_fixed_dense32", "mimic_fixed_dense32"),
    ("prismatic_arrow", "prismatic_arrow"),
]
IDS = [c[0] for c in CASES]
BY_NAME = dict(CASES)


def _setup(name, tmp_path):
    spec = BY_NAME[name]
    if isinstance(spec, str):
        return SC.build(SC.BY_ID[spec], tmp_path)
    return build_product(*spec), build_oracle(*spec)


def _inputs(o, lengths, seed):
    T = max(int(max(lengths)), 1)
    kp, fixed = SV.stream_inputs(o, len(lengths), T, seed)
    pk = np.concatenate([kp[s, :n] for s, n in enumerate(lengths)]).reshape(-1, 21, 3)
    pf = None if fixed is None else np.concatenate([fixed[s, :n] for s, n in enumerate(lengths)]).reshape(-1, fixed.shape[2])
    return pk, pf


def _smoothed(seq, o, lengths, seed):
    """Inputs, the state before, the causal tape and the emulated smoother's answer of `lengths` clips."""
    pk, pf = _inputs(o, lengths, seed)
    rng = np.random.RandomState(seed + 1)
    st0 = fresh_state(seq, len(lengths))
    st0["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(len(lengths), o.opt_dof),
                                    o.joint_limits[:, 0], o.joint_limits[:, 1])
    st = {k: None if v is None else v.copy() for k, v in st0.items()}
    _, _, _, tape = P.solve_packed(seq, pk, P.offsets_of(lengths), state=st, fixed_qpos=pf, record=True)
    q, _, status, _ = SM.smooth_packed(seq, pk, P.offsets_of(lengths), tape["qpos"], last_qpos=st0["last_qpos"],
                                       projected=st0["projected"], fixed_qpos=pf)
    return dict(kp=pk, fixed=pf, st0=st0, tape=tape, q=q, status=status, offs=P.offsets_of(lengths))


def _cotangents(seq, Nf, seed):
    rng = np.random.RandomState(seed)
    return (rng.randn(Nf, seq.optimizer.opt_dof).astype(np.float32),
            rng.randn(Nf, seq.optimizer.robot.dof).astype(np.float32))


def _vjp(seq, r, gq, grq, **kw):
    return SVH.smooth_vjp_packed(seq, r["kp"], r["offs"], r["q"], last_qpos=r["st0"]["last_qpos"],
                                 projected=r["st0"]["projected"], fixed_qpos=r["fixed"], grad_qpos=gq,
                                 grad_robot_qpos=grq, **kw)


def _models(seq, o, r, gq, grq, X=None):
    nd = float(seq.optimizer.params().norm_delta)
    anch = SMC.clipped_anchor(o, r["st0"]["last_qpos"])
    out = []
    for s in range(len(r["offs"]) - 1):
        a, b = int(r["offs"][s]), int(r["offs"][s + 1])
        if b == a:
            out.append(None)
            continue
        fl = None if r["tape"]["projected"] is None else r["tape"]["projected"][a:b]
        fx = None if r["fixed"] is None else r["fixed"][a:b]
        m = SMC.Model(o, r["kp"][a:b], fx, fl, anch[s], nd)
        out.append(SVC.model_stream(m, r["q"][a:b] if X is None else X[a:b], r["kp"][a:b], fx, fl, r["st0"]["last_qpos"][s],
                                    gq[a:b], grq[a:b]))
    return out


@pytest.mark.parametrize("name", ["allegro_vector", "mimic_fixed_dense16"])
def test_model_matches_central_differences_of_the_minimiser(name, tmp_path):
    """<theta_bar, delta> of the model equals the central difference of l(X*(theta +- h delta)) with X* re-polished in
    float64, for l(X) = sum <grad_qpos, x_t> + <grad_robot_qpos, robot_qpos_t>, on 4- and 6-frame clips."""
    seq, o = SC.build(SC.BY_ID[name], tmp_path) if name in SC.BY_ID else _setup(name, tmp_path)
    r = _smoothed(seq, o, [4, 6], 31)
    nd = float(seq.optimizer.params().norm_delta)
    gq, grq = _cotangents(seq, len(r["q"]), 32)
    Mx, Mf = SVC.maps(o)
    rng = np.random.RandomState(33)
    lim = o.joint_limits
    for s in range(2):
        a, b = int(r["offs"][s]), int(r["offs"][s + 1])
        kp, fx = r["kp"][a:b].astype(np.float64), None if r["fixed"] is None else r["fixed"][a:b].astype(np.float64)
        fl = None if r["tape"]["projected"] is None else r["tape"]["projected"][a:b]
        a_raw = r["st0"]["last_qpos"][s].astype(np.float64)

        def model(kp_, fx_, a_):
            return SMC.Model(o, kp_, fx_, fl, np.clip(a_, lim[:, 0], lim[:, 1]), nd)

        m0 = model(kp, fx, a_raw)
        X0 = m0.polish(r["q"][a:b].astype(np.float64), iters=60)
        md = SVC.model_stream(m0, X0, kp, fx, fl, a_raw, gq[a:b], grq[a:b])
        assert not md["not_pd"], s  # (variables at a bound stay there under the small perturbations)
        dk = np.zeros_like(kp)
        used = sorted({int(i) for i in np.asarray(o.target_link_human_indices).reshape(-1)})
        dk[:, used] = rng.randn(b - a, len(used), 3)
        df = None if fx is None else rng.randn(*fx.shape)
        da = rng.randn(o.opt_dof) * ((a_raw > lim[:, 0]) & (a_raw < lim[:, 1]))  # (one-sided at a limit: left out)
        h = 1e-5
        vals = []
        for sg in (1, -1):
            kp_, fx_, a_ = kp + sg * h * dk, None if fx is None else fx + sg * h * df, a_raw + sg * h * da
            fxl = 0 if fx_ is None else fx_ @ Mf.T
            X = model(kp_, fx_, a_).polish(X0, iters=60)
            vals.append(float((gq[a:b] * X).sum() + (grq[a:b] * (X @ Mx.T + fxl)).sum()))
        fd = (vals[0] - vals[1]) / (2 * h)
        pred = float((md["keypoints"] * dk).sum() + (0 if df is None else (md["fixed"] * df).sum()) + (md["last"] * da).sum())
        assert abs(fd - pred) <= 2e-3 * max(abs(fd), 1e-3), (s, fd, pred)


@pytest.mark.parametrize("name", IDS)
def test_emulation_matches_the_model(name, tmp_path):
    seq, o = _setup(name, tmp_path)
    r = _smoothed(seq, o, [4, 6], 41)
    assert not (r["status"] & ((1 << 24) | (1 << 25))).any()
    gq, grq = _cotangents(seq, len(r["q"]), 42)
    res = _vjp(seq, r, gq, grq)
    assert not (res[3] & (SVC.STATUS_NOT_PD | SVC.STATUS_NONFINITE)).any(), res[3]
    ratio, checked = SVC.compare(res, _models(seq, o, r, gq, grq), r["offs"])
    assert checked >= 1, name
    if len(o.idx_pin2fixed):
        assert np.abs(res[1]).max() > 0  # the fixed-joint block is not vacuous


def test_gradient_is_not_causal(tmp_path):
    """A cotangent on one frame alone reaches the keypoints of the frames after it (the causal VJP never does)."""
    seq, o = _setup("allegro_vector", tmp_path)
    r = _smoothed(seq, o, [8], 51)
    gq = np.zeros_like(r["q"])
    gq[2] = np.random.RandomState(52).randn(o.opt_dof)
    g_kp, _, _, status = _vjp(seq, r, gq, None)
    assert (status == 0).all()
    assert all(np.abs(g_kp[t]).max() > 0 for t in range(3, 8))
    assert all(np.abs(g_kp[t]).max() > 0 for t in range(0, 2))


def test_missing_frames_carry_the_chain(tmp_path):
    seq, o = _setup("mimic_fixed_dense32", tmp_path)
    lengths = [9]
    pk, pf = _inputs(o, lengths, 61)
    pk[[0, 4, 8]] = np.nan
    st0 = fresh_state(seq, 1)
    st0["last_qpos"][...] = o.joint_limits.mean(1)
    st = {k: None if v is None else v.copy() for k, v in st0.items()}
    _, _, _, tape = P.solve_packed(seq, pk, P.offsets_of(lengths), state=st, fixed_qpos=pf, record=True)
    q, _, st_f, _ = SM.smooth_packed(seq, pk, P.offsets_of(lengths), tape["qpos"], last_qpos=st0["last_qpos"],
                                     fixed_qpos=pf)
    r = dict(kp=pk, fixed=pf, st0=st0, tape=tape, q=q, status=st_f, offs=P.offsets_of(lengths))
    gq, grq = _cotangents(seq, 9, 63)
    g_kp, g_f, g_l, status = _vjp(seq, r, gq, grq)
    miss = np.zeros(9, bool)
    miss[[0, 4, 8]] = True
    np.testing.assert_array_equal(status, np.where(miss, SVC.STATUS_MISSING, 0))
    assert (g_kp[miss] == 0).all() and (g_f[miss] == 0).all()
    assert np.isfinite(g_kp).all() and np.isfinite(g_l).all() and np.abs(g_l).max() > 0
    md = _models(seq, o, r, gq, grq)[0]
    SVC.compare((g_kp, g_f, g_l, status), [md], r["offs"])


def test_not_pd_and_nonfinite_streams(tmp_path):
    """Random points without an anchor or smoothing are far from any minimum: the stacked Hessian is indefinite, the stream
    gets zeros and NOT_PD on every frame.  A NaN in one stream's qpos makes that stream NaN and NONFINITE; its neighbour's
    bits do not change."""
    seq, o = _setup("allegro_vector", tmp_path)
    lengths = [3, 4]
    pk, pf = _inputs(o, lengths, 71)
    offs = P.offsets_of(lengths)
    rng = np.random.RandomState(72)
    lo, hi = o.joint_limits[:, 0], o.joint_limits[:, 1]
    X = rng.uniform(lo + 0.1 * (hi - lo), hi - 0.1 * (hi - lo), size=(7, o.opt_dof)).astype(np.float32)
    gq, _ = _cotangents(seq, 7, 73)
    g_kp, _, _, status = SVH.smooth_vjp_packed(seq, pk, offs, X, grad_qpos=gq, smooth_weight=0.0)
    for s in range(2):
        a, b = offs[s], offs[s + 1]
        m = SMC.Model(o, pk[a:b], None, None, None, 0.0)
        md = SVC.model_stream(m, X[a:b], pk[a:b], None, None, None, gq[a:b])
        if md["not_pd"]:
            assert (status[a:b] == SVC.STATUS_NOT_PD).all() and (g_kp[a:b] == 0).all(), s
    assert (status == SVC.STATUS_NOT_PD).any()
    # non-finite: stream 1 only
    r = _smoothed(seq, o, lengths, 74)
    gq, grq = _cotangents(seq, 7, 75)
    base = _vjp(seq, r, gq, grq)
    r["q"] = r["q"].copy()
    r["q"][offs[1] + 2, 1] = np.nan
    bad = _vjp(seq, r, gq, grq)
    assert np.isnan(bad[0][offs[1]:]).all() and np.isnan(bad[2][1]).all()
    assert (bad[3][offs[1]:] == SVC.STATUS_NONFINITE).all()
    for i in (0, 2, 3):
        np.testing.assert_array_equal(bad[i][:offs[1]] if i != 2 else bad[i][0], base[i][:offs[1]] if i != 2 else base[i][0])


def test_layout_zero_length_and_malformed_ranges(tmp_path):
    """Each stream's bits are those of the stream alone; a stream of length 0 writes nothing per frame and a zero anchor
    cotangent; malformed ranges read as empty."""
    seq, o = _setup("leap_dexpilot", tmp_path)
    lengths = [3, 0, 1, 4]
    r = _smoothed(seq, o, lengths, 81)
    gq, grq = _cotangents(seq, len(r["q"]), 82)
    g_kp, g_f, g_l, status = _vjp(seq, r, gq, grq)
    assert (g_l[1] == 0).all()
    offs = r["offs"]
    for s in (0, 2, 3):
        a, b = offs[s], offs[s + 1]
        sub = dict(kp=r["kp"][a:b], fixed=None, q=r["q"][a:b], offs=P.offsets_of([b - a]),
                   st0={k: None if v is None else v[s:s + 1] for k, v in r["st0"].items()})
        k1, _, l1, st1 = _vjp(seq, sub, gq[a:b], grq[a:b])
        np.testing.assert_array_equal(k1, g_kp[a:b])
        np.testing.assert_array_equal(l1[0], g_l[s])
        np.testing.assert_array_equal(st1, status[a:b])
    bad = np.array([0, 9, 2, -1, 8], np.int64)  # past N, decreasing, negative, past N: every stream reads as empty
    st2 = np.repeat(r["st0"]["last_qpos"][:1], 4, axis=0)
    k2, _, l2, s2 = SVH.smooth_vjp_packed(seq, r["kp"], bad, r["q"], last_qpos=st2, grad_qpos=gq)
    assert np.isnan(k2).all() and (s2 == -1).all() and (l2 == 0).all()


def test_argument_checks(tmp_path):
    seq, o = _setup("allegro_vector", tmp_path)
    r = _smoothed(seq, o, [3], 91)
    gq, _ = _cotangents(seq, 3, 92)

    def err(**kw):
        with pytest.raises(EmulationError) as e:
            _vjp(seq, r, gq, None, **kw)
        assert e.value.code == N_INVALID
        return e.value.msg

    assert "required" in err(null=("qpos",))
    assert "required" in err(null=("keypoints",))
    assert "required" in err(null=("grad_keypoints",))
    assert "offsets" in err(null=("offsets",))
    assert "workspace" in err(workspace_bytes=SM.workspace_bytes(seq, 3) - 4)
    assert "workspace" in err(null=("workspace",))
    assert "smooth_weight" in err(smooth_weight=float("inf"))
    assert "last_qpos" in err(null=("last_qpos",))
    prm = seq.optimizer.params(raw_hand=None)
    prm.preprocess = 1
    assert "preprocess" in err(params=prm)
    assert "sizes" in err(num_streams=-1)
    seq2, o2 = _setup("fixed_dense16", tmp_path)
    r2 = _smoothed(seq2, o2, [2], 93)
    with pytest.raises(EmulationError, match="fixed"):
        SVH.smooth_vjp_packed(seq2, r2["kp"], r2["offs"], r2["q"], null=("fixed_qpos",))


def test_smooth_vjp_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v`: both dexr_smooth_vjp_kernel instantiations spill nothing."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    ks = {k: v for k, v in stores.items() if "dexr_smooth_vjp_kernel" in k}
    assert len(ks) == 2, sorted(stores)
    assert all(v == 0 for v in ks.values()), ks


def test_gpu_smooth_vjp_file_passes_against_the_emulation():
    """tests/test_gpu_smooth_vjp.py dry-run on the CPU (tests/tools/emu_gpu_smooth_vjp.py)."""
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_smooth_vjp.py")], capture_output=True,
                         text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-2000:]
