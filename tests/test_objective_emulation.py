"""Objective evaluation (`dexr_eval_objective`, Optimizer.objective_batch / get_objective_function) through the host emulation
of the kernels' own driver (tests/emu runs evaluate_frame of dexr_kernels.cuh): against the values and gradients the
reference's closure returned, against the float64 oracle on every packaged configuration and every synthetic structure case,
against the solver's own reported cost and flags, with raw landmarks, with non-finite inputs, and its argument checks.
The GPU test file tests/test_gpu_objective.py is dry-run here as well."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_eval_host
import emu_host
import objective_cases as OC
import structure_cases as SC
from helpers import build_oracle, build_product, configs, synth_problems

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID


def _eval(opt, pts, form="ref_value", projected=None, **kw):
    inputs = {form: pts[form]}
    return emu_eval_host.eval_objective(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                        projected=projected, **inputs, **kw)


@pytest.mark.parametrize("case", OC.REF_CASES)
def test_reference_closure_values_and_gradients(case):
    """Each problem of the fixture with its 3 points as 3 frames, flags starting at 0: L(x) and the gradient are what the
    reference's own closure returned, and the flags after the call are the reference's."""
    fr = OC.reference_frames(case)
    opt = build_product(fr["key"]).optimizer
    proj = OC.initial_flags(opt, len(fr["qpos"]))
    loss, cost, grad = emu_eval_host.eval_objective(opt, fr["qpos"], ref_value=fr["ref_value"], fixed_qpos=fr["fixed_qpos"],
                                                    last_qpos=fr["last_qpos"], projected=proj)
    OC.reference_errors(loss, grad, fr["values"], fr["grads"])
    reg = opt.norm_delta * ((fr["qpos"].astype(np.float64) - fr["last_qpos"]) ** 2).sum(1)
    np.testing.assert_allclose(cost, fr["values"] + reg, rtol=OC.REF_LOSS_RTOL, atol=OC.REF_LOSS_ATOL)
    if proj is not None:
        np.testing.assert_array_equal(proj, fr["projected"])


def _against_oracle(opt, o, seed):
    for with_last in (True, False):
        pts = OC.oracle_points(o, 6, seed, with_last=with_last)
        L, Cst, G, P = OC.oracle_expect(o, pts)
        for form in ("ref_value", "keypoints"):
            proj = OC.initial_flags(opt, 6)
            loss, cost, grad = _eval(opt, pts, form, projected=proj)
            OC.oracle_errors(loss, cost, grad, L, Cst, G)
            if not with_last:
                np.testing.assert_array_equal(loss, cost)  # no anchor: no regulariser
            if proj is not None:
                np.testing.assert_array_equal(proj, P)


@pytest.mark.parametrize("key", sorted(configs()))
def test_packaged_configurations_match_oracle(key):
    """Every packaged configuration: points up to 0.2 rad beyond the bounds, keypoint and ref_value forms, with and without
    an anchor."""
    _against_oracle(build_product(key).optimizer, build_oracle(key), seed=hash(key) % 1000)


@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.id)
def test_structure_cases_match_oracle(case, tmp_path):
    """Synthetic robots at the edges of the table format: mimic and fixed joints, block widths 4 and 8, arrow tables, up to
    4 links per joint, 1 to 31 DoF, DexPilot on two and three fingers."""
    seq, o = SC.build(case, tmp_path)
    _against_oracle(seq.optimizer, o, seed=5)


@pytest.mark.parametrize("key", OC.SOLVER_CASES)
def test_agrees_with_the_solver_at_its_answer(key):
    """At the emulated solve's answer, anchored at its warm start: the solve's reported cost up to its F + dF drift, the
    solve's DexPilot flags, and a projected gradient at the fp32 floor on converged frames."""
    o, opt = build_oracle(key), build_product(key).optimizer
    refs, fixed, x0, _ = synth_problems(o, 6, np.random.RandomState(8), init_noise=0.05, target_noise=0.01)
    fixed = fixed if fixed.size else None
    proj_s = OC.initial_flags(opt, 6)
    q, status, cost = emu_host.solve_frames(opt, x0, ref_value=refs, fixed_qpos=fixed, projected=proj_s)
    proj_e = OC.initial_flags(opt, 6)
    _, cost_e, grad = emu_eval_host.eval_objective(opt, q, ref_value=refs, fixed_qpos=fixed, last_qpos=x0, projected=proj_e)
    x_start = np.clip(x0, np.float32(o.lower), np.float32(o.upper))
    _, cost0, _ = emu_eval_host.eval_objective(opt, x_start, ref_value=refs, fixed_qpos=fixed, last_qpos=x0,
                                               projected=OC.initial_flags(opt, 6), want_grad=False)
    OC.check_after_solve(o, q, status, cost, proj_s, cost0, cost_e, grad, proj_e)


@pytest.mark.parametrize("key,hand", [("teleop/allegro_hand_right", "right"), ("teleop/leap_hand_right_dexpilot", "right"),
                                      ("offline/shadow_hand_left", "left")])
def test_raw_landmarks_match_preprocessed_keypoints(key, hand):
    """params.preprocess: raw detector landmarks give what the detector's pre-processed keypoints give."""
    from oracle.preprocess import preprocess

    opt, o = build_product(key).optimizer, build_oracle(key)
    pts = OC.oracle_points(o, 6, seed=3)
    rng = np.random.RandomState(4)
    raw = []
    for k in pts["keypoints"]:
        if hand == "left":
            k = k * np.float32([-1, 1, 1])
        A, _ = np.linalg.qr(rng.randn(3, 3))
        raw.append(k @ (A * np.sign(np.linalg.det(A))).T + rng.randn(3) * 0.3)
    raw = np.array(raw, np.float32)
    pre = np.stack([preprocess(r, hand)[0] for r in raw]).astype(np.float32)
    p_raw, p_pre = OC.initial_flags(opt, 6), OC.initial_flags(opt, 6)
    a = _eval(opt, dict(pts, keypoints=raw), "keypoints", projected=p_raw, raw_hand=hand)
    b = _eval(opt, dict(pts, keypoints=pre), "keypoints", projected=p_pre)
    for u, v in zip(a, b):
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-6 * np.abs(v).max())
    if p_raw is not None:
        np.testing.assert_array_equal(p_raw, p_pre)


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_non_finite_input_stays_in_its_frame(key):
    """A NaN in one frame's qpos, and one in another frame's keypoints: those frames' outputs are non-finite, every other
    frame is bit-identical to a clean run (16-lane robots share a warp between two frames)."""
    opt, o = build_product(key).optimizer, build_oracle(key)
    pts = OC.oracle_points(o, 5, seed=9)
    clean = _eval(opt, pts, "keypoints", projected=OC.initial_flags(opt, 5))
    bad = dict(pts, qpos=pts["qpos"].copy(), keypoints=pts["keypoints"].copy())
    bad["qpos"][1, 0] = np.nan
    used = int(np.asarray(opt.target_link_human_indices).reshape(-1)[-1])
    bad["keypoints"][2, used, 1] = np.nan
    got = _eval(opt, bad, "keypoints", projected=OC.initial_flags(opt, 5))
    for out_clean, out in zip(clean, got):
        for f in (1, 2):
            assert not np.all(np.isfinite(out[f]))
        for f in (0, 3, 4):
            np.testing.assert_array_equal(out[f], out_clean[f])


def test_abi_layout_and_argument_checks(tmp_path):
    """dexr_eval_t agrees with its binding; the library rejects null arguments without a GPU, and the checks that read the
    robot's table (eval_io_error, which the library and the emulation share) reject every malformed buffer set."""
    from dex_retargeting_b200 import _native as N

    lib = N.load()
    assert lib.dexr_eval_sizeof() == C.sizeof(N.DexrEval) == 72
    p, io = N.default_params(), N.DexrEval()
    assert lib.dexr_eval_objective(None, C.byref(p), C.byref(io), 1, None) == N_INVALID
    assert b"null" in lib.dexr_last_error()
    assert lib.dexr_eval_objective(None, None, C.byref(io), 1, None) == N_INVALID

    opt = build_product("teleop/allegro_hand_right").optimizer
    x = np.zeros((2, opt.opt_dof), np.float32)
    ref = np.zeros((2, opt.num_residuals, 3), np.float32)
    kp = np.zeros((2, 21, 3), np.float32)
    for kw, msg in [(dict(qpos=None, ref_value=ref), "qpos is required"),
                    (dict(qpos=x), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, keypoints=kp), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, raw_hand="right"), "preprocess needs raw keypoints")]:
        with pytest.raises(emu_eval_host.EmulationError) as e:
            emu_eval_host.eval_objective(opt, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg
    seq, _ = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    with pytest.raises(emu_eval_host.EmulationError, match="fixed joints but fixed_qpos is NULL"):
        emu_eval_host.eval_objective(seq.optimizer, np.zeros((1, seq.optimizer.opt_dof), np.float32),
                                ref_value=np.zeros((1, seq.optimizer.num_residuals, 3), np.float32))


def test_gpu_objective_file_passes_against_the_emulation():
    """tests/test_gpu_objective.py dry-run on the CPU (tests/tools/emu_gpu_objective.py, objective_batch served by the emulation)."""
    count = 24
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_objective.py")],
                         capture_output=True, text=True, timeout=900)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
