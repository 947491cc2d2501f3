"""Backpropagation through the solve (`dexr_solve_vjp`, Optimizer.retarget_batch_vjp, objective.differentiable_retarget)
through the host emulation of the kernel's own driver (tests/emu runs vjp_frame of dexr_kernels.cuh): against the float64
implicit-function model of tests/vjp_cases.py on every reference fixture family, every packaged configuration and every
synthetic structure case, in both input forms, with and without an anchor, with preset DexPilot flags and with active
bounds; the keypoint form against the ref_value form, NaN isolation, indefinite frames, the argument checks, the kernels'
register budget.  The GPU test file tests/test_gpu_vjp.py is dry-run here as well."""
import ctypes as C
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

import emu_vjp_host
import objective_cases as OC
import structure_cases as SC
import vjp_cases as V
from helpers import build_oracle, build_product, configs

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID


def _emu(opt, pts, form, projected=None):
    proj = pts["flags"] if projected is None else projected
    return emu_vjp_host.solve_vjp(opt, pts["gbar"], pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                   projected=proj, **{form: pts[form]})


def _against_model(opt, o, n, seed, forms_no_anchor=("ref_value",)):
    """Both forms with an anchor, `forms_no_anchor` without; returns the worst error / tau."""
    worst = 0.0
    for with_last, forms in ((True, ("ref_value", "keypoints")), (False, forms_no_anchor)):
        pts = V.solved_points(o, n, seed, with_last=with_last)
        for form in forms:
            flags_before = None if pts["flags"] is None else pts["flags"].copy()
            res = _emu(opt, pts, form)
            if flags_before is not None:
                np.testing.assert_array_equal(pts["flags"], flags_before)  # read only
            worst = max(worst, V.compare(res, V.model_batch(o, pts, form), pts))
    return worst


@pytest.mark.parametrize("case", OC.REF_CASES)
def test_reference_fixture_families_match_model(case):
    """The fixture's problems (targets, fixed joints, anchors), solved to their float64 minimiser from the anchor."""
    from oracle.solvers import solve_converged

    fr = OC.reference_frames(case)
    key = fr["key"]
    o, opt = build_oracle(key), build_product(key).optimizer
    idx = np.arange(0, len(fr["qpos"]), 3)[:4]
    X, F = [], []
    for i in idx:
        if o.type == "dexpilot":
            o.projected[:] = False
        fixed = fr["fixed_qpos"][i] if fr["fixed_qpos"] is not None else np.zeros(0, np.float32)
        x, _, _ = solve_converged(o, fr["ref_value"][i], fixed, fr["last_qpos"][i])
        X.append(x.astype(np.float32))
        if o.type == "dexpilot":
            F.append(o.projected.astype(np.uint8))
    pts = dict(qpos=np.array(X), ref_value=fr["ref_value"][idx], last_qpos=fr["last_qpos"][idx],
               fixed_qpos=None if fr["fixed_qpos"] is None else fr["fixed_qpos"][idx], flags=np.array(F) if F else None,
               gbar=np.random.RandomState(2).randn(len(idx), o.opt_dof).astype(np.float32))
    ratio = V.compare(_emu(opt, pts, "ref_value"), V.model_batch(o, pts, "ref_value"), pts)
    print(case, "worst error / tau %.3f" % ratio)


@pytest.mark.parametrize("key", sorted(configs()))
def test_packaged_configurations_match_model(key):
    ratio = _against_model(build_product(key).optimizer, build_oracle(key), 3, seed=zlib.crc32(key.encode()) % 1000)
    print(key, "worst error / tau %.3f" % ratio)


@pytest.mark.parametrize("case", SC.CASES, ids=lambda c: c.id)
def test_structure_cases_match_model(case, tmp_path):
    """Fixed joints, mimic joints (the fold M^T H M and M v), prismatic joints, block widths 8, arrow tables and the
    free-flying trunk."""
    seq, o = SC.build(case, tmp_path)
    ratio = _against_model(seq.optimizer, o, 3, seed=7, forms_no_anchor=("ref_value", "keypoints"))
    print(case.id, "worst error / tau %.3f" % ratio)


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right", "teleop/ability_hand_right"])
def test_active_bounds_get_zero_sensitivity(key):
    """Anchors 0.3 beyond the joint limits: the minimisers sit on their bounds, the active variables get zero sensitivity
    (their anchor cotangent is exactly 0) and the free ones still match the model."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 4, seed=31)
    rng = np.random.RandomState(32)
    side = rng.rand(*pts["last_qpos"].shape) < 0.5
    pts["last_qpos"] = np.where(side, o.joint_limits[:, 0] - 0.3, o.joint_limits[:, 1] + 0.3).astype(np.float32)
    from oracle.solvers import solve_converged

    nf = len(o.idx_pin2fixed)
    for i in range(4):
        fixed = pts["fixed_qpos"][i] if nf else np.zeros(0, np.float32)
        pts["qpos"][i] = solve_converged(o, pts["ref_value"][i], fixed, pts["last_qpos"][i])[0].astype(np.float32)
    m = V.model_batch(o, pts, "ref_value")
    assert m["n_active"] >= 4, m["n_active"]
    res = _emu(opt, pts, "ref_value")
    at_bound = (pts["qpos"] <= np.float32(o.lower)) | (pts["qpos"] >= np.float32(o.upper))
    assert np.all(res[2][at_bound & (m["last"] == 0)] == 0)
    print(key, m["n_active"], "active variables, worst error / tau %.3f" % V.compare(res, m, pts))


def test_dexpilot_preset_flags():
    """Flags given in a state the targets move out of: the kernel runs prepare_targets on them as a solve would, the model
    holds the flags that rule gives, and the caller's buffer is unchanged."""
    key = "teleop/leap_hand_right_dexpilot"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 6, seed=33)
    preset = (np.random.RandomState(34).rand(*pts["flags"].shape) < 0.5).astype(np.uint8)
    effective = []
    for i in range(6):
        o.projected[:] = preset[i].astype(bool)
        o.prepare(pts["ref_value"][i], update_state=True)
        effective.append(o.projected.astype(np.uint8))
    given = preset.copy()
    res = _emu(opt, pts, "keypoints", projected=given)
    np.testing.assert_array_equal(given, preset)
    assert not np.array_equal(np.array(effective), preset)
    pts["flags"] = np.array(effective)
    print("worst error / tau %.3f" % V.compare(res, V.model_batch(o, pts, "keypoints"), pts))


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right", "teleop/allegro_hand_right"])
def test_keypoint_form_is_the_gather_transpose_of_the_ref_value_form(key):
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 4, seed=35)
    g_ref = _emu(opt, pts, "ref_value")
    g_kp = _emu(opt, pts, "keypoints")
    np.testing.assert_array_equal(g_ref[3], g_kp[3])
    hi = np.asarray(opt.target_link_human_indices)
    task, origin = (hi.reshape(-1), None) if opt.retargeting_type == "POSITION" else (hi[1], hi[0])
    want = np.zeros((4, 21, 3))
    for k in range(len(task)):
        want[:, task[k]] += g_ref[0][:, k]
        if origin is not None:
            want[:, origin[k]] -= g_ref[0][:, k]
    scale = np.abs(want).max()
    np.testing.assert_allclose(g_kp[0], want, rtol=0, atol=1e-5 * scale)
    np.testing.assert_array_equal(g_kp[2], g_ref[2])


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_non_finite_input_stays_in_its_frame(key):
    """A NaN in one frame's qpos, grad_qpos and keypoints: that frame's outputs are NaN with DEXR_STATUS_NONFINITE, every
    other frame is bit-identical to a clean run (16-lane robots share a warp between two frames)."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 5, seed=37)
    clean = _emu(opt, pts, "keypoints")
    used = int(np.asarray(opt.target_link_human_indices).reshape(-1)[-1])
    for f, name, at in ((1, "qpos", (1, 0)), (2, "gbar", (2, 1)), (3, "keypoints", (3, used, 1))):
        bad = dict(pts, **{name: pts[name].copy()})
        bad[name][at] = np.nan
        got = _emu(opt, bad, "keypoints")
        assert got[3][f] == V.STATUS_NONFINITE
        for out_clean, out in zip(clean[:3], got[:3]):
            if out is None:
                continue
            assert np.all(np.isnan(out[f]))
            keep = [i for i in range(5) if i != f]
            np.testing.assert_array_equal(out[keep], out_clean[keep])


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right"])
def test_indefinite_frames_give_zeros_and_not_pd(key):
    """Random points without an anchor are far from any minimum: the model's free Hessian is indefinite there.  Every output
    of those frames is 0 and the status is DEXR_STATUS_NOT_PD."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = OC.oracle_points(o, 6, 39, with_last=False)
    pts["flags"], pts["gbar"] = None, np.random.RandomState(40).randn(6, o.opt_dof).astype(np.float32)
    m = V.model_batch(o, pts, "ref_value")
    assert m["not_pd"].all()
    g_t, g_f, g_l, status = _emu(opt, pts, "ref_value")
    assert np.all(status == V.STATUS_NOT_PD)
    assert np.all(g_t == 0) and g_l is None and (g_f is None or np.all(g_f == 0))


def test_abi_layout_and_argument_checks(tmp_path):
    """dexr_vjp_t agrees with its binding; the library rejects null arguments without a GPU, and the checks that read the
    robot's table (vjp_io_error, shared by the library and the emulation) reject every malformed buffer set."""
    from dex_retargeting_b200 import _native as N

    lib = N.load()
    assert lib.dexr_vjp_sizeof() == C.sizeof(N.DexrVjp) == 96
    p, io = N.default_params(), N.DexrVjp()
    assert lib.dexr_solve_vjp(None, C.byref(p), C.byref(io), 1, None) == N_INVALID
    assert b"null" in lib.dexr_last_error()
    assert lib.dexr_solve_vjp(None, None, C.byref(io), 1, None) == N_INVALID

    opt = build_product("teleop/allegro_hand_right").optimizer
    x = np.zeros((2, opt.opt_dof), np.float32)
    ref = np.zeros((2, opt.num_residuals, 3), np.float32)
    kp = np.zeros((2, 21, 3), np.float32)
    for kw, msg in [(dict(qpos=None, ref_value=ref), "qpos is required"),
                    (dict(qpos=x, ref_value=ref, null_grad_qpos=True), "grad_qpos is required"),
                    (dict(qpos=x), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, keypoints=kp), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, keypoints=kp, raw_hand="right"), "pre-processing is not differentiated")]:
        with pytest.raises(emu_vjp_host.EmulationError) as e:
            emu_vjp_host.solve_vjp(opt, x, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg
    seq, _ = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    o2 = seq.optimizer
    with pytest.raises(emu_vjp_host.EmulationError, match="fixed joints but fixed_qpos is NULL"):
        emu_vjp_host.solve_vjp(o2, np.zeros((1, o2.opt_dof), np.float32), np.zeros((1, o2.opt_dof), np.float32),
                                ref_value=np.zeros((1, o2.num_residuals, 3), np.float32))


def test_differentiable_retarget_refuses_to_differentiate_raw_landmarks():
    torch = pytest.importorskip("torch")
    from dex_retargeting_b200.objective import differentiable_retarget

    opt = build_product("teleop/allegro_hand_right").optimizer
    kp = torch.zeros((2, 21, 3), requires_grad=True)
    with pytest.raises(ValueError, match="raw-landmark pre-processing is not differentiated"):
        differentiable_retarget(opt, keypoints=kp, last_qpos=torch.zeros((2, opt.opt_dof)), raw_hand="right")
    with pytest.raises(ValueError, match="exactly one of keypoints / ref_value"):
        differentiable_retarget(opt, last_qpos=torch.zeros((2, opt.opt_dof)))


def test_vjp_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v` of dexr_vjp_kernel<16> and <32>: no spill stores (the ptxas helpers of test_block_kernel_budget)."""
    import shutil

    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    for g in (16, 32):
        name = f"_ZN4dexr15dexr_vjp_kernelILi{g}EEEvNS_7VjpArgsE"
        assert stores.get(name) == 0, (name, stores.get(name))


def test_gpu_vjp_file_passes_against_the_emulation():
    """tests/test_gpu_vjp.py dry-run on the CPU (tests/tools/emu_gpu_vjp.py, retarget_batch_vjp served by the emulation)."""
    count = 13
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_vjp.py")], capture_output=True, text=True,
                         timeout=1800)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
