"""Per-frame Jacobians of the solve (`dexr_solve_jacobian`, Optimizer.retarget_batch_jacobian) through the host emulation of
the kernel's own driver (tests/emu runs jacobian_frame of dexr_kernels.cuh): against the float64 model of
tests/jacobian_cases.py on every reference fixture family, every packaged configuration and every synthetic structure case,
in both input forms, with and without an anchor, with active bounds and preset DexPilot flags; every row against the VJP
driver with the unit cotangent; the block structure (gather-transpose, symmetric anchor block, zero active rows and
columns); NaN isolation, indefinite frames, the argument checks, the kernels' register budget, and the VJP drivers' outputs
pinned across the split of their per-frame core.  The GPU test file tests/test_gpu_jacobian.py is dry-run here as well."""
import ctypes as C
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

import emu_jacobian_host as EJ
import emu_seq_vjp_host as SH
import emu_vjp_host
import jacobian_cases as JC
import objective_cases as OC
import structure_cases as SC
import vjp_cases as V
from helpers import build_oracle, build_product, configs, keypoint_trajectory

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID


def _emu(opt, pts, form, projected=None):
    proj = pts["flags"] if projected is None else projected
    return EJ.solve_jacobian(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"], projected=proj,
                             **{form: pts[form]})


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
            worst = max(worst, JC.compare(res, JC.model_batch(o, pts, form)))
    return worst


def _vjp_rows(opt, pts, form, projected=None):
    """The VJP driver once per unit cotangent e_i: (targets [B,n,...], fixed [B,n,nf] or None, last [B,n,n] or None,
    statuses [n,B])."""
    n = pts["qpos"].shape[1]
    proj = pts["flags"] if projected is None else projected
    rows = []
    for i in range(n):
        e = np.zeros_like(pts["qpos"])
        e[:, i] = 1.0
        rows.append(emu_vjp_host.solve_vjp(opt, e, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                           projected=proj, **{form: pts[form]}))
    stack = [None if rows[0][k] is None else np.stack([r[k] for r in rows], axis=1) for k in range(3)]
    return (*stack, np.stack([r[3] for r in rows]))


@pytest.mark.parametrize("case", OC.REF_CASES)
def test_reference_fixture_families_match_model(case):
    """The fixture's problems (targets, fixed joints, anchors), solved to their float64 minimiser from the anchor."""
    from oracle.solvers import solve_converged

    fr = OC.reference_frames(case)
    o, opt = build_oracle(fr["key"]), build_product(fr["key"]).optimizer
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
               fixed_qpos=None if fr["fixed_qpos"] is None else fr["fixed_qpos"][idx], flags=np.array(F) if F else None)
    ratio = JC.compare(_emu(opt, pts, "ref_value"), JC.model_batch(o, pts, "ref_value"))
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


def _at_bounds(o, n, seed):
    """Solved points whose anchors lie 0.3 beyond the joint limits: the minimisers sit on their bounds."""
    from oracle.solvers import solve_converged

    pts = V.solved_points(o, n, seed=seed)
    rng = np.random.RandomState(seed + 1)
    side = rng.rand(*pts["last_qpos"].shape) < 0.5
    pts["last_qpos"] = np.where(side, o.joint_limits[:, 0] - 0.3, o.joint_limits[:, 1] + 0.3).astype(np.float32)
    nf = len(o.idx_pin2fixed)
    for i in range(n):
        if o.type == "dexpilot":
            o.projected[:] = False
        fixed = pts["fixed_qpos"][i] if nf else np.zeros(0, np.float32)
        pts["qpos"][i] = solve_converged(o, pts["ref_value"][i], fixed, pts["last_qpos"][i])[0].astype(np.float32)
        if o.type == "dexpilot":
            pts["flags"][i] = o.projected.astype(np.uint8)
    return pts


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right", "teleop/ability_hand_right"])
def test_active_bounds_give_zero_rows_and_columns(key):
    """Minimisers on their bounds: the rows of the active variables are zero in every block, their columns of the anchor
    block too, and the free rows still match the model."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = _at_bounds(o, 4, seed=31)
    m = JC.model_batch(o, pts, "ref_value")
    assert m["active"].sum() >= 4, m["active"].sum()
    res = _emu(opt, pts, "ref_value")
    act = m["active"] & (res[3] == 0)[:, None]
    assert act.sum() >= 4
    for blk in res[:3]:
        if blk is not None:
            assert np.all(blk[act] == 0)
    assert np.all(np.transpose(res[2], (0, 2, 1))[act] == 0)
    print(key, int(m["active"].sum()), "active variables, worst error / tau %.3f" % JC.compare(res, m))


def test_dexpilot_preset_flags():
    """Flags given in a state the targets move out of: the kernel runs prepare_targets on them as a solve would, the model
    holds the flags that rule gives, and the caller's buffer is unchanged."""
    key = "teleop/leap_hand_right_dexpilot"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 4, seed=33)
    preset = (np.random.RandomState(34).rand(*pts["flags"].shape) < 0.5).astype(np.uint8)
    effective = []
    for i in range(4):
        o.projected[:] = preset[i].astype(bool)
        o.prepare(pts["ref_value"][i], update_state=True)
        effective.append(o.projected.astype(np.uint8))
    given = preset.copy()
    res = _emu(opt, pts, "keypoints", projected=given)
    np.testing.assert_array_equal(given, preset)
    assert not np.array_equal(np.array(effective), preset)
    pts["flags"] = np.array(effective)
    print("worst error / tau %.3f" % JC.compare(res, JC.model_batch(o, pts, "keypoints")))


ROWS_CASES = ["teleop/allegro_hand_right", "teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right",
              "mimic_fixed_dense16", "fixed_dense32"]


@pytest.mark.parametrize("key", ROWS_CASES)
def test_rows_are_the_vjps_of_the_unit_cotangents(key, tmp_path):
    """Row i of every block equals the VJP driver's output for grad_qpos = e_i, and the statuses agree: both forms, with and
    without an anchor, with active bounds, a non-finite frame and (without an anchor) frames that are not positive
    definite.  The rows run the VJP's own tail, so they are equal, not merely close."""
    if "/" in key:
        o, opt = build_oracle(key), build_product(key).optimizer
    else:
        seq, o = SC.build(SC.BY_ID[key], tmp_path)
        opt = seq.optimizer
    pts = V.solved_points(o, 3, seed=41)
    bnd = _at_bounds(o, 2, seed=43)
    pts = {k: None if pts[k] is None else np.concatenate([pts[k], bnd[k]]) for k in pts}
    pts["qpos"][1, 0] = np.nan
    rand = OC.oracle_points(o, 2, 45, with_last=False)
    for with_last in (True, False):
        p = dict(pts)
        if not with_last:
            p["last_qpos"] = None
            p["qpos"] = np.concatenate([pts["qpos"], rand["qpos"]])
            for k in ("keypoints", "ref_value", "fixed_qpos", "flags"):
                if pts[k] is not None:
                    p[k] = np.concatenate([pts[k], pts[k][:2]])
        for form in ("ref_value", "keypoints"):
            jac = _emu(opt, p, form)
            rows = _vjp_rows(opt, p, form)
            for st in rows[3]:
                np.testing.assert_array_equal(st, jac[3])
            for a, b in zip(jac[:3], rows[:3]):
                assert (a is None) == (b is None)
                if a is not None:
                    np.testing.assert_array_equal(a, b)
        if not with_last:
            assert np.any(jac[3] == V.STATUS_NOT_PD), jac[3]
    assert jac[3][1] == V.STATUS_NONFINITE


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right", "teleop/allegro_hand_right"])
def test_keypoint_block_is_the_gather_transpose_of_the_ref_value_block(key):
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 3, seed=35)
    j_ref = _emu(opt, pts, "ref_value")
    j_kp = _emu(opt, pts, "keypoints")
    np.testing.assert_array_equal(j_ref[3], j_kp[3])
    hi = np.asarray(opt.target_link_human_indices)
    task, origin = (hi.reshape(-1), None) if opt.retargeting_type == "POSITION" else (hi[1], hi[0])
    want = np.zeros(j_kp[0].shape)
    for k in range(len(task)):
        want[:, :, task[k]] += j_ref[0][:, :, k]
        if origin is not None:
            want[:, :, origin[k]] -= j_ref[0][:, :, k]
    scale = np.abs(want).max()
    np.testing.assert_allclose(j_kp[0], want, rtol=0, atol=1e-5 * scale)
    np.testing.assert_array_equal(j_kp[2], j_ref[2])


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right", "teleop/ability_hand_right"])
def test_anchor_block_is_symmetric(key):
    """2 norm_delta H_ff^-1 is symmetric: on the free variables to float32 rounding of the solves, with bounds active."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = _at_bounds(o, 3, seed=47)
    j = _emu(opt, pts, "ref_value")[2]
    for f in range(j.shape[0]):
        scale = np.abs(j[f]).max()
        assert np.abs(j[f] - j[f].T).max() <= 2e-5 * scale, (f, np.abs(j[f] - j[f].T).max() / scale)


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_non_finite_input_stays_in_its_frame(key):
    """A NaN in one frame's qpos, keypoints or anchor: that frame's blocks are NaN with DEXR_STATUS_NONFINITE, every other
    frame is bit-identical to a clean run (16-lane robots share a warp between two frames)."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 5, seed=37)
    clean = _emu(opt, pts, "keypoints")
    used = int(np.asarray(opt.target_link_human_indices).reshape(-1)[-1])
    for f, name, at in ((1, "qpos", (1, 0)), (2, "last_qpos", (2, 1)), (3, "keypoints", (3, used, 1))):
        bad = dict(pts, **{name: pts[name].copy()})
        bad[name][at] = np.nan
        got = _emu(opt, bad, "keypoints")
        assert got[3][f] == V.STATUS_NONFINITE
        keep = [i for i in range(5) if i != f]
        np.testing.assert_array_equal(got[3][keep], clean[3][keep])
        for out_clean, out in zip(clean[:3], got[:3]):
            if out is None:
                continue
            assert np.all(np.isnan(out[f]))
            np.testing.assert_array_equal(out[keep], out_clean[keep])


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right"])
def test_indefinite_frames_give_zeros_and_not_pd(key):
    """Random points without an anchor are far from any minimum: the model's free Hessian is indefinite there.  Every block
    of those frames is 0 and the status is DEXR_STATUS_NOT_PD."""
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = OC.oracle_points(o, 4, 39, with_last=False)
    pts["flags"] = None
    m = JC.model_batch(o, pts, "ref_value")
    assert m["not_pd"].all()
    j_t, j_f, j_l, status = _emu(opt, pts, "ref_value")
    assert np.all(status == V.STATUS_NOT_PD)
    assert np.all(j_t == 0) and j_l is None and (j_f is None or np.all(j_f == 0))


def test_abi_layout_and_argument_checks(tmp_path):
    """dexr_jacobian_t agrees with its binding; the library rejects null arguments without a GPU, and the checks that read
    the robot's table (jacobian_io_error, shared by the library and the emulation) reject every malformed buffer set."""
    from dex_retargeting_b200 import _native as N

    lib = N.load()
    assert lib.dexr_jacobian_sizeof() == C.sizeof(N.DexrJacobian) == 88
    p, io = N.default_params(), N.DexrJacobian()
    assert lib.dexr_solve_jacobian(None, C.byref(p), C.byref(io), 1, None) == N_INVALID
    assert b"null" in lib.dexr_last_error()
    assert lib.dexr_solve_jacobian(None, None, C.byref(io), 1, None) == N_INVALID

    opt = build_product("teleop/allegro_hand_right").optimizer
    x = np.zeros((2, opt.opt_dof), np.float32)
    ref = np.zeros((2, opt.num_residuals, 3), np.float32)
    kp = np.zeros((2, 21, 3), np.float32)
    for kw, msg in [(dict(qpos=None, ref_value=ref), "qpos is required"),
                    (dict(qpos=x), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, keypoints=kp), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, keypoints=kp, raw_hand="right"), "pre-processing is not differentiated")]:
        with pytest.raises(EJ.EmulationError) as e:
            EJ.solve_jacobian(opt, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg
    seq, _ = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    o2 = seq.optimizer
    with pytest.raises(EJ.EmulationError, match="fixed joints but fixed_qpos is NULL"):
        EJ.solve_jacobian(o2, np.zeros((1, o2.opt_dof), np.float32), ref_value=np.zeros((1, o2.num_residuals, 3), np.float32))
    # a block without its input, straight through the shared check
    table, prm = opt.build_table(), opt.params()
    xs = np.zeros((2, 21, 3, opt.opt_dof), np.float32)
    for fields, msg in [(dict(ref_value=ref, jac_keypoints=xs), "jac_keypoints needs the keypoints form"),
                        (dict(keypoints=kp, jac_ref_value=xs), "jac_ref_value needs the ref_value form"),
                        (dict(ref_value=ref, jac_last_qpos=xs), "jac_last_qpos needs last_qpos")]:
        io = N.DexrJacobian()
        io.qpos = x.ctypes.data
        for k, v in fields.items():
            setattr(io, k, v.ctypes.data)
        err = C.create_string_buffer(600)
        rc = EJ.load().emu_solve_jacobian(C.byref(table), C.byref(prm), C.byref(io), C.c_longlong(2), err, C.c_int(600))
        assert rc == N_INVALID and msg in err.value.decode(), (rc, err.value)


def test_jacobian_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v` of dexr_jacobian_kernel<16> and <32>: no spill stores (the ptxas helpers of test_block_kernel_budget)."""
    import shutil

    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    for g in (16, 32):
        name = f"_ZN4dexr20dexr_jacobian_kernelILi{g}EEEvNS_12JacobianArgsE"
        assert stores.get(name) == 0, (name, stores.get(name))


# crc32 of the emulated VJP drivers' outputs on the inputs below, as computed before their per-frame core was split into the
# front and the tail the Jacobian shares: the split must not change a bit of them
VJP_DIGESTS = {
    "ability_dexpilot_mimic": 2845471730, "allegro_vector": 2902819548, "inspire_position_mimic_dummy": 3541589151,
    "leap_dexpilot": 997135756, "panda_vector_prismatic": 1504466911, "shadow_position_dummy": 2952938229,
    "svh_vector_mimic": 4256713039, "teleop/allegro_hand_right": 543524722, "teleop/leap_hand_right_dexpilot": 1837741438,
    "offline/shadow_hand_right": 293488371, "seq teleop/allegro_hand_right": 3934735876,
    "seq teleop/leap_hand_right_dexpilot": 4012154107, "seq offline/shadow_hand_right": 4273979692,
}


def _crc(arrays):
    c = 0
    for a in arrays:
        if a is not None:
            c = zlib.crc32(np.ascontiguousarray(a).tobytes(), c)
    return c


def _streams():
    """Emulated solves of recorded keypoint streams: key -> (S, T, keypoints, tape qpos, warm start, tape flags)."""
    traj = keypoint_trajectory().astype(np.float32)
    out = {}
    for key in ("teleop/allegro_hand_right", "teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"):
        seq = build_product(key)
        S, T = 3, 3
        kp = np.ascontiguousarray(traj[:S * T * 7:7].reshape(S, T, 21, 3))
        state = SH.fresh_state(seq, S)
        last0 = state["last_qpos"].copy()
        _, _, _, tape = SH.solve_sequences_tape(seq, kp, state)
        out[key] = (S, T, kp, tape["qpos"], last0, tape["projected"])
    return out


def test_vjp_driver_outputs_are_unchanged():
    """dexr_solve_vjp's driver on the 7 reference fixture families (ref_value form, with and without the anchor) and on
    solved keypoint streams of three hands (keypoint form), and dexr_solve_sequences_vjp's on the same streams: bit for bit
    what they wrote before vjp_front / vjp_tail."""
    got = {}
    for case in OC.REF_CASES:
        fr = OC.reference_frames(case)
        opt = build_product(fr["key"]).optimizer
        g = np.random.RandomState(2).randn(*fr["qpos"].shape).astype(np.float32)
        res = []
        for last in (fr["last_qpos"], None):
            res += emu_vjp_host.solve_vjp(opt, g, fr["qpos"], ref_value=fr["ref_value"], fixed_qpos=fr["fixed_qpos"],
                                          last_qpos=last, projected=fr["projected"])
        got[case] = _crc(res)
    for key, (S, T, kp, X, last0, F) in _streams().items():
        seq = build_product(key)
        n, dof = seq.optimizer.opt_dof, seq.optimizer.robot.dof
        anchor = np.concatenate([last0[:, None], X[:, :-1]], axis=1).reshape(-1, n)
        g = np.random.RandomState(4).randn(S * T, n).astype(np.float32)
        res = []
        for last in (anchor, None):
            res += emu_vjp_host.solve_vjp(seq.optimizer, g, X.reshape(-1, n), keypoints=kp.reshape(-1, 21, 3), last_qpos=last,
                                          projected=None if F is None else F.reshape(S * T, -1))
        got[key] = _crc(res)
        rng = np.random.RandomState(5)
        got["seq " + key] = _crc(SH.solve_sequences_vjp(seq, kp, X, last0, np.zeros(S, np.uint8), F,
                                                        grad_robot_qpos=rng.randn(S, T, dof).astype(np.float32),
                                                        grad_last_qpos=rng.randn(S, n).astype(np.float32),
                                                        grad_filter_state=rng.randn(S, dof).astype(np.float32)))
    assert got == VJP_DIGESTS


def test_gpu_jacobian_file_passes_against_the_emulation():
    """tests/test_gpu_jacobian.py dry-run on the CPU (tests/tools/emu_gpu_jacobian.py, retarget_batch_jacobian and
    retarget_batch_vjp served by the emulation)."""
    count = 13
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_jacobian.py")], capture_output=True,
                         text=True, timeout=3000)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
