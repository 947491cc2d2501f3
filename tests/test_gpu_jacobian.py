"""Per-frame Jacobians of the solve on the GPU (`dexr_solve_jacobian` through Optimizer.retarget_batch_jacobian): the float64
model of tests/jacobian_cases.py, the host emulation of the same driver, the loop of one `retarget_batch_vjp` launch per unit
cotangent, finite differences of the oracle's converged solution, determinism across batch layouts, a bench-size batch and
the library's argument checks.
Also dry-run on the CPU by tests/test_jacobian_emulation.py (tests/tools/emu_gpu_jacobian.py)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import jacobian_cases as JC
import vjp_cases as V
from helpers import build_oracle, build_product
from test_gpu_parity import _dev, gpu_solve

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
KEYS = ["teleop/allegro_hand_right", "teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right",
        "teleop/ability_hand_right", "teleop/schunk_svh_hand_right", "offline/inspire_hand_right"]


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def gpu_jacobian(opt, qpos, fixed_qpos=None, last_qpos=None, projected=None, **target):
    """retarget_batch_jacobian on device copies of numpy inputs -> (jac_targets, jac_fixed or None, jac_last or None, status)."""
    B = qpos.shape[0]
    status = torch.full((B,), -1, dtype=torch.int32, device=_dev())
    out = opt.retarget_batch_jacobian(_t(qpos), fixed_qpos=_t(fixed_qpos), last_qpos=_t(last_qpos), projected=_t(projected),
                                      status_out=status, **{k: _t(v) for k, v in target.items()})
    torch.cuda.synchronize()
    return tuple(None if a is None else a.cpu().numpy() for a in (*out, status))


def vjp_loop(opt, qpos, fixed_qpos=None, last_qpos=None, projected=None, **target):
    """The loop of n retarget_batch_vjp launches with grad_qpos = e_i, stacked as Jacobian rows (+ the statuses [n,B])."""
    B, n = qpos.shape
    rows, sts = [], []
    for i in range(n):
        e = np.zeros((B, n), np.float32)
        e[:, i] = 1.0
        st = torch.full((B,), -1, dtype=torch.int32, device=_dev())
        out = opt.retarget_batch_vjp(_t(e), _t(qpos), fixed_qpos=_t(fixed_qpos), last_qpos=_t(last_qpos),
                                     projected=_t(projected), status_out=st, **{k: _t(v) for k, v in target.items()})
        torch.cuda.synchronize()
        rows.append([None if a is None else a.cpu().numpy() for a in out])
        sts.append(st.cpu().numpy())
    return (*[None if rows[0][k] is None else np.stack([r[k] for r in rows], axis=1) for k in range(3)], np.stack(sts))


def _close(a, b, rel):
    """Per frame and block: |a - b|_inf <= rel |b|_inf; returns the worst ratio |a - b|_inf / |b|_inf."""
    worst = 0.0
    for x, y in zip(a, b):
        if y is None:
            continue
        scale = np.abs(y).reshape(len(y), -1).max(1)
        d = np.abs(x - y).reshape(len(y), -1).max(1)
        assert np.all(d <= rel * scale + 1e-12), (d / np.maximum(scale, 1e-30)).max()
        worst = max(worst, float((d / np.maximum(scale, 1e-30)).max()))
    return worst


@pytest.mark.parametrize("key", KEYS)
def test_matches_the_float64_model(key):
    """At the oracle's minimisers rounded to float32, both input forms, with and without an anchor: within the VJP model's
    tau of the model; `projected` is not written."""
    o, opt = build_oracle(key), build_product(key).optimizer
    for with_last in (True, False):
        pts = V.solved_points(o, 4, seed=21, with_last=with_last)
        for form in ("ref_value", "keypoints"):
            proj = None if pts["flags"] is None else pts["flags"].copy()
            res = gpu_jacobian(opt, pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], proj, **{form: pts[form]})
            if proj is not None:
                np.testing.assert_array_equal(proj, pts["flags"])
            ratio = JC.compare(res, JC.model_batch(o, pts, form))
            print(key, form, "anchor" if with_last else "no anchor", "worst error / tau %.3f" % ratio)


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right", "teleop/ability_hand_right"])
def test_matches_the_host_emulation(key):
    import emu_jacobian_host

    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 6, seed=23)
    for form in ("ref_value", "keypoints"):
        g = gpu_jacobian(opt, pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], pts["flags"], **{form: pts[form]})
        e = emu_jacobian_host.solve_jacobian(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                             projected=pts["flags"], **{form: pts[form]})
        np.testing.assert_array_equal(g[3], e[3])
        print(key, form, "worst |gpu - emulation| / |emulation|_inf %.2e" % _close(g[:3], e[:3], 1e-4))


def test_rows_match_the_vjp_loop():
    """Every row of one Jacobian launch against the n-launch loop of retarget_batch_vjp with grad_qpos = e_i, with active
    bounds and both input forms; the statuses are equal."""
    key = "teleop/leap_hand_right_dexpilot"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 6, seed=49)
    pts["last_qpos"][:2] = np.where(np.random.RandomState(50).rand(2, o.opt_dof) < 0.5, o.joint_limits[:, 0] - 0.3,
                                    o.joint_limits[:, 1] + 0.3).astype(np.float32)
    for form in ("ref_value", "keypoints"):
        args = (pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], pts["flags"])
        j = gpu_jacobian(opt, *args, **{form: pts[form]})
        loop = vjp_loop(opt, *args, **{form: pts[form]})
        for st in loop[3]:
            np.testing.assert_array_equal(st, j[3])
        print(form, "worst |jacobian row - vjp| / |vjp|_inf %.2e" % _close(j[:3], loop[:3], 1e-6))


def test_jacobian_predicts_the_perturbed_solution():
    """J delta against central differences of the oracle's converged minimiser in three keypoint coordinates, on
    well-conditioned frames whose free variables lie 1e-3 or more inside the bounds and keep the same active set."""
    from oracle.solvers import solve_converged

    key = "teleop/allegro_hand_right"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 6, seed=25)
    jac, _, j_last, status = gpu_jacobian(opt, pts["qpos"], last_qpos=pts["last_qpos"], keypoints=pts["keypoints"])
    m = JC.model_batch(o, pts, "keypoints")
    JC.compare((jac, None, j_last, status), m)
    h, checked = 1e-4, 0
    lo32, hi32 = np.float32(o.lower), np.float32(o.upper)
    for i in range(6):
        qn = pts["qpos"][i]
        at_bound = (qn <= lo32) | (qn >= hi32)
        near = ~at_bound & ((qn < lo32 + 1e-3) | (qn > hi32 - 1e-3))
        if m["skip"][i] or near.any() or status[i] != 0:
            continue
        for (kid, c) in ((4, 0), (8, 1), (16, 2)):
            xs = []
            for s in (1.0, -1.0):
                k2 = pts["keypoints"][i].astype(np.float64)
                k2[kid, c] += s * h
                x, kkt, _ = solve_converged(o, o.ref_from_keypoints(k2), np.zeros(0), pts["last_qpos"][i], x_init=qn)
                assert kkt < 1e-7, kkt
                assert np.array_equal((x <= o.lower + 1e-7) | (x >= o.upper - 1e-7), at_bound)
                xs.append(x)
            fd = (xs[0] - xs[1]) / (2 * h)
            got = jac[i, :, kid, c].astype(np.float64)
            scale = float(np.abs(m["targets"][i]).max())
            assert np.abs(got - fd).max() <= 2e-3 * scale, (i, kid, c, got, fd, scale)
        checked += 1
    assert checked >= 2
    print("J delta agrees with finite differences of the converged solution on", checked, "frames")


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_frame_outputs_do_not_depend_on_the_batch_layout(key):
    """Bit-identical per frame whatever its position in the batch, the batch size and the pointer offset (16 and 32 lanes)."""
    import objective_cases as OC

    o, opt = build_oracle(key), build_product(key).optimizer
    B = 120
    pts = OC.oracle_points(o, B, seed=29)
    res = gpu_solve(opt, fixed=pts["fixed_qpos"], x0=pts["last_qpos"], keypoints=pts["keypoints"], want_proj=True)
    pts["qpos"], flags = res["q"], res.get("projected")

    def run(idx, pad=0):
        def sub(a):
            if a is None:
                return None
            big = np.zeros((len(idx) + pad,) + a.shape[1:], a.dtype)
            big[pad:] = a[idx]
            return torch.from_numpy(big).to(_dev())[pad:]
        st = torch.empty((len(idx),), dtype=torch.int32, device=_dev())
        out = opt.retarget_batch_jacobian(sub(pts["qpos"]), fixed_qpos=sub(pts["fixed_qpos"]), last_qpos=sub(pts["last_qpos"]),
                                          keypoints=sub(pts["keypoints"]), projected=sub(flags), status_out=st)
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in out if t is not None] + [st.cpu().numpy()]

    full = run(np.arange(B))
    perm = np.random.RandomState(1).permutation(B)
    for idx, pad in ((perm, 0), (np.arange(7, 40), 1), (np.arange(B - 1, B), 3), (np.arange(5, 6), 0)):
        for a, b in zip(run(idx, pad), full):
            np.testing.assert_array_equal(a, b[idx])


def test_full_bench_batch():
    """The bench's 65 536 Allegro frames (tools/workloads.py) solved, then differentiated: every output finite, and the same
    statuses as one VJP launch on the same frames."""
    sys.path.insert(0, str(ROOT / "tools"))
    import workloads as W
    from dex_retargeting_b200 import _native as N

    seq = W.build(W.METRIC_KEY)
    opt = seq.optimizer
    kp, x0, _, _ = W.frames(seq, 65536, W.METRIC_SEED)
    res = gpu_solve(opt, x0=x0, keypoints=kp)
    j_kp, _, j_last, status = gpu_jacobian(opt, res["q"], last_qpos=x0, keypoints=kp)
    vst = torch.full((65536,), -1, dtype=torch.int32, device=_dev())
    opt.retarget_batch_vjp(_t(np.ones_like(x0)), _t(res["q"]), last_qpos=_t(x0), keypoints=_t(kp), status_out=vst)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(status, vst.cpu().numpy())
    counts = {"ok": int((status == 0).sum()), "not_pd": int((status & N.STATUS_NOT_PD != 0).sum()),
              "nonfinite": int((status & N.STATUS_NONFINITE != 0).sum())}
    print("65 536 frames, status counts", counts)
    assert counts["nonfinite"] == 0 and counts["ok"] + counts["not_pd"] == 65536
    assert np.isfinite(j_kp).all() and np.isfinite(j_last).all()


def test_argument_errors_are_rejected_with_a_message(tmp_path):
    """Every rejected argument set of dexr_solve_jacobian, on a robot handle (the robot with fixed joints is synthetic)."""
    import structure_cases as SC
    from dex_retargeting_b200 import _native as N

    dev = _dev()
    seq, _ = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    opt = seq.optimizer
    eng, lib = opt.engine(), N.load()
    n = opt.opt_dof
    x = torch.zeros((2, n), device=dev)
    ref = torch.zeros((2, opt.num_residuals, 3), device=dev)
    kp = torch.zeros((2, 21, 3), device=dev)
    fixed = torch.zeros((2, len(opt.idx_pin2fixed)), device=dev)
    jac = torch.zeros((2, n, 21, 3), device=dev)

    def call(B=2, robot=eng.handle, preprocess=0, **ptrs):
        io = N.DexrJacobian()
        for k, v in ptrs.items():
            setattr(io, k, v.data_ptr())
        p = opt.params()
        p.preprocess = preprocess
        return lib.dexr_solve_jacobian(robot, C.byref(p), C.byref(io), B, None), lib.dexr_last_error().decode()

    ok = dict(qpos=x, ref_value=ref, fixed_qpos=fixed)
    assert call(robot=None, **ok)[1].endswith("null argument")
    for kw, msg in [(dict(ok, qpos=None), "qpos is required"),
                    (dict(ok, ref_value=None), "exactly one of keypoints / ref_value"),
                    (dict(ok, keypoints=kp), "exactly one of keypoints / ref_value"),
                    (dict(ok, preprocess=1), "pre-processing is not differentiated"),
                    (dict(ok, fixed_qpos=None), "fixed joints but fixed_qpos is NULL"),
                    (dict(ok, jac_keypoints=jac), "jac_keypoints needs the keypoints form"),
                    (dict(ok, jac_last_qpos=jac), "jac_last_qpos needs last_qpos"),
                    (dict(ok, B=-1), "num_frames < 0")]:
        rc, err = call(**{k: v for k, v in kw.items() if v is not None or k in ("B", "preprocess")})
        assert rc == -1 and msg in err, (kw.keys(), rc, err)
    assert call(B=0, **ok)[0] == 0
