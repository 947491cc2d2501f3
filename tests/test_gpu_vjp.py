"""Backpropagation through the solve on the GPU (`dexr_solve_vjp` through Optimizer.retarget_batch_vjp and
objective.differentiable_retarget): the float64 implicit-function model of tests/vjp_cases.py, the host emulation of the same
driver, finite differences of the oracle's converged solution, a two-frame chain through last_qpos, determinism across batch
layouts, a bench-size batch and the library's argument checks.
Also dry-run on the CPU by tests/test_vjp_emulation.py (tests/tools/emu_gpu_vjp.py)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

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


def gpu_vjp(opt, gbar, qpos, fixed_qpos=None, last_qpos=None, projected=None, **target):
    """retarget_batch_vjp on device copies of numpy inputs -> (grad_targets, grad_fixed or None, grad_last or None, status)."""
    B = qpos.shape[0]
    status = torch.full((B,), -1, dtype=torch.int32, device=_dev())
    out = opt.retarget_batch_vjp(_t(gbar), _t(qpos), fixed_qpos=_t(fixed_qpos), last_qpos=_t(last_qpos),
                                 projected=_t(projected), status_out=status, **{k: _t(v) for k, v in target.items()})
    torch.cuda.synchronize()
    return tuple(None if a is None else a.cpu().numpy() for a in (*out, status))


@pytest.mark.parametrize("key", KEYS)
def test_matches_the_float64_model(key):
    """At the oracle's minimisers rounded to float32, both input forms, with and without an anchor: within V.TAU of the
    model; `projected` is not written."""
    o, opt = build_oracle(key), build_product(key).optimizer
    for with_last in (True, False):
        pts = V.solved_points(o, 6, seed=21, with_last=with_last)
        for form in ("ref_value", "keypoints"):
            proj = None if pts["flags"] is None else pts["flags"].copy()
            res = gpu_vjp(opt, pts["gbar"], pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], proj, **{form: pts[form]})
            if proj is not None:
                np.testing.assert_array_equal(proj, pts["flags"])
            ratio = V.compare(res, V.model_batch(o, pts, form), pts)
            print(key, form, "anchor" if with_last else "no anchor", "worst error / tau %.3f" % ratio)


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right", "teleop/ability_hand_right"])
def test_matches_the_host_emulation(key):
    import emu_vjp_host

    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 8, seed=23)
    for form in ("ref_value", "keypoints"):
        g = gpu_vjp(opt, pts["gbar"], pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], pts["flags"], **{form: pts[form]})
        e = emu_vjp_host.solve_vjp(opt, pts["gbar"], pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                    projected=pts["flags"], **{form: pts[form]})
        np.testing.assert_array_equal(g[3], e[3])
        worst = 0.0
        for a, b in zip(g[:3], e[:3]):
            if b is None:
                continue
            scale = np.abs(b).reshape(len(b), -1).max(1)
            d = np.abs(a - b).reshape(len(b), -1).max(1)
            assert np.all(d <= 1e-4 * scale + 1e-12), (d / scale).max()
            worst = max(worst, float((d / np.maximum(scale, 1e-30)).max()))
        print(key, form, "worst |gpu - emulation| / |emulation|_inf %.2e" % worst)


def test_differentiable_retarget_end_to_end():
    """backward() of a loss on the solved joint angles: the model at the GPU's own answers, and finite differences of the
    oracle's converged solution on well-conditioned frames with no active bound."""
    from dex_retargeting_b200.objective import differentiable_retarget
    from oracle.solvers import solve_converged

    key = "teleop/allegro_hand_right"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 8, seed=25)
    kp = _t(pts["keypoints"]).requires_grad_(True)
    last = _t(pts["last_qpos"]).requires_grad_(True)
    q = differentiable_retarget(opt, keypoints=kp, last_qpos=last)
    w = torch.from_numpy(pts["gbar"]).to(_dev())
    (q * w).sum().backward()
    torch.cuda.synchronize()
    qn = q.detach().cpu().numpy()
    model_pts = dict(pts, qpos=qn)
    m = V.model_batch(o, model_pts, "keypoints")
    res = (kp.grad.cpu().numpy(), None, last.grad.cpu().numpy(), np.zeros(8, np.int32))
    print("backward() against the model at the GPU's answers: worst error / tau %.3f" % V.compare(res, m, model_pts))
    # finite differences of the converged minimiser in three keypoint coordinates, on the frames whose free variables all lie
    # 1e-3 or more inside the bounds; the perturbed minimisers must keep the same variables at their bounds
    h, checked = 1e-4, 0
    lo32, hi32 = np.float32(o.lower), np.float32(o.upper)
    for i in range(8):
        at_bound = (qn[i] <= lo32) | (qn[i] >= hi32)
        near = ~at_bound & ((qn[i] < lo32 + 1e-3) | (qn[i] > hi32 - 1e-3))
        if m["skip"][i] or near.any():
            continue
        for (kid, c) in ((4, 0), (8, 1), (16, 2)):
            xs = []
            for s in (1.0, -1.0):
                k2 = pts["keypoints"][i].astype(np.float64)
                k2[kid, c] += s * h
                x, kkt, _ = solve_converged(o, o.ref_from_keypoints(k2), np.zeros(0), pts["last_qpos"][i], x_init=qn[i])
                assert kkt < 1e-7, kkt
                assert np.array_equal((x <= o.lower + 1e-7) | (x >= o.upper - 1e-7), at_bound)
                xs.append(x)
            fd = float(pts["gbar"][i].astype(np.float64) @ (xs[0] - xs[1]) / (2 * h))
            got = float(kp.grad[i, kid, c])
            scale = float(np.abs(m["targets"][i]).max())
            assert abs(got - fd) <= 2e-3 * scale, (i, kid, c, got, fd, scale)
        checked += 1
    assert checked >= 2
    print("finite differences of the converged solution agree on", checked, "frames")


def test_two_frame_chain_through_last_qpos():
    """Frame 2 anchored at frame 1's answer: backward() through both solves equals the chained model."""
    from dex_retargeting_b200.objective import differentiable_retarget

    key = "teleop/leap_hand_right_dexpilot"
    o, opt = build_oracle(key), build_product(key).optimizer
    pts = V.solved_points(o, 2, seed=27)
    kp = _t(pts["keypoints"])
    k1, k2 = kp[0:1].clone().requires_grad_(True), kp[1:2].clone().requires_grad_(True)
    a0 = _t(pts["last_qpos"][0:1]).requires_grad_(True)
    lp = opt._objective_spec().len_proj
    flags = torch.zeros((1, lp), dtype=torch.uint8, device=_dev())
    x1 = differentiable_retarget(opt, keypoints=k1, last_qpos=a0, projected=flags)
    f1 = flags.cpu().numpy().copy()
    x2 = differentiable_retarget(opt, keypoints=k2, last_qpos=x1, projected=flags)
    f2 = flags.cpu().numpy().copy()
    w = torch.from_numpy(pts["gbar"][1:2]).to(_dev())
    (x2 * w).sum().backward()
    torch.cuda.synchronize()
    X1, X2 = x1.detach().cpu().numpy()[0], x2.detach().cpu().numpy()[0]
    m2 = V.model_vjp(o, X2, pts["gbar"][1], None, X1, f2[0], keypoints=pts["keypoints"][1])
    m1 = V.model_vjp(o, X1, m2["last"].astype(np.float32), None, pts["last_qpos"][0], f1[0], keypoints=pts["keypoints"][0])
    for got, want in ((k2.grad[0], m2["targets"]), (k1.grad[0], m1["targets"]), (a0.grad[0], m1["last"])):
        got = got.cpu().numpy().astype(np.float64)
        assert np.abs(got - want).max() <= V.TAU * np.abs(want).max(), (np.abs(got - want).max(), np.abs(want).max())


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_frame_outputs_do_not_depend_on_the_batch_layout(key):
    """Bit-identical per frame whatever its position in the batch, the batch size and the pointer offset (16 and 32 lanes)."""
    o, opt = build_oracle(key), build_product(key).optimizer
    import objective_cases as OC

    B = 300
    pts = OC.oracle_points(o, B, seed=29)
    gbar = np.random.RandomState(30).randn(B, opt.opt_dof).astype(np.float32)
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
        out = opt.retarget_batch_vjp(sub(gbar), sub(pts["qpos"]), fixed_qpos=sub(pts["fixed_qpos"]), last_qpos=sub(pts["last_qpos"]),
                                     keypoints=sub(pts["keypoints"]), projected=sub(flags), status_out=st)
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in out if t is not None] + [st.cpu().numpy()]

    full = run(np.arange(B))
    perm = np.random.RandomState(1).permutation(B)
    for idx, pad in ((perm, 0), (np.arange(7, 40), 1), (np.arange(B - 1, B), 3), (np.arange(5, 6), 0)):
        for a, b in zip(run(idx, pad), full):
            np.testing.assert_array_equal(a, b[idx])


def test_full_bench_batch():
    """The bench's 65 536 Allegro frames (tools/workloads.py) solved, then backpropagated: every output finite."""
    sys.path.insert(0, str(ROOT / "tools"))
    import workloads as W
    from dex_retargeting_b200 import _native as N

    seq = W.build(W.METRIC_KEY)
    opt = seq.optimizer
    kp, x0, _, _ = W.frames(seq, 65536, W.METRIC_SEED)
    res = gpu_solve(opt, x0=x0, keypoints=kp)
    gbar = np.random.RandomState(5).randn(*x0.shape).astype(np.float32)
    g_kp, _, g_last, status = gpu_vjp(opt, gbar, res["q"], last_qpos=x0, keypoints=kp)
    counts = {"ok": int((status == 0).sum()), "not_pd": int((status & N.STATUS_NOT_PD != 0).sum()),
              "nonfinite": int((status & N.STATUS_NONFINITE != 0).sum())}
    print("65 536 frames, status counts", counts)
    assert counts["nonfinite"] == 0 and counts["ok"] + counts["not_pd"] == 65536
    assert np.isfinite(g_kp).all() and np.isfinite(g_last).all()


def test_argument_errors_are_rejected_with_a_message(tmp_path):
    """Every rejected argument set of dexr_solve_vjp, on a robot handle (the robot with fixed joints is synthetic)."""
    import structure_cases as SC
    from dex_retargeting_b200 import _native as N

    dev = _dev()
    seq, _ = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    opt = seq.optimizer
    eng, lib = opt.engine(), N.load()
    x = torch.zeros((2, opt.opt_dof), device=dev)
    ref = torch.zeros((2, opt.num_residuals, 3), device=dev)
    kp = torch.zeros((2, 21, 3), device=dev)
    fixed = torch.zeros((2, len(opt.idx_pin2fixed)), device=dev)

    def call(B=2, robot=eng.handle, preprocess=0, **ptrs):
        io = N.DexrVjp()
        for k, v in ptrs.items():
            setattr(io, k, v.data_ptr())
        p = opt.params()
        p.preprocess = preprocess
        return lib.dexr_solve_vjp(robot, C.byref(p), C.byref(io), B, None), lib.dexr_last_error().decode()

    ok = dict(qpos=x, grad_qpos=x, ref_value=ref, fixed_qpos=fixed)
    assert call(robot=None, **ok)[1].endswith("null argument")
    for kw, msg in [(dict(ok, qpos=None), "qpos is required"), (dict(ok, grad_qpos=None), "grad_qpos is required"),
                    (dict(ok, ref_value=None), "exactly one of keypoints / ref_value"),
                    (dict(ok, keypoints=kp), "exactly one of keypoints / ref_value"),
                    (dict(ok, preprocess=1), "pre-processing is not differentiated"),
                    (dict(ok, fixed_qpos=None), "fixed joints but fixed_qpos is NULL"),
                    (dict(ok, grad_keypoints=kp), "grad_keypoints needs the keypoints form"),
                    (dict(ok, grad_last_qpos=x), "grad_last_qpos needs last_qpos"),
                    (dict(ok, B=-1), "num_frames < 0")]:
        rc, err = call(**{k: v for k, v in kw.items() if v is not None or k in ("B", "preprocess")})
        assert rc == -1 and msg in err, (kw.keys(), rc, err)
    assert call(B=0, **ok)[0] == 0
