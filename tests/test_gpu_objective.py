"""Objective evaluation on the GPU (`dexr_eval_objective` through Optimizer.objective_batch, get_objective_function and
objective.retargeting_cost): the reference closure's values, the host emulation of the same driver, the solver's reported
cost and flags, determinism across batch layouts, autograd, argument checks, a full bench-size batch.
Also dry-run on the CPU by tests/test_objective_emulation.py (tests/tools/emu_gpu_objective.py)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import objective_cases as OC
from helpers import build_oracle, build_product, synth_problems
from test_gpu_parity import _dev, gpu_solve

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent


def gpu_eval(opt, qpos, ref_value=None, fixed_qpos=None, last_qpos=None, keypoints=None, projected=None, want_grad=True,
             raw_hand=None):
    """objective_batch on device copies of numpy inputs -> (loss, cost, grad or None); `projected` is updated in place."""
    dev = _dev()

    def t(a):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    proj = t(projected)
    loss, cost, grad = opt.objective_batch(t(qpos), t(ref_value), t(fixed_qpos), t(last_qpos), keypoints=t(keypoints),
                                           projected=proj, want_grad=want_grad, raw_hand=raw_hand)
    torch.cuda.synchronize()
    if projected is not None:
        projected[...] = proj.cpu().numpy()
    return loss.cpu().numpy(), cost.cpu().numpy(), None if grad is None else grad.cpu().numpy()


@pytest.mark.parametrize("case", OC.REF_CASES)
def test_reference_closure_values_through_objective_batch(case):
    fr = OC.reference_frames(case)
    opt = build_product(fr["key"]).optimizer
    proj = OC.initial_flags(opt, len(fr["qpos"]))
    loss, cost, grad = gpu_eval(opt, fr["qpos"], fr["ref_value"], fr["fixed_qpos"], fr["last_qpos"], projected=proj)
    print(case, "worst relative loss / grad error", OC.reference_errors(loss, grad, fr["values"], fr["grads"]))
    if proj is not None:
        np.testing.assert_array_equal(proj, fr["projected"])


@pytest.mark.parametrize("case", OC.REF_CASES)
def test_reference_closure_values_through_get_objective_function(case):
    """The reference's calling convention: objective(x, grad) -> L(x), grad filled when it has a size; DexPilot's flags are
    set when the closure is made."""
    fr = OC.reference_frames(case)
    opt = build_product(fr["key"]).optimizer
    P = 3
    for i in range(len(fr["qpos"]) // P):
        if opt.retargeting_type == "DEXPILOT":
            opt.projected = np.zeros_like(opt.projected)
        f0 = i * P
        fixed = fr["fixed_qpos"][f0] if fr["fixed_qpos"] is not None else np.zeros(0, np.float32)
        fn = opt.get_objective_function(fr["ref_value"][f0], fixed, fr["last_qpos"][f0].astype(np.float64))
        if fr["projected"] is not None:
            np.testing.assert_array_equal(opt.projected, fr["projected"][f0].astype(bool))
        vals, grads = [], []
        for p in range(P):
            g = np.zeros(opt.opt_dof)
            vals.append(fn(fr["qpos"][f0 + p].astype(np.float64), g))
            grads.append(g)
            empty = np.zeros(0)
            assert fn(fr["qpos"][f0 + p].astype(np.float64), empty) == vals[-1] and empty.size == 0
        OC.reference_errors(np.array(vals), np.array(grads), fr["values"][f0:f0 + P], fr["grads"][f0:f0 + P])
    with pytest.raises(ValueError, match="non_target_qpos"):
        opt.get_objective_function(fr["ref_value"][0], np.zeros(len(opt.idx_pin2fixed) + 1), fr["last_qpos"][0])


@pytest.mark.parametrize("key", OC.SOLVER_CASES)
def test_matches_the_host_emulation(key):
    """The kernel against the host emulation of the same driver, same inputs, within the reference-value tolerances."""
    import emu_eval_host

    opt, o = build_product(key).optimizer, build_oracle(key)
    for form in ("ref_value", "keypoints"):
        pts = OC.oracle_points(o, 40, seed=11)
        inputs = {form: pts[form]}
        pg, pe = OC.initial_flags(opt, 40), OC.initial_flags(opt, 40)
        lg, cg, gg = gpu_eval(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"], projected=pg, **inputs)
        le, ce, ge = emu_eval_host.eval_objective(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                                  projected=pe, **inputs)
        for a, b in ((lg, le), (cg, ce)):
            np.testing.assert_allclose(a, b, rtol=OC.REF_LOSS_RTOL, atol=OC.REF_LOSS_ATOL)
        dg = np.abs(gg - ge).max(1)
        assert np.all(dg <= OC.REF_GRAD_RTOL * np.abs(ge).max(1) + OC.REF_GRAD_ATOL)
        print(key, form, "worst |gpu - emulation|: loss rel %.2e, grad rel %.2e" % (
            (np.abs(lg - le) / np.abs(le)).max(), (dg / np.abs(ge).max(1)).max()))
        if pg is not None:
            np.testing.assert_array_equal(pg, pe)


@pytest.mark.parametrize("key", OC.SOLVER_CASES)
def test_agrees_with_retarget_batch_at_its_answer(key):
    o, opt = build_oracle(key), build_product(key).optimizer
    refs, fixed, x0, _ = synth_problems(o, 64, np.random.RandomState(8), init_noise=0.05, target_noise=0.01)
    fixed = fixed if fixed.size else None
    res = gpu_solve(opt, refs, fixed, x0, want_proj=True)
    proj = OC.initial_flags(opt, 64)
    _, cost, grad = gpu_eval(opt, res["q"], refs, fixed, x0, projected=proj)
    x_start = np.clip(x0, np.float32(o.lower), np.float32(o.upper))
    _, cost0, _ = gpu_eval(opt, x_start, refs, fixed, x0, projected=OC.initial_flags(opt, 64), want_grad=False)
    drift, pgrad = OC.check_after_solve(o, res["q"], res["status"], res["cost"], res.get("projected"), cost0, cost, grad, proj)
    print(key, "worst cost drift %.1f ulp, worst projected gradient %.2e" % (drift, pgrad))


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right"])
def test_frame_outputs_do_not_depend_on_the_batch_layout(key):
    """Bit-identical per frame whatever its position in the batch, the batch size and the pointer offset (16 and 32 lanes)."""
    opt, o = build_product(key).optimizer, build_oracle(key)
    B = 300
    pts = OC.oracle_points(o, B, seed=13)

    def run(idx, pad=0):
        """Frames `idx`, every input placed `pad` rows into a larger buffer (pad > 0: the views start off their allocation)."""
        def sub(a):
            if a is None:
                return None
            big = np.zeros((len(idx) + pad,) + a.shape[1:], a.dtype)
            big[pad:] = a[idx]
            return torch.from_numpy(big).to(_dev())[pad:]
        proj = OC.initial_flags(opt, len(idx) + pad)
        P = None if proj is None else torch.from_numpy(proj).to(_dev())[pad:]
        out = opt.objective_batch(sub(pts["qpos"]), None, sub(pts["fixed_qpos"]), sub(pts["last_qpos"]),
                                  keypoints=sub(pts["keypoints"]), projected=P)
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in out] + ([] if P is None else [P.cpu().numpy()])

    full = run(np.arange(B))
    perm = np.random.RandomState(1).permutation(B)
    for idx, pad in ((perm, 0), (np.arange(7, 40), 1), (np.arange(B - 1, B), 3), (np.arange(5, 6), 0)):
        got = run(idx, pad)
        for a, b in zip(got, full):
            np.testing.assert_array_equal(a, b[idx])


def test_retargeting_cost_backpropagates_the_evaluated_gradient():
    from dex_retargeting_b200.objective import retargeting_cost

    key = "teleop/ability_hand_right"
    opt, o = build_product(key).optimizer, build_oracle(key)
    dev = _dev()
    pts = OC.oracle_points(o, 24, seed=17)
    t = {k: None if v is None else torch.from_numpy(v).to(dev) for k, v in pts.items()}
    x = t["qpos"].clone().requires_grad_(True)
    cost = retargeting_cost(opt, x, keypoints=t["keypoints"], fixed_qpos=t["fixed_qpos"], last_qpos=t["last_qpos"])
    w = torch.linspace(-1.0, 2.0, 24, device=dev)
    (cost * w).sum().backward()
    _, cost_b, grad_b = opt.objective_batch(t["qpos"], None, t["fixed_qpos"], t["last_qpos"], keypoints=t["keypoints"])
    torch.cuda.synchronize()
    assert torch.equal(cost.detach(), cost_b)
    assert torch.equal(x.grad, w[:, None] * grad_b)
    for name in ("keypoints", "last_qpos"):
        kw = dict(keypoints=t["keypoints"], last_qpos=t["last_qpos"])
        kw[name] = kw[name].clone().requires_grad_(True)
        with pytest.raises(ValueError, match=f"{name} requires grad"):
            retargeting_cost(opt, x, **kw)


def test_argument_errors_are_rejected_with_a_message(tmp_path):
    """Every rejected argument set of dexr_eval_objective, on a robot handle (the robot with fixed joints is synthetic)."""
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
        io = N.DexrEval()
        for k, v in ptrs.items():
            setattr(io, k, v.data_ptr())
        p = opt.params()
        p.preprocess = preprocess
        return lib.dexr_eval_objective(robot, C.byref(p), C.byref(io), B, None), lib.dexr_last_error().decode()

    assert call(robot=None, qpos=x, ref_value=ref, fixed_qpos=fixed)[1].endswith("null argument")
    for kw, msg in [(dict(ref_value=ref, fixed_qpos=fixed), "qpos is required"),
                    (dict(qpos=x, fixed_qpos=fixed), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, keypoints=kp, fixed_qpos=fixed), "exactly one of keypoints / ref_value"),
                    (dict(qpos=x, ref_value=ref, fixed_qpos=fixed, preprocess=1), "preprocess needs raw keypoints"),
                    (dict(qpos=x, ref_value=ref), "fixed joints but fixed_qpos is NULL"),
                    (dict(qpos=x, ref_value=ref, fixed_qpos=fixed, B=-1), "num_frames < 0")]:
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
    assert call(B=0, qpos=x, ref_value=ref, fixed_qpos=fixed)[0] == 0


def test_full_bench_batch():
    """The bench's 65 536 Allegro frames (tools/workloads.py) at their warm starts, anchored 0.05 rad away: all finite,
    equal to the oracle on a seeded sample of 256 frames."""
    sys.path.insert(0, str(ROOT / "tools"))
    import workloads as W

    seq = W.build(W.METRIC_KEY)
    opt, o = seq.optimizer, build_oracle(W.METRIC_KEY)
    kp, x, _, _ = W.frames(seq, 65536, W.METRIC_SEED)
    last = (x + 0.05 * np.random.RandomState(2).randn(*x.shape)).astype(np.float32)
    loss, cost, grad = gpu_eval(opt, x, keypoints=kp, last_qpos=last)
    assert np.isfinite(loss).all() and np.isfinite(cost).all() and np.isfinite(grad).all()
    idx = np.random.RandomState(3).choice(65536, 256, replace=False)
    pts = dict(qpos=x[idx], last_qpos=last[idx], fixed_qpos=None, ref_value=np.stack([o.ref_from_keypoints(k) for k in kp[idx]]))
    L, Cst, G, _ = OC.oracle_expect(o, pts)
    print("full batch, oracle sample: worst loss / cost / grad error", OC.oracle_errors(loss[idx], cost[idx], grad[idx], L, Cst, G))
