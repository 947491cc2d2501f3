"""The evaluation, backpropagation, Jacobian and smoothing kernels on the GPU on the synthetic robots of
tests/structure_cases.py: fixed joints (grad_fixed_qpos / jac_fixed_qpos, which no packaged configuration has), mimic
groups of four with negative multipliers and sources after their followers, prismatic joints, 1 to 31 DoF, n_res = 16,
four links on one joint, block width 8 and arrow tables (run on the dense Solver<G, 0>), DexPilot on two and three fingers.
Each entry point against the float64 models the host emulation is held to (tests/objective_cases.py, vjp_cases.py,
jacobian_cases.py, seq_vjp_cases.py, smooth_cases.py), at their seeds, sizes and tolerances, plus the GPU against the host
emulation of the same drivers.  Every case must keep at least half its frames after the models' skip rules, a fixed-joint
case a fixed-joint block that is not all zero, a prismatic case a prismatic variable free in a kept frame.
Also dry-run on the CPU by tests/test_structure_derivatives_emulation.py (tests/tools/emu_gpu_structure_derivatives.py)."""
import numpy as np
import pytest

import jacobian_cases as JC
import objective_cases as OC
import seq_vjp_cases as SV
import smooth_cases as SMC
import structure_cases as SC
import test_gpu_smooth as GS
import vjp_cases as V
from test_gpu_jacobian import _close, gpu_jacobian, vjp_loop
from test_gpu_objective import gpu_eval
from test_gpu_packed_streams import _assert_same, _state_copy, _state_np
from test_gpu_parity import _dev
from test_gpu_vjp import gpu_vjp
from test_packed_streams_emulation import _cotangents, _inputs
from test_seq_vjp_emulation import _problem

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ALL = [c.id for c in SC.CASES]
NO_FILTER = {"low_pass_alpha": -1.0}
SEQ_CASES = ["mimic_dense16", "mimic_dense32", "fixed_dense16", "fixed_dense32", "mimic_fixed_dense16", "mimic_fixed_dense32",
             "prismatic_block4", "prismatic_arrow", "dof1_vector", "dof31_vector", "dexpilot_3fingers"]
SEQ_SIZE = (3, 3)  # streams x frames: S odd, so that one 16-lane warp holds a stream and an idle group
PACKED_CASES = ["fixed_dense16", "mimic_fixed_dense32", "prismatic_arrow", "dof1_vector", "dof31_vector", "dexpilot_2fingers"]
RAGGED = [3, 0, 1, 2, 0, 4, 1]  # 16-lane warps pair 3 with 0, 1 with 2, 0 with 4, and 1 with an idle group
SMOOTH_CASES = ["fixed_dense16", "fixed_dense32", "mimic_dense16", "mimic_dense32", "prismatic_block4", "prismatic_arrow",
                "dof1_vector", "dof31_vector", "bw8_888_vector", "links_dense16_max_position", "dexpilot_3fingers"]
# clips of the smoothing check (lengths uniform over [lo, hi]), how many the float64 model polishes, and the length of the
# dropped-frame clip
SMOOTH_CLIPS = (8, 5, 20)
SMOOTH_CHECKED = 3
# clips of SMOOTH_CLIPS that end at max_iters, as many on the H100 as in the host emulation: there the 4-joint mimic groups
# and the 9-joint trunk leave valleys where F changes by 1e-4 relative over 0.1 rad, and the clip returns its last accepted
# iterate (as the Shadow hand without an anchor does, DESIGN.md 3.12); every other case converges on every clip
SMOOTH_MAXITER = {"mimic_dense16": 2, "dof31_vector": 1}
DROP_LENGTH = 20
DIFF_CASES = ["fixed_dense16", "mimic_fixed_dense32"]


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _build(cid, tmp_path, override=None):
    seq, o = SC.build(SC.BY_ID[cid], tmp_path, override)
    return seq, seq.optimizer, o


def _prismatic_vars(cid, o):
    names = set(SC.BY_ID[cid].opts.get("prismatic", ()))
    return [i for i, n in enumerate(o.target_joint_names) if n in names]


def _not_vacuous(cid, o, keep, qpos, fixed_block):
    """At least half the frames kept; a fixed-joint block that is not all zero on the kept frames; a prismatic variable
    strictly inside its bounds in a kept frame."""
    keep = np.asarray(keep, bool)
    assert 2 * keep.sum() >= keep.size, (cid, "kept frames", int(keep.sum()), keep.size)
    if len(o.idx_pin2fixed):
        assert np.abs(np.asarray(fixed_block)[keep]).max() > 0, (cid, "fixed-joint block all zero")
    pv = _prismatic_vars(cid, o)
    if pv:
        q = np.asarray(qpos)[keep][:, pv]
        lo, hi = np.float32(o.lower)[pv], np.float32(o.upper)[pv]
        assert ((q > lo) & (q < hi)).any(), (cid, "no free prismatic variable")


# ---- dexr_eval_objective ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cid", ALL)
def test_objective_matches_the_oracle(cid, tmp_path):
    """Loss, cost and gradient against the float64 oracle, both forms, with and without an anchor (the seeds and sizes of
    test_objective_emulation.test_structure_cases_match_oracle)."""
    seq, opt, o = _build(cid, tmp_path)
    worst = np.zeros(3)
    for with_last in (True, False):
        pts = OC.oracle_points(o, 6, 5, with_last=with_last)
        L, Cst, G, P = OC.oracle_expect(o, pts)
        for form in ("ref_value", "keypoints"):
            proj = OC.initial_flags(opt, 6)
            loss, cost, grad = gpu_eval(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                        projected=proj, **{form: pts[form]})
            worst = np.maximum(worst, OC.oracle_errors(loss, cost, grad, L, Cst, G))
            if not with_last:
                np.testing.assert_array_equal(loss, cost)
            if proj is not None:
                np.testing.assert_array_equal(proj, P)
    print(cid, "worst loss / cost / grad error", worst)


@pytest.mark.parametrize("cid", ALL)
def test_objective_matches_the_host_emulation(cid, tmp_path):
    import emu_eval_host

    seq, opt, o = _build(cid, tmp_path)
    for form in ("ref_value", "keypoints"):
        pts = OC.oracle_points(o, 6, 5)
        pg, pe = OC.initial_flags(opt, 6), OC.initial_flags(opt, 6)
        lg, cg, gg = gpu_eval(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"], projected=pg,
                              **{form: pts[form]})
        le, ce, ge = emu_eval_host.eval_objective(opt, pts["qpos"], fixed_qpos=pts["fixed_qpos"], last_qpos=pts["last_qpos"],
                                                  projected=pe, **{form: pts[form]})
        for a, b in ((lg, le), (cg, ce)):
            np.testing.assert_allclose(a, b, rtol=OC.REF_LOSS_RTOL, atol=OC.REF_LOSS_ATOL)
        dg = np.abs(gg - ge).max(1)
        assert np.all(dg <= OC.REF_GRAD_RTOL * np.abs(ge).max(1) + OC.REF_GRAD_ATOL)
        if pg is not None:
            np.testing.assert_array_equal(pg, pe)
        print(cid, form, "worst |gpu - emulation|: grad rel %.2e" % (dg / np.maximum(np.abs(ge).max(1), 1e-30)).max())


# ---- dexr_solve_vjp -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cid", ALL)
def test_vjp_matches_the_float64_model(cid, tmp_path):
    """Both input forms with and without an anchor at V.TAU of the model, the NOT_PD status of the model, `projected` read
    only (the seeds and sizes of test_vjp_emulation.test_structure_cases_match_model)."""
    seq, opt, o = _build(cid, tmp_path)
    worst, seen = 0.0, []
    for with_last in (True, False):
        pts = V.solved_points(o, 3, 7, with_last=with_last)
        for form in ("ref_value", "keypoints"):
            proj = None if pts["flags"] is None else pts["flags"].copy()
            res = gpu_vjp(opt, pts["gbar"], pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], proj, **{form: pts[form]})
            assert (res[1] is None) == (len(o.idx_pin2fixed) == 0)
            if proj is not None:
                np.testing.assert_array_equal(proj, pts["flags"])
            m = V.model_batch(o, pts, form)
            worst = max(worst, V.compare(res, m, pts))
            seen.append((~m["skip"], pts["qpos"], m["fixed"]))
    _not_vacuous(cid, o, *map(np.concatenate, zip(*seen)))
    print(cid, "worst error / tau %.3f" % worst)


@pytest.mark.parametrize("cid", ALL)
def test_vjp_matches_the_host_emulation(cid, tmp_path):
    """Equal status words and 1e-4 relative per frame and block, on the frames the model keeps: on a frame whose free
    Hessian is nearly singular (V.SINGULAR; without an anchor on bw8_88_vector and dof3_position) the last bits of the
    Hessian decide NOT_PD and move H_ff^-1 by far more than 1e-4, on the H100 as between any two fp32 orderings."""
    import emu_vjp_host

    seq, opt, o = _build(cid, tmp_path)
    worst = 0.0
    for with_last in (True, False):
        pts = V.solved_points(o, 3, 7, with_last=with_last)
        for form in ("ref_value", "keypoints"):
            g = gpu_vjp(opt, pts["gbar"], pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], pts["flags"], **{form: pts[form]})
            e = emu_vjp_host.solve_vjp(opt, pts["gbar"], pts["qpos"], fixed_qpos=pts["fixed_qpos"],
                                        last_qpos=pts["last_qpos"], projected=pts["flags"], **{form: pts[form]})
            keep = ~V.model_batch(o, pts, form)["skip"]
            np.testing.assert_array_equal(g[3][keep], e[3][keep])
            if keep.any():
                worst = max(worst, _close([None if a is None else a[keep] for a in g[:3]],
                                          [None if b is None else b[keep] for b in e[:3]], 1e-4))
    print(cid, "worst |gpu - emulation| / |emulation|_inf %.2e" % worst)


# ---- dexr_solve_jacobian ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cid", ALL)
def test_jacobian_matches_the_model_and_the_vjp_rows(cid, tmp_path):
    """Every block (jac_fixed_qpos wherever n_fixed > 0) against the jacobian_cases model, and every row equal, bit for bit,
    to the GPU VJP of its unit cotangent with the same status."""
    seq, opt, o = _build(cid, tmp_path)
    worst, seen = 0.0, []
    for with_last in (True, False):
        pts = V.solved_points(o, 3, 7, with_last=with_last)
        for form in ("ref_value", "keypoints"):
            args = (pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], pts["flags"])
            res = gpu_jacobian(opt, *args, **{form: pts[form]})
            assert (res[1] is None) == (len(o.idx_pin2fixed) == 0)
            m = JC.model_batch(o, pts, form)
            worst = max(worst, JC.compare(res, m))
            seen.append((~m["skip"], pts["qpos"], m["fixed"]))
            rows = vjp_loop(opt, *args, **{form: pts[form]})
            for st in rows[3]:
                np.testing.assert_array_equal(st, res[3])
            for a, b in zip(res[:3], rows[:3]):
                assert (a is None) == (b is None)
                if a is not None:
                    np.testing.assert_array_equal(a, b)
    _not_vacuous(cid, o, *map(np.concatenate, zip(*seen)))
    print(cid, "worst error / tau %.3f" % worst)


GUARD, SENTINEL = 64, 12345.0  # rows of sentinel before and after every output block of test_outputs_stay_inside_their_buffers


def _guarded(shape):
    """(buffer, view): `shape` rows in the middle of a buffer whose GUARD rows before and after hold SENTINEL."""
    big = torch.full((shape[0] + 2 * GUARD,) + tuple(shape[1:]), SENTINEL, device=_dev())
    return big, big[GUARD:GUARD + shape[0]]


def _check_guarded(bufs, got, want):
    """The returned blocks equal the plain call's bit for bit and every guard row still holds the sentinel."""
    for (name, (big, _)), g, w in zip(bufs.items(), got, want):
        _assert_same(_np(g), w, name)
        b = _np(big)
        assert (b[:GUARD] == SENTINEL).all() and (b[-GUARD:] == SENTINEL).all(), (name, "write outside the block")


@pytest.mark.parametrize("cid", ["fixed_dense16", "mimic_fixed_dense32", "dof31_vector"])
def test_outputs_stay_inside_their_buffers(cid, tmp_path, monkeypatch):
    """Every output block of the VJP, Jacobian and packed-VJP calls written into a view inside a larger buffer: the rows
    before and after it keep their sentinel, and the blocks equal the calls' own buffers.  A wrong per-frame stride or
    offset (grad_fixed_qpos strided by n_var instead of n_fixed, say) lands in the guard rows."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    seq, opt, o = _build(cid, tmp_path)
    n, nf, dof = opt.opt_dof, len(o.idx_pin2fixed), opt.robot.dof
    pts = V.solved_points(o, 3, 7)
    B = 3
    args = dict(fixed_qpos=_t(pts["fixed_qpos"]), last_qpos=_t(pts["last_qpos"]), keypoints=_t(pts["keypoints"]))
    plain = gpu_vjp(opt, pts["gbar"], pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], keypoints=pts["keypoints"])
    bufs = dict(grad_keypoints_out=_guarded((B, 21, 3)), grad_fixed_qpos_out=_guarded((B, nf)),
                grad_last_qpos_out=_guarded((B, n)))
    if not nf:
        del bufs["grad_fixed_qpos_out"]
    got = opt.retarget_batch_vjp(_t(pts["gbar"]), _t(pts["qpos"]), **args, **{k: v[1] for k, v in bufs.items()})
    torch.cuda.synchronize()
    _check_guarded(bufs, [g for g in got if g is not None], [w for w in plain[:3] if w is not None])

    plain = gpu_jacobian(opt, pts["qpos"], pts["fixed_qpos"], pts["last_qpos"], keypoints=pts["keypoints"])
    bufs = dict(jac_keypoints_out=_guarded((B, n, 21, 3)), jac_fixed_qpos_out=_guarded((B, n, nf)),
                jac_last_qpos_out=_guarded((B, n, n)))
    if not nf:
        del bufs["jac_fixed_qpos_out"]
    got = opt.retarget_batch_jacobian(_t(pts["qpos"]), **args, **{k: v[1] for k, v in bufs.items()})
    torch.cuda.synchronize()
    _check_guarded(bufs, [g for g in got if g is not None], [w for w in plain[:3] if w is not None])

    lengths = [3, 0, 1, 2]
    S, N_ = len(lengths), sum(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=84)
    st0 = _seeded_state(seq, o, S, seed=85)
    cot = _cotangents(seq, S, N_, seed=86)
    plain = _packed_all(seq, pk, pf, lengths, st0, cot)
    layout = seq.pack_streams(np.asarray(lengths, np.int64))
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(_t(pk), layout, _state_copy(st0), fixed_qpos=_t(pf), tape=tape)
    bufs = dict(grad_keypoints_out=_guarded((N_, 21, 3)), grad_fixed_qpos_out=_guarded((N_, nf)),
                grad_last_qpos_out=_guarded((S, n)), grad_filter_state_out=_guarded((S, dof)))
    if not nf:
        del bufs["grad_fixed_qpos_out"]
    got = seq.retarget_packed_sequences_vjp(_t(pk), layout, tape, st0.last_qpos, st0.filter_init, grad_robot_qpos=_t(cot[0]),
                                            grad_last_qpos=_t(cot[1]), grad_filter_state=_t(cot[2]), fixed_qpos=_t(pf),
                                            **{k: v[1] for k, v in bufs.items()})
    torch.cuda.synchronize()
    _check_guarded(bufs, [g for g in got if g is not None], [w for w in plain["grads"] if w is not None])


# ---- dexr_solve_sequences_tape / dexr_solve_sequences_vjp --------------------------------------------------------------

def _state(seq, p):
    st = seq.make_stream_state(len(p["last0"]))
    st.last_qpos.copy_(_t(p["last0"]))
    st.filter_state.copy_(_t(p["y0"]))
    st.filter_init.copy_(_t(p["finit"]))
    return st


@pytest.mark.parametrize("filtered", [True, False], ids=["filter", "nofilter"])
@pytest.mark.parametrize("cid", SEQ_CASES)
def test_sequence_vjp_matches_the_model(cid, filtered, tmp_path):
    """The taped forward equals the unrecorded one bit for bit; the backward at the oracle's streams against
    SV.model_stream, with all three cotangents."""
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq, opt, o = _build(cid, tmp_path, None if filtered else NO_FILTER)
    S, T = SEQ_SIZE
    p = _problem(seq, o, S, T, seed=21, pinch=o.type == "dexpilot", filter_init=1)
    if o.type == "dexpilot":  # the flags switch on and off again inside the streams
        on = p["F"].any(axis=2)
        assert on.any() and (~on).any(), on
    st_u, st_r = _state(seq, p), _state(seq, p)
    su, sr = (torch.empty((S, T), dtype=torch.int32, device=_dev()) for _ in range(2))
    out_u, _ = seq.retarget_sequences(_t(p["kp"]), st_u, fixed_qpos=_t(p["fixed"]), status_out=su)
    tape_r = seq.make_sequence_tape(S, T)
    out_r, _ = seq.retarget_sequences(_t(p["kp"]), st_r, fixed_qpos=_t(p["fixed"]), status_out=sr, tape=tape_r)
    _assert_same(_np(out_u), _np(out_r), "recorded forward")
    _assert_same(_np(su), _np(sr), "recorded forward status")
    for k, v in _state_np(st_u).items():
        _assert_same(v, _state_np(st_r)[k], k)
    _assert_same(_np(tape_r.qpos[:, -1]), _np(st_r.last_qpos), "tape end")

    status = torch.empty((S, T), dtype=torch.int32, device=_dev())
    got = seq.retarget_sequences_vjp(_t(p["kp"]), SequenceTape(qpos=_t(p["X"]), projected=_t(p["F"])), _t(p["last0"]),
                                     _t(p["finit"]), grad_robot_qpos=_t(p["g_out"]), grad_last_qpos=_t(p["g_last"]),
                                     grad_filter_state=_t(p["g_filter"]), fixed_qpos=_t(p["fixed"]), status_out=status)
    got = tuple(_np(g) for g in got) + (_np(status),)
    assert (got[1] is None) == (p["fixed"] is None)
    worst, keep, fx = 0.0, [], []
    for s in range(S):
        m = SV.model_stream(o, p["kp"][s], None if p["fixed"] is None else p["fixed"][s], p["last0"][s], p["finit"][s],
                            p["X"][s], None if p["F"] is None else p["F"][s], g_out=p["g_out"][s], g_last=p["g_last"][s],
                            g_filter=p["g_filter"][s])
        worst = max(worst, SV.compare_stream(tuple(None if g is None else g[s] for g in got), m))
        keep.append(~m["skip"])
        fx.append(m["fixed"])
    _not_vacuous(cid, o, np.concatenate(keep), p["X"].reshape(S * T, -1), np.concatenate(fx))
    print(cid, "filter" if filtered else "no filter", "worst error / tau %.3f" % worst)


# ---- dexr_solve_sequences_packed / dexr_solve_sequences_packed_vjp ------------------------------------------------------

def _seeded_state(seq, o, S, seed):
    rng = np.random.RandomState(seed)
    last0 = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0], o.joint_limits[:, 1])
    return _state(seq, dict(last0=last0.astype(np.float32), finit=np.ones(S, np.uint8),
                            y0=rng.uniform(-0.3, 0.3, size=(S, o.robot.dof)).astype(np.float32)))


def _packed_all(seq, pk, pf, lengths, st0, cot):
    """Unrecorded and recorded packed forward (equal bit for bit) and the packed VJP from state st0 (not modified)."""
    N_ = int(np.sum(lengths))
    layout = seq.pack_streams(np.asarray(lengths, np.int64))
    st_u, st = _state_copy(st0), _state_copy(st0)
    out_u, _ = seq.retarget_packed_sequences(_t(pk), layout, st_u, fixed_qpos=_t(pf))
    status = torch.empty((N_,), dtype=torch.int32, device=_dev())
    tape = seq.make_packed_sequence_tape(layout)
    out, _ = seq.retarget_packed_sequences(_t(pk), layout, st, fixed_qpos=_t(pf), status_out=status, tape=tape)
    _assert_same(_np(out_u), _np(out), "unrecorded packed forward")
    for k, v in _state_np(st_u).items():
        _assert_same(v, _state_np(st)[k], k)
    vstatus = torch.empty((N_,), dtype=torch.int32, device=_dev())
    grads = seq.retarget_packed_sequences_vjp(_t(pk), layout, tape, st0.last_qpos, st0.filter_init,
                                              grad_robot_qpos=_t(cot[0]), grad_last_qpos=_t(cot[1]),
                                              grad_filter_state=_t(cot[2]), fixed_qpos=_t(pf), status_out=vstatus)
    return dict(out=_np(out), status=_np(status), state=_state_np(st), tape_qpos=_np(tape.qpos),
                tape_proj=_np(tape.projected), grads=[_np(g) for g in grads], vstatus=_np(vstatus))


def _sub_state(st, s):
    return {k: None if v is None else v[s:s + 1] for k, v in _state_np(st).items()}


@pytest.mark.parametrize("cid", PACKED_CASES)
def test_packed_ragged_streams_are_each_stream_alone(cid, tmp_path, monkeypatch):
    """Lengths 3, 0, 1, 2, 0, 4, 1: each stream's outputs, status, final state, tape and gradients equal the same stream
    packed alone; a stream of length 0 keeps its state and passes its cotangents through.  Without duo mode, which would
    split a lone 16-lane stream over two half-warps."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    seq, opt, o = _build(cid, tmp_path)
    lengths = RAGGED
    S = len(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=84, pinch=o.type == "dexpilot")
    st0 = _seeded_state(seq, o, S, seed=85)
    cot = _cotangents(seq, S, sum(lengths), seed=86)
    got = _packed_all(seq, pk, pf, lengths, st0, cot)
    assert (got["grads"][1] is None) == (pf is None)
    offs = np.concatenate([[0], np.cumsum(lengths)])
    for s, n in enumerate(lengths):
        a, b = offs[s], offs[s + 1]
        mine = {k: None if v is None else v[s:s + 1] for k, v in got["state"].items()}
        if n == 0:
            for k, v in _sub_state(st0, s).items():
                _assert_same(mine[k], v, f"empty stream {s} {k}")
            _assert_same(got["grads"][2][s], cot[1][s], "empty stream: grad_last_qpos passes through")
            _assert_same(got["grads"][3][s], cot[2][s], "empty stream: grad_filter_state passes through")
            continue
        one = seq.make_stream_state(1)
        for k in ("last_qpos", "filter_state", "filter_init"):
            getattr(one, k).copy_(getattr(st0, k)[s:s + 1])
        alone = _packed_all(seq, pk[a:b], None if pf is None else pf[a:b], [n], one,
                            (cot[0][a:b], cot[1][s:s + 1], cot[2][s:s + 1]))
        _assert_same(got["out"][a:b], alone["out"], f"stream {s} robot_qpos")
        _assert_same(got["status"][a:b], alone["status"], f"stream {s} status")
        for k, v in alone["state"].items():
            _assert_same(mine[k], v, f"stream {s} {k}")
        _assert_same(got["tape_qpos"][a:b], alone["tape_qpos"], f"stream {s} tape")
        if alone["tape_proj"] is not None:
            _assert_same(got["tape_proj"][a:b], alone["tape_proj"], f"stream {s} flag tape")
        g_kp, g_fixed, g_last, g_filter = got["grads"]
        _assert_same(g_kp[a:b], alone["grads"][0], f"stream {s} grad_keypoints")
        if g_fixed is not None:
            _assert_same(g_fixed[a:b], alone["grads"][1], f"stream {s} grad_fixed_qpos")
        _assert_same(g_last[s], alone["grads"][2][0], f"stream {s} grad_last_qpos")
        _assert_same(g_filter[s], alone["grads"][3][0], f"stream {s} grad_filter_state")
        _assert_same(got["vstatus"][a:b], alone["vstatus"], f"stream {s} vjp status")


@pytest.mark.parametrize("cid", PACKED_CASES)
def test_packed_equal_lengths_are_the_rectangular_calls(cid, tmp_path, monkeypatch):
    """Every stream T frames: forward, tape, final state, gradients and statuses equal dexr_solve_sequences / _tape / _vjp."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    seq, opt, o = _build(cid, tmp_path)
    S, T = SEQ_SIZE
    kp, fixed, pk, pf = _inputs(o, [T] * S, seed=81, pinch=o.type == "dexpilot")
    st0 = _seeded_state(seq, o, S, seed=82)
    cot = _cotangents(seq, S, S * T, seed=83)
    got = _packed_all(seq, pk, pf, [T] * S, st0, cot)
    st = _state_copy(st0)
    status = torch.empty((S, T), dtype=torch.int32, device=_dev())
    tape = seq.make_sequence_tape(S, T)
    out, _ = seq.retarget_sequences(_t(kp), st, fixed_qpos=_t(fixed), status_out=status, tape=tape)
    _assert_same(got["out"], _np(out).reshape(S * T, -1), "robot_qpos")
    _assert_same(got["status"], _np(status).reshape(-1), "status")
    for k, v in _state_np(st).items():
        _assert_same(got["state"][k], v, k)
    _assert_same(got["tape_qpos"], _np(tape.qpos).reshape(S * T, -1), "tape.qpos")
    if tape.projected is not None:
        _assert_same(got["tape_proj"], _np(tape.projected).reshape(S * T, -1), "tape.projected")
    vstatus = torch.empty((S, T), dtype=torch.int32, device=_dev())
    grads = seq.retarget_sequences_vjp(_t(kp), tape, st0.last_qpos, st0.filter_init, grad_robot_qpos=_t(cot[0].reshape(S, T, -1)),
                                       grad_last_qpos=_t(cot[1]), grad_filter_state=_t(cot[2]), fixed_qpos=_t(fixed),
                                       status_out=vstatus)
    for a, b, name in zip(got["grads"], grads, ("grad_keypoints", "grad_fixed_qpos", "grad_last_qpos", "grad_filter_state")):
        _assert_same(a, None if b is None else _np(b).reshape(a.shape), name)
    _assert_same(got["vstatus"], _np(vstatus).reshape(-1), "vjp status")


@pytest.mark.parametrize("cid", PACKED_CASES)
def test_packed_vjp_matches_the_model(cid, tmp_path):
    """The packed VJP of two streams (and an empty one between them) at the oracle streams' tape against
    SV.model_stream."""
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq, opt, o = _build(cid, tmp_path)
    lengths = [3, 0, 2]
    S = len(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=87, pinch=o.type == "dexpilot")
    st0 = _seeded_state(seq, o, S, seed=88)
    last0, y0 = _np(st0.last_qpos), _np(st0.filter_state)
    cot = _cotangents(seq, S, sum(lengths), seed=89)
    offs = np.concatenate([[0], np.cumsum(lengths)])
    refs = [None if n == 0 else SV.oracle_stream(o, kp[s, :n], None if fixed is None else fixed[s, :n], last0[s], y0[s], 1)
            for s, n in enumerate(lengths)]
    X = np.concatenate([r["qpos"] for r in refs if r is not None]).astype(np.float32)
    F = None if refs[0]["flags"] is None else np.concatenate([r["flags"] for r in refs if r is not None])
    status = torch.empty((len(X),), dtype=torch.int32, device=_dev())
    grads = seq.retarget_packed_sequences_vjp(_t(pk), seq.pack_streams(np.asarray(lengths, np.int64)),
                                              SequenceTape(qpos=_t(X), projected=_t(F)), st0.last_qpos, st0.filter_init,
                                              grad_robot_qpos=_t(cot[0]), grad_last_qpos=_t(cot[1]),
                                              grad_filter_state=_t(cot[2]), fixed_qpos=_t(pf), status_out=status)
    grads = [_np(g) for g in grads] + [_np(status)]
    worst, keep, fx = 0.0, [], []
    for s, n in enumerate(lengths):
        if n == 0:
            continue
        a, b = offs[s], offs[s + 1]
        m = SV.model_stream(o, kp[s, :n], None if fixed is None else fixed[s, :n], last0[s], 1, refs[s]["qpos"],
                            refs[s]["flags"], g_out=cot[0][a:b], g_last=cot[1][s], g_filter=cot[2][s])
        one = (grads[0][a:b], None if grads[1] is None else grads[1][a:b], grads[2][s], grads[3][s], grads[4][a:b])
        worst = max(worst, SV.compare_stream(one, m))
        keep.append(~m["skip"])
        fx.append(m["fixed"])
    _not_vacuous(cid, o, np.concatenate(keep), X, np.concatenate(fx))
    print(cid, "worst error / tau %.3f" % worst)


# ---- dexr_smooth_sequences_packed ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("cid", SMOOTH_CASES)
def test_smoothing_minimiser_and_descent(cid, tmp_path):
    """test_gpu_smooth.test_minimiser_and_descent on short ragged clips: finite, every clip descends from the causal tape,
    and on SMOOTH_CHECKED of the clips that converged the float64 polish moves the answer by no more than PARITY and finds no
    lower F.  Instead of GS.MAXITER_FRACTION (which allows no clip of 8), no more clips end at max_iters than SMOOTH_MAXITER
    states per case."""
    seq, opt, o = _build(cid, tmp_path)
    S, lo, hi = SMOOTH_CLIPS
    kp, lengths = GS.W.ragged_streams(S, lo, hi, 11)
    fixed = GS._fixed(o, int(lengths.sum()), 1)
    r = GS._run(seq, kp, lengths, fixed)
    assert np.isfinite(r["q"]).all() and not (r["status"] & GS.STATUS_NONFINITE).any()
    offs = np.concatenate([[0], np.cumsum(lengths)])
    maxiter = (r["status"][offs[:-1]] & GS.STATUS_MAXITER) != 0
    assert maxiter.sum() <= SMOOTH_MAXITER.get(cid, 0), (cid, np.flatnonzero(maxiter))
    for s, a, b, m in GS._models(seq, o, r, fixed, range(S)):
        f, f0 = m.value(r["q"][a:b]), m.value(r["tape_q"][a:b])
        assert f <= f0 * (1 + 1e-6), (cid, s, f, f0)  # descent from the causal start
    worst = 0.0
    chosen = np.random.RandomState(0).choice(np.flatnonzero(~maxiter), SMOOTH_CHECKED, replace=False)
    for s, a, b, m in GS._models(seq, o, r, fixed, chosen):
        X = r["q"][a:b].astype(np.float64)
        f = m.value(X)
        Xp = m.polish(X)
        worst = max(worst, float(np.abs(Xp - X).max()))
        assert np.abs(Xp - X).max() <= SMC.PARITY, (cid, s, np.abs(Xp - X).max())
        assert m.value(Xp) >= f - 1e-6 * abs(f), (cid, s, f)
    print(cid, int(maxiter.sum()), "of", S, "clips at max_iters; worst polish move / PARITY %.3f" % (worst / SMC.PARITY))


def test_smoothing_interpolates_dropped_frames_with_fixed_joints(tmp_path):
    """Leading, interior and trailing gaps of a clip of fixed_dense16: flagged missing and filled by the interpolation."""
    seq, opt, o = _build("fixed_dense16", tmp_path)
    T = DROP_LENGTH
    kp, _ = GS.W.ragged_streams(1, T, T, 6)
    drop = np.r_[0:2, T // 2 - 2:T // 2 + 1, T - 3:T]
    fixed = GS._fixed(o, T, 3)
    r = GS._run(seq, kp, np.array([T], np.int64), fixed, drop=drop)
    miss = np.zeros(T, bool)
    miss[drop] = True
    np.testing.assert_array_equal((r["status"] & GS.STATUS_MISSING) != 0, miss)
    q = r["q"].astype(np.float64)
    anchor = SMC.clipped_anchor(o, _np(r["state"].last_qpos))[0]
    i0, i1 = T // 2 - 2, T // 2 + 1
    np.testing.assert_allclose(q[i0:i1], SMC.interpolation(q[i0 - 1], q[i1], i1 - i0), atol=1e-5)
    np.testing.assert_allclose(q[T - 3:], SMC.interpolation(q[T - 4], None, 3, has_next=False), atol=1e-5)
    np.testing.assert_allclose(q[0:2], SMC.interpolation(anchor, q[2], 2), atol=1e-5)


# ---- autograd with fixed_qpos.requires_grad -----------------------------------------------------------------------------

@pytest.mark.parametrize("cid", DIFF_CASES)
def test_differentiable_retarget_fixed_joint_gradient(cid, tmp_path):
    """fixed_qpos.grad of backward() equals the direct VJP call bit for bit, the model at the GPU's answers, and central
    differences of the oracle's converged minimiser in each fixed joint (h = 1e-4) on frames with no variable within 1e-3
    of a bound and an unchanged active set."""
    from dex_retargeting_b200.objective import differentiable_retarget
    from oracle.solvers import solve_converged

    seq, opt, o = _build(cid, tmp_path)
    B = 6
    pts = V.solved_points(o, B, seed=25)
    fx = _t(pts["fixed_qpos"]).requires_grad_(True)
    q = differentiable_retarget(opt, keypoints=_t(pts["keypoints"]), fixed_qpos=fx, last_qpos=_t(pts["last_qpos"]))
    (q * _t(pts["gbar"])).sum().backward()
    torch.cuda.synchronize()
    qn, g_fx = _np(q), _np(fx.grad)
    direct = gpu_vjp(opt, pts["gbar"], qn, pts["fixed_qpos"], pts["last_qpos"], keypoints=pts["keypoints"])
    np.testing.assert_array_equal(g_fx, direct[1])
    model_pts = dict(pts, qpos=qn)
    m = V.model_batch(o, model_pts, "keypoints")
    ratio = V.compare(direct, m, model_pts)
    _not_vacuous(cid, o, ~m["skip"], qn, m["fixed"])
    h, checked = 1e-4, 0
    lo32, hi32 = np.float32(o.lower), np.float32(o.upper)
    for i in range(B):
        at_bound = (qn[i] <= lo32) | (qn[i] >= hi32)
        near = ~at_bound & ((qn[i] < lo32 + 1e-3) | (qn[i] > hi32 - 1e-3))
        if m["skip"][i] or near.any() or direct[3][i] != 0:
            continue
        ref = o.ref_from_keypoints(pts["keypoints"][i].astype(np.float64))
        scale = float(np.abs(m["fixed"][i]).max())
        for k in range(fx.shape[1]):
            xs = []
            for s in (1.0, -1.0):
                f2 = pts["fixed_qpos"][i].astype(np.float64)
                f2[k] += s * h
                x, kkt, _ = solve_converged(o, ref, f2, pts["last_qpos"][i], x_init=qn[i])
                assert kkt < 1e-7, kkt
                assert np.array_equal((x <= o.lower + 1e-7) | (x >= o.upper - 1e-7), at_bound)
                xs.append(x)
            fd = float(pts["gbar"][i].astype(np.float64) @ (xs[0] - xs[1]) / (2 * h))
            assert abs(g_fx[i, k] - fd) <= 2e-3 * scale, (cid, i, k, g_fx[i, k], fd, scale)
        checked += 1
    assert checked >= 2, checked
    print(cid, "model worst error / tau %.3f;" % ratio, "central differences agree on", checked, "frames")


@pytest.mark.parametrize("cid", DIFF_CASES)
def test_differentiable_retarget_sequences_fixed_joint_gradient(cid, tmp_path):
    """fixed_qpos.grad of backward() through differentiable_retarget_sequences equals the direct retarget_sequences_vjp
    call on a recorded forward bit for bit, and the model at the GPU's tape."""
    from dex_retargeting_b200.objective import differentiable_retarget_sequences

    seq, opt, o = _build(cid, tmp_path)
    S, T = SEQ_SIZE
    kp, fixed = SV.stream_inputs(o, S, T, seed=45)
    g_out = np.random.RandomState(46).randn(S, T, opt.robot.dof).astype(np.float32)
    fx = _t(fixed).requires_grad_(True)
    out, _ = differentiable_retarget_sequences(seq, _t(kp), seq.make_stream_state(S), fixed_qpos=fx)
    (out * _t(g_out)).sum().backward()
    st = seq.make_stream_state(S)
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    tape = seq.make_sequence_tape(S, T)
    out2, _ = seq.retarget_sequences(_t(kp), st, fixed_qpos=_t(fixed), tape=tape)
    _assert_same(_np(out), _np(out2), "differentiable forward")
    status = torch.empty((S, T), dtype=torch.int32, device=_dev())
    direct = seq.retarget_sequences_vjp(_t(kp), tape, last0, finit0, grad_robot_qpos=_t(g_out), fixed_qpos=_t(fixed),
                                        status_out=status)
    direct = tuple(_np(g) for g in direct) + (_np(status),)
    np.testing.assert_array_equal(_np(fx.grad), direct[1])
    X, l0, f0 = _np(tape.qpos), _np(last0), _np(finit0)
    worst, keep, fxm = 0.0, [], []
    for s in range(S):
        m = SV.model_stream(o, kp[s], fixed[s], l0[s], f0[s], X[s], None, g_out=g_out[s])
        worst = max(worst, SV.compare_stream(tuple(g[s] for g in direct), m))
        keep.append(~m["skip"])
        fxm.append(m["fixed"])
    _not_vacuous(cid, o, np.concatenate(keep), X.reshape(S * T, -1), np.concatenate(fxm))
    print(cid, "worst error / tau %.3f" % worst)


@pytest.mark.parametrize("cid", DIFF_CASES)
def test_differentiable_retarget_packed_sequences_fixed_joint_gradient(cid, tmp_path, monkeypatch):
    """As for the rectangular streams, through differentiable_retarget_packed_sequences on lengths 3, 0, 2."""
    from dex_retargeting_b200.objective import differentiable_retarget_packed_sequences

    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    seq, opt, o = _build(cid, tmp_path)
    lengths = [3, 0, 2]
    S, N_ = len(lengths), sum(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=47, pinch=o.type == "dexpilot")
    layout = seq.pack_streams(np.asarray(lengths, np.int64))
    g_out = np.random.RandomState(48).randn(N_, opt.robot.dof).astype(np.float32)
    fx = _t(pf).requires_grad_(True)
    out, _ = differentiable_retarget_packed_sequences(seq, _t(pk), layout, seq.make_stream_state(S), fixed_qpos=fx)
    (out * _t(g_out)).sum().backward()
    st = seq.make_stream_state(S)
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    tape = seq.make_packed_sequence_tape(layout)
    out2, _ = seq.retarget_packed_sequences(_t(pk), layout, st, fixed_qpos=_t(pf), tape=tape)
    _assert_same(_np(out), _np(out2), "differentiable forward")
    status = torch.empty((N_,), dtype=torch.int32, device=_dev())
    direct = seq.retarget_packed_sequences_vjp(_t(pk), layout, tape, last0, finit0, grad_robot_qpos=_t(g_out),
                                               fixed_qpos=_t(pf), status_out=status)
    direct = [_np(g) for g in direct] + [_np(status)]
    np.testing.assert_array_equal(_np(fx.grad), direct[1])
    X, l0, f0 = _np(tape.qpos), _np(last0), _np(finit0)
    offs = np.concatenate([[0], np.cumsum(lengths)])
    worst, keep, fxm = 0.0, [], []
    for s, n in enumerate(lengths):
        if n == 0:
            continue
        a, b = offs[s], offs[s + 1]
        m = SV.model_stream(o, kp[s, :n], fixed[s, :n], l0[s], f0[s], X[a:b], None, g_out=g_out[a:b])
        one = (direct[0][a:b], direct[1][a:b], direct[2][s], direct[3][s], direct[4][a:b])
        worst = max(worst, SV.compare_stream(one, m))
        keep.append(~m["skip"])
        fxm.append(m["fixed"])
    _not_vacuous(cid, o, np.concatenate(keep), X, np.concatenate(fxm))
    print(cid, "worst error / tau %.3f" % worst)
