"""Backpropagation through the sequence solve on the GPU (`dexr_solve_sequences_tape`, `dexr_solve_sequences_vjp`,
SeqRetargeting.retarget_sequences_vjp, objective.differentiable_retarget_sequences): the recorded forward against the
unrecorded one bit for bit, the fused backward against the float64 model of tests/seq_vjp_cases.py and the host emulation,
against the per-frame loop of retarget_batch_vjp with the clip, mask and filter in torch, against central differences of
whole oracle streams, across chunk boundaries, across batch layouts, and the library's argument checks."""
import sys
from pathlib import Path

import numpy as np
import pytest

import seq_vjp_cases as SV
from helpers import build_oracle, build_product

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KEYS = ["teleop/leap_hand_right_dexpilot", "teleop/allegro_hand_right", "offline/shadow_hand_right"]
# streams x steps of the recorded-forward check and of the per-frame-loop comparison (the CPU dry run,
# tests/tools/emu_gpu_seq_vjp.py, shrinks them: the emulation solves a few frames per second)
FORWARD_SIZE = (96, 40)
LOOP_SIZE = (32, 12)


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def _bench_streams(S, T, seed):
    """The benchmark's seeded stream workload (tools/workloads.py `streams`): the first T recorded frames with a 2 mm
    offset per stream."""
    return W.streams(S, T, seed)


def _seq(key, override=None):
    return build_product(key, override, device=0)


def _state_copy(st):
    from dex_retargeting_b200.seq_retarget import StreamState

    return StreamState(**{k: None if getattr(st, k) is None else getattr(st, k).clone() for k in StreamState._FIELDS})


@pytest.mark.parametrize("key", KEYS)
def test_recorded_forward_is_bit_identical(key):
    seq = _seq(key)
    S, T = FORWARD_SIZE
    kp = _t(_bench_streams(S, T, seed=W.STREAM_SEED))
    st_a = seq.make_stream_state(S)
    st_b = _state_copy(st_a)
    sa, sb = torch.empty((S, T), dtype=torch.int32, device=_dev()), torch.empty((S, T), dtype=torch.int32, device=_dev())
    out_a, _ = seq.retarget_sequences(kp, st_a, status_out=sa)
    tape = seq.make_sequence_tape(S, T)
    out_b, _ = seq.retarget_sequences(kp, st_b, status_out=sb, tape=tape)
    torch.cuda.synchronize()
    assert torch.equal(out_a, out_b) and torch.equal(sa, sb)
    for k in ("last_qpos", "filter_state", "filter_init", "projected", "damping"):
        if getattr(st_a, k) is not None:
            assert torch.equal(getattr(st_a, k), getattr(st_b, k)), k
    assert torch.equal(tape.qpos[:, -1], st_b.last_qpos)
    if tape.projected is not None:
        assert torch.equal(tape.projected[:, -1], st_b.projected)


def _oracle_problem(key, override, S, T, seed, pinch=False):
    seq = _seq(key, override)
    o = build_oracle(key, override)
    kp, fixed = SV.stream_inputs(o, S, T, seed, pinch=pinch)
    rng = np.random.RandomState(seed + 1)
    last0 = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0],
                    o.joint_limits[:, 1]).astype(np.float32)
    y0 = rng.uniform(-0.3, 0.3, size=(S, o.robot.dof)).astype(np.float32)
    finit = np.zeros(S, np.uint8)
    ref = SV.oracle_streams(o, kp, fixed, last0, y0, finit)
    g = dict(g_out=rng.randn(S, T, o.robot.dof).astype(np.float32), g_last=rng.randn(S, o.opt_dof).astype(np.float32),
             g_filter=rng.randn(S, o.robot.dof).astype(np.float32))
    return seq, o, dict(kp=kp, fixed=fixed, last0=last0, y0=y0, finit=finit, X=ref["qpos"], F=ref["flags"], **g)


@pytest.mark.parametrize("key,pinch", [(KEYS[0], True), (KEYS[1], False), (KEYS[2], False)])
def test_backward_matches_model_and_emulation(key, pinch):
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq, o, p = _oracle_problem(key, None, 3, 4, seed=41, pinch=pinch)
    tape = SequenceTape(qpos=_t(p["X"]), projected=_t(p["F"]))
    status = torch.empty((3, 4), dtype=torch.int32, device=_dev())
    got = seq.retarget_sequences_vjp(_t(p["kp"]), tape, _t(p["last0"]), _t(p["finit"]), grad_robot_qpos=_t(p["g_out"]),
                                     grad_last_qpos=_t(p["g_last"]), grad_filter_state=_t(p["g_filter"]),
                                     fixed_qpos=_t(p["fixed"]), status_out=status)
    got = tuple(_np(g) for g in got) + (_np(status),)
    for s in range(3):
        m = SV.model_stream(o, p["kp"][s], None, p["last0"][s], p["finit"][s], p["X"][s],
                            None if p["F"] is None else p["F"][s], g_out=p["g_out"][s], g_last=p["g_last"][s],
                            g_filter=p["g_filter"][s])
        SV.compare_stream(tuple(None if g is None else g[s] for g in got), m)
    import emu_seq_vjp_host as H

    emu = H.solve_sequences_vjp(seq, p["kp"], p["X"], p["last0"], p["finit"], p["F"], grad_robot_qpos=p["g_out"],
                                grad_last_qpos=p["g_last"], grad_filter_state=p["g_filter"])
    np.testing.assert_array_equal(got[4], emu[4])
    for a, b in ((got[0], emu[0]), (got[2], emu[2]), (got[3], emu[3])):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-4 * max(np.abs(b).max(), 1e-6))


def _per_frame_loop(seq, kp, fixed, last0, finit, tape, g_out):
    """The backward written as T retarget_batch_vjp launches with the clip, the clip mask and the filter in torch."""
    opt = seq.optimizer
    S, T = kp.shape[:2]
    alpha = seq.low_pass_alpha
    use_filter = 0 <= alpha <= 1
    lim = torch.from_numpy(np.ascontiguousarray(seq.joint_limits, dtype=np.float32)).to(_dev())
    M = torch.zeros((opt.robot.dof, opt.opt_dof), device=_dev())  # dq/dx of scatter + mimic
    for j in range(opt.opt_dof):
        M[:, j] = torch.as_tensor(_full_q(opt, j), device=_dev())
    gy = torch.zeros((S, opt.robot.dof), device=_dev())
    c = torch.zeros((S, opt.opt_dof), device=_dev())
    g_kp = torch.empty_like(kp)
    for t in range(T - 1, -1, -1):
        if use_filter:
            gy = gy + g_out[:, t]
            init = torch.ones(S, dtype=torch.bool, device=_dev()) if t > 0 else finit.bool()
            gq = torch.where(init[:, None], alpha * gy, gy)
            gy = torch.where(init[:, None], (1 - alpha) * gy, torch.zeros_like(gy))
        else:
            gq = g_out[:, t]
        gbar = (gq @ M + c).contiguous()
        xp = tape.qpos[:, t - 1] if t > 0 else last0
        anchor = torch.clamp(xp, lim[:, 0], lim[:, 1]).contiguous()
        proj = None if tape.projected is None else tape.projected[:, t].contiguous()
        gk, _, ga = opt.retarget_batch_vjp(gbar, tape.qpos[:, t].contiguous(), keypoints=kp[:, t].contiguous(),
                                           last_qpos=anchor, projected=proj,
                                           fixed_qpos=None if fixed is None else fixed[:, t].contiguous())
        g_kp[:, t] = gk
        c = ga * ((xp >= lim[:, 0]) & (xp <= lim[:, 1]))
    return g_kp, c, gy


def _full_q(opt, j):
    x = np.zeros(opt.opt_dof)
    x[j] = 1.0
    q = np.zeros(opt.robot.dof)
    q[opt.idx_pin2target] = x
    if opt.adaptor is not None:
        q = opt.adaptor.forward_qpos(q) - opt.adaptor.forward_qpos(np.zeros(opt.robot.dof))
    return q.astype(np.float32)


@pytest.mark.parametrize("key", KEYS[:2])
def test_fused_backward_matches_the_per_frame_loop(key):
    seq = _seq(key)
    S, T = LOOP_SIZE
    kp_np = _bench_streams(S, T, seed=43)
    kp = _t(kp_np)
    state = seq.make_stream_state(S)
    last0, finit = state.last_qpos.clone(), state.filter_init.clone()
    tape = seq.make_sequence_tape(S, T)
    seq.retarget_sequences(kp, state, tape=tape)
    g_out = torch.randn((S, T, seq.optimizer.robot.dof), generator=torch.Generator().manual_seed(44)).to(_dev())
    g_kp, _, g_last, g_filter = seq.retarget_sequences_vjp(kp, tape, last0, finit, grad_robot_qpos=g_out)
    l_kp, l_last, l_filter = _per_frame_loop(seq, kp, None, last0, finit, tape, g_out)
    for a, b in ((g_kp, l_kp), (g_last, l_last), (g_filter, l_filter)):
        scale = float(b.abs().max())
        assert float((a - b).abs().max()) <= 1e-4 * max(scale, 1e-6), (float((a - b).abs().max()), scale)


def test_differentiable_retarget_sequences_against_central_differences():
    from dex_retargeting_b200.objective import differentiable_retarget_sequences

    key = "teleop/allegro_hand_right"
    seq, o, p = _oracle_problem(key, None, 1, 4, seed=45)
    state = seq.make_stream_state(1)
    state.last_qpos.copy_(_t(p["last0"]))
    state.filter_state.copy_(_t(p["y0"]))
    state.filter_init.fill_(1)
    kp = _t(p["kp"]).requires_grad_(True)
    last = state.last_qpos.clone().requires_grad_(True)
    filt = state.filter_state.clone().requires_grad_(True)
    state.last_qpos, state.filter_state = last, filt
    out, new = differentiable_retarget_sequences(seq, kp, state)
    w = _t(p["g_out"])
    (w * out).sum().backward()
    g = w[0].double().cpu().numpy()

    def loss(kp_=p["kp"][0], last0=p["last0"][0], y0=p["y0"][0]):
        r = SV.oracle_stream(o, kp_, None, last0, y0, 1)
        return float((g * r["robot_qpos"]).sum())

    h = 1e-3
    used = int(np.asarray(o.target_link_human_indices).reshape(-1)[-1])
    for name, at, grad in (("kp_", (0, used, 1), kp.grad[0]), ("kp_", (3, used, 0), kp.grad[0]),
                           ("last0", (2,), last.grad[0]), ("y0", (1,), filt.grad[0])):
        base = dict(kp_=p["kp"][0], last0=p["last0"][0], y0=p["y0"][0])[name].astype(np.float64)
        plus, minus = base.copy(), base.copy()
        plus[at] += h
        minus[at] -= h
        fd = (loss(**{name: plus}) - loss(**{name: minus})) / (2 * h)
        an = float(grad[at])
        assert abs(an - fd) <= 5e-2 * max(abs(fd), 2e-2), (name, at, an, fd)


@pytest.mark.parametrize("key", KEYS[:2])
def test_chunked_streams_give_bit_identical_gradients(key):
    from dex_retargeting_b200.objective import differentiable_retarget_sequences

    seq = _seq(key)
    S, T, T1 = 8, 10, 4
    kp_np = _bench_streams(S, T, seed=47)
    w = torch.randn((S, T, seq.optimizer.robot.dof), generator=torch.Generator().manual_seed(48)).to(_dev())

    def run(split):
        kp = _t(kp_np).requires_grad_(True)
        state = seq.make_stream_state(S)
        last = state.last_qpos.clone().requires_grad_(True)
        state.last_qpos = last
        if split:
            o1, s1 = differentiable_retarget_sequences(seq, kp[:, :T1], state)
            o2, _ = differentiable_retarget_sequences(seq, kp[:, T1:], s1)
            out = torch.cat([o1, o2], dim=1)
        else:
            out, _ = differentiable_retarget_sequences(seq, kp, state)
        (w * out).sum().backward()
        return out.detach(), kp.grad, last.grad

    a, b = run(False), run(True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_stream_gradients_do_not_depend_on_the_batch_layout():
    key = KEYS[0]
    seq = _seq(key)
    S, T = 5, 6
    kp_np = _bench_streams(S, T, seed=49)
    g_np = np.random.RandomState(50).randn(S, T, seq.optimizer.robot.dof).astype(np.float32)

    def grads(rows):
        kp = _t(kp_np[rows])
        state = seq.make_stream_state(len(rows))
        last0, finit = state.last_qpos.clone(), state.filter_init.clone()
        tape = seq.make_sequence_tape(len(rows), T)
        seq.retarget_sequences(kp, state, tape=tape)
        return [_np(x) for x in seq.retarget_sequences_vjp(kp, tape, last0, finit, grad_robot_qpos=_t(g_np[rows]))
                if x is not None]

    full = grads(list(range(S)))
    alone = grads([3])
    moved = grads([3, 0, 1])
    for f, a, m in zip(full, alone, moved):
        np.testing.assert_array_equal(f[3], a[0])
        np.testing.assert_array_equal(f[3], m[0])


def test_argument_errors_are_rejected_with_a_message():
    from dex_retargeting_b200._native import DexrError
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq = _seq(KEYS[0])
    S, T = 2, 3
    kp = torch.zeros((S, T, 21, 3), device=_dev())
    state = seq.make_stream_state(S)
    tape = seq.make_sequence_tape(S, T)
    with pytest.raises(DexrError, match="flag tape"):
        seq.retarget_sequences(kp, state, tape=SequenceTape(qpos=tape.qpos, projected=None))
    with pytest.raises(DexrError, match="DexPilot needs the flag tape"):
        seq.retarget_sequences_vjp(kp, SequenceTape(qpos=tape.qpos, projected=None), state.last_qpos, state.filter_init)
    with pytest.raises(ValueError, match="tape.projected"):  # a flag tape narrower than the robot's len_proj
        seq.retarget_sequences(kp, state, tape=SequenceTape(qpos=tape.qpos, projected=tape.projected[:, :, :1].contiguous()))
    with pytest.raises(ValueError, match="tape.qpos"):
        seq.retarget_sequences_vjp(kp, SequenceTape(qpos=tape.qpos[:, :2].contiguous(), projected=tape.projected),
                                   state.last_qpos, state.filter_init)
