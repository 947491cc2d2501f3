#!/usr/bin/env python
"""Backpropagation through the sequence solve (`dexr_solve_sequences_vjp`) against its forward, on the stream workloads of
tools/workloads.py (`workloads.streams`: the first T recorded frames with a 2 mm per-stream offset, fresh stream state).

  python tools/bench_seq_vjp.py [--seconds 1.0] [--steps 300] [--out result.json]

Per workload, CUDA events around back-to-back calls after warm-up, at least --seconds of calls per number:
  forward        retarget_sequences (dexr_solve_sequences), state reset before every call
  taped forward  the same with a SequenceTape (dexr_solve_sequences_tape)
  fused backward retarget_sequences_vjp (dexr_solve_sequences_vjp), seeded dl/drobot_qpos
  per-frame loop the same backward as T retarget_batch_vjp launches with the clip, the clip mask and the filter in torch
Workloads: LEAP DexPilot 2048 x T (BASELINE config 4), Allegro vector 2048 x T, Shadow position 512 x T.
DEXR_SEQ_VJP_SPW=1 in the environment runs the one-stream-per-warp launch shape of the backward (16-lane robots).
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import workloads as W  # noqa: E402
from bench_objective import card  # noqa: E402

WORKLOADS = [("leap_dexpilot", W.LEAP_DEXPILOT_KEY, 2048), ("allegro_vector", W.METRIC_KEY, 2048),
             ("shadow_position", W.SHADOW_POS_KEY, 512)]


def time_calls(fn, seconds):
    """(seconds per call, calls): CUDA events around back-to-back calls, at least `seconds` of them, after two warm-ups."""
    fn()
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    one = max(time.perf_counter() - t0, 1e-6)
    calls = max(3, int(seconds / one) + 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / calls, calls


def per_frame_loop(seq, kp, last0, finit, tape, g_out, lim, M):
    """The backward as T retarget_batch_vjp launches with the clip, the clip mask and the filter in torch."""
    opt = seq.optimizer
    S, T = kp.shape[:2]
    alpha = seq.low_pass_alpha
    use_filter = 0 <= alpha <= 1
    gy = torch.zeros((S, opt.robot.dof), device=kp.device)
    c = torch.zeros((S, opt.opt_dof), device=kp.device)
    g_kp = torch.empty_like(kp)
    for t in range(T - 1, -1, -1):
        if use_filter:
            gy = gy + g_out[:, t]
            init = torch.ones(S, dtype=torch.bool, device=kp.device) if t > 0 else finit.bool()
            gq = torch.where(init[:, None], alpha * gy, gy)
            gy = torch.where(init[:, None], (1 - alpha) * gy, torch.zeros_like(gy))
        else:
            gq = g_out[:, t]
        gbar = (gq @ M + c).contiguous()
        xp = tape.qpos[:, t - 1] if t > 0 else last0
        anchor = torch.clamp(xp, lim[:, 0], lim[:, 1]).contiguous()
        proj = None if tape.projected is None else tape.projected[:, t].contiguous()
        gk, _, ga = opt.retarget_batch_vjp(gbar, tape.qpos[:, t].contiguous(), keypoints=kp[:, t].contiguous(),
                                           last_qpos=anchor, projected=proj)
        g_kp[:, t] = gk
        c = ga * ((xp >= lim[:, 0]) & (xp <= lim[:, 1]))
    return g_kp, c, gy


def scatter_matrix(opt, dev):
    """dq/dx [dof, opt_dof] of the scatter + mimic."""
    M = np.zeros((opt.robot.dof, opt.opt_dof), np.float32)
    for j in range(opt.opt_dof):
        q = np.zeros(opt.robot.dof)
        q[opt.idx_pin2target[j]] = 1.0
        if opt.adaptor is not None:
            q = opt.adaptor.forward_qpos(q) - opt.adaptor.forward_qpos(np.zeros(opt.robot.dof))
        M[:, j] = q
    return torch.from_numpy(M).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    T = args.steps
    result = dict(card=card(), steps=T, seconds_per_number=args.seconds, workloads=[])
    for name, key, S in WORKLOADS:
        seq = W.build(key, device=0)
        opt = seq.optimizer
        kp = torch.from_numpy(W.streams(S, T)).to(dev)
        fresh = seq.make_stream_state(S)
        state = seq.make_stream_state(S)
        out = torch.empty((S, T, opt.robot.dof), device=dev)
        status = torch.empty((S, T), dtype=torch.int32, device=dev)
        tape = seq.make_sequence_tape(S, T)

        def reset():
            for k in ("last_qpos", "filter_state", "filter_init", "projected", "damping"):
                if getattr(state, k) is not None:
                    getattr(state, k).copy_(getattr(fresh, k))

        def forward():
            reset()
            seq.retarget_sequences(kp, state, out=out, status_out=status)

        def forward_taped():
            reset()
            seq.retarget_sequences(kp, state, out=out, status_out=status, tape=tape)

        t_fwd, n_fwd = time_calls(forward, args.seconds)
        t_tape, n_tape = time_calls(forward_taped, args.seconds)
        fst = status.cpu().numpy()
        g_out = torch.from_numpy(np.random.RandomState(3).randn(S, T, opt.robot.dof).astype(np.float32)).to(dev)
        vstatus = torch.empty((S, T), dtype=torch.int32, device=dev)
        g_kp = torch.empty((S, T, 21, 3), device=dev)
        g_last, g_filter = torch.empty((S, opt.opt_dof), device=dev), torch.empty((S, opt.robot.dof), device=dev)

        def backward():
            seq.retarget_sequences_vjp(kp, tape, fresh.last_qpos, fresh.filter_init, grad_robot_qpos=g_out,
                                       grad_keypoints_out=g_kp, grad_last_qpos_out=g_last, grad_filter_state_out=g_filter,
                                       status_out=vstatus)

        t_vjp, n_vjp = time_calls(backward, args.seconds)
        li = opt.engine().launch_info()
        lim = torch.from_numpy(np.ascontiguousarray(seq.joint_limits, dtype=np.float32)).to(dev)
        M = scatter_matrix(opt, dev)
        t_loop, n_loop = time_calls(lambda: per_frame_loop(seq, kp, fresh.last_qpos, fresh.filter_init, tape, g_out, lim, M),
                                    args.seconds)
        l_kp, l_last, _ = per_frame_loop(seq, kp, fresh.last_qpos, fresh.filter_init, tape, g_out, lim, M)
        backward()
        torch.cuda.synchronize()
        vs = vstatus.cpu().numpy()
        finite = torch.isfinite(g_kp).all(dim=(2, 3))
        scale = float(l_kp[finite].abs().max()) if bool(finite.any()) else 0.0
        loop_diff = float((g_kp - l_kp)[finite].abs().max()) / max(scale, 1e-30) if bool(finite.any()) else float("nan")
        row = dict(workload=name, key=key, streams=S, steps=T,
                   forward=dict(ms=t_fwd * 1e3, calls=n_fwd), taped_forward=dict(ms=t_tape * 1e3, calls=n_tape),
                   fused_backward=dict(ms=t_vjp * 1e3, calls=n_vjp, grid=li["grid"], block=li["block"], smem_bytes=li["smem_bytes"]),
                   per_frame_loop=dict(ms=t_loop * 1e3, calls=n_loop),
                   taped_over_forward=t_tape / t_fwd, backward_over_forward=t_vjp / t_fwd, loop_over_fused=t_loop / t_vjp,
                   fused_vs_loop_keypoint_rel_diff=loop_diff,
                   forward_status=dict(maxiter=int(((fst >> 24) & 1).sum()), nonfinite=int(((fst >> 25) & 1).sum())),
                   backward_status=dict(not_pd=int(((vs >> 26) & 1).sum()), nonfinite=int(((vs >> 25) & 1).sum()),
                                        frames=int(vs.size)))
        print(name, S, T, "forward %.2f ms  taped %.2f ms  fused backward %.2f ms  per-frame loop %.2f ms  bwd/fwd %.3f  "
              "loop/fused %.2f  NOT_PD %d  NONFINITE %d" % (row["forward"]["ms"], row["taped_forward"]["ms"],
                                                             row["fused_backward"]["ms"], row["per_frame_loop"]["ms"],
                                                             row["backward_over_forward"], row["loop_over_fused"],
                                                             row["backward_status"]["not_pd"],
                                                             row["backward_status"]["nonfinite"]), flush=True)
        result["workloads"].append(row)
        del kp, out, status, tape, g_out, vstatus, g_kp, g_last, g_filter, l_kp, l_last
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)
    print(json.dumps(dict(card=result["card"])))


if __name__ == "__main__":
    main()
