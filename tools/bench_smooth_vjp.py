#!/usr/bin/env python
"""Backpropagation through the offline smoother (`dexr_smooth_sequences_packed_vjp` through
SeqRetargeting.smooth_packed_sequences_vjp) against the smoother's forward and the causal packed VJP, on the workloads of
tools/bench_smooth.py (tools/workloads.py `ragged_streams`: clip lengths uniform over [60, 300], fresh state).

  python tools/bench_smooth_vjp.py [--seconds 1.0] [--out result.json]

Per workload and arm, CUDA events around back-to-back calls after warm-up (at least --seconds of calls per number):
  smooth      the smoother from the causal tape (the forward)
  vjp         its VJP with seeded cotangents on robot_qpos and qpos
  causal_vjp  the causal packed VJP (dexr_solve_sequences_packed_vjp) of the tape, for scale
and from one VJP call: streams NOT_PD, and NOT_PD among the streams the forward left at max_iters.  Arm "dropped" repeats it
with 5 % of the frames set to NaN in bursts of 1-10 frames.  Workloads: LEAP DexPilot and Allegro vector with 2048 clips,
Shadow position with 512.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))
import workloads as W  # noqa: E402
from bench_objective import card  # noqa: E402
from bench_seq_vjp import time_calls  # noqa: E402
from bench_smooth import WORKLOADS, drop_bursts  # noqa: E402

STATUS_MAXITER, STATUS_NOT_PD = 1 << 24, 1 << 26


def run_arm(seq, kp_np, lengths, seconds, seed):
    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    layout = seq.pack_streams(lengths)
    S = len(lengths)
    kp = torch.from_numpy(kp_np).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((layout.num_frames, nf), device=dev) if nf else None
    fresh = seq.make_stream_state(S)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(kp, layout, seq.make_stream_state(S), fixed_qpos=fixed, tape=tape)
    gen = torch.Generator(device=dev).manual_seed(seed)
    grq = torch.randn((layout.num_frames, opt.robot.dof), device=dev, generator=gen)
    gq = torch.randn((layout.num_frames, opt.opt_dof), device=dev, generator=gen)

    def smooth():
        return seq.smooth_packed_sequences(kp, layout, fresh, fixed_qpos=fixed, qpos_init=tape.qpos)

    t_smooth, _ = time_calls(smooth, seconds)
    _, q, status = smooth()
    vst = torch.empty(layout.num_frames, dtype=torch.int32, device=dev)

    def vjp():
        return seq.smooth_packed_sequences_vjp(kp, layout, q, fresh.last_qpos, fresh.projected, gq, grq, fixed_qpos=fixed,
                                               status_out=vst)

    def causal_vjp():
        return seq.retarget_packed_sequences_vjp(kp, layout, tape, fresh.last_qpos, fresh.filter_init, grad_robot_qpos=grq,
                                                 fixed_qpos=fixed)

    t_vjp, calls = time_calls(vjp, seconds)
    t_causal, _ = time_calls(causal_vjp, seconds)
    vjp()
    torch.cuda.synchronize()
    status, vst = status.cpu().numpy(), vst.cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(lengths)])[:-1][lengths > 0]
    maxit = (status[offs] & STATUS_MAXITER) != 0
    npd = (vst[offs] & STATUS_NOT_PD) != 0
    return dict(smooth_ms=t_smooth * 1e3, vjp_ms=t_vjp * 1e3, vjp_over_smooth=t_vjp / t_smooth,
                causal_vjp_ms=t_causal * 1e3, calls=calls, streams=int(len(offs)), not_pd=int(npd.sum()),
                at_max_iters=int(maxit.sum()), not_pd_at_max_iters=int((npd & maxit).sum()),
                nonfinite=int(((vst[offs] >> 25) & 1).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = dict(card=card(), workloads={})
    print(result["card"])
    for name, key, S in WORKLOADS:
        seq = W.build(key, device=0)
        kp, lengths = W.ragged_streams(S)
        rows = dict(clean=run_arm(seq, kp, lengths, args.seconds, 1))
        kp_d = kp.copy()
        kp_d[drop_bursts(lengths, 0.05, 2)] = np.nan
        rows["dropped"] = run_arm(seq, kp_d, lengths, args.seconds, 3)
        result["workloads"][name] = dict(streams=S, frames=int(lengths.sum()), **rows)
        for arm, r in rows.items():
            print(f"{name:16s} {arm:8s} smooth {r['smooth_ms']:8.2f} ms  vjp {r['vjp_ms']:7.2f} ms  "
                  f"vjp/smooth {r['vjp_over_smooth']:.3f}  causal vjp {r['causal_vjp_ms']:7.2f} ms  "
                  f"NOT_PD {r['not_pd']}/{r['streams']}  (at max_iters {r['not_pd_at_max_iters']}/{r['at_max_iters']})  "
                  f"nonfinite {r['nonfinite']}", flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
