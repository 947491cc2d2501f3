#!/usr/bin/env python
"""The acceleration penalty of the offline smoother (`dexr_smooth_sequences_packed_accel` and its `_vjp` through
SeqRetargeting.smooth_packed_sequences(_vjp)(..., accel_weight=c)) on the workloads of tools/bench_smooth.py
(tools/workloads.py `ragged_streams`: clip lengths uniform over [60, 300], fresh state, smoother started from the causal
tape), for c = 0 (the velocity-only smoother) and c = --accel times the robot's norm_delta (the default velocity weight w).

  python tools/bench_smooth_accel.py [--accel 1,10,100] [--seconds 1.0] [--out result.json]

Per workload and c, CUDA events around back-to-back calls after warm-up (at least --seconds of calls per number):
  smooth   the smoother from the causal tape, and its time over the c = 0 smoother's
  vjp      its VJP with seeded cotangents on robot_qpos and qpos
and from one call of each: accepted outer iterations (mean, max) and the fraction of streams at max_iters; NOT_PD streams of
the VJP; jitter, the mean |second difference| of qpos over the clips (DESIGN.md 3.14); fidelity, the mean per-frame data
loss L_t at the answer (Optimizer.objective_batch with norm_delta's term left out, the flags of the causal tape), and the
same two numbers for the causal tape itself.  The card's name and power limit are read in the same run.
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
from bench_smooth import WORKLOADS  # noqa: E402
from smooth_accel_cases import jitter  # noqa: E402

STATUS_MAXITER, STATUS_NOT_PD = 1 << 24, 1 << 26


def fidelity(seq, kp, q, fixed, flags):
    """Mean L_t over the frames: the data loss alone at q [N,opt_dof] (a CUDA tensor), flags [N,len_proj] or None."""
    loss, _, _ = seq.optimizer.objective_batch(q, keypoints=kp, fixed_qpos=fixed,
                                               projected=None if flags is None else flags.clone(), want_grad=False)
    return float(loss.double().mean())


def run_workload(seq, kp_np, lengths, rels, seconds, seed):
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
    offs = np.concatenate([[0], np.cumsum(lengths)])
    first = offs[:-1][lengths > 0]
    nd = float(opt.params().norm_delta)
    rows = dict(causal=dict(jitter=jitter(tape.qpos.cpu().numpy(), offs),
                            fidelity=fidelity(seq, kp, tape.qpos, fixed, tape.projected)))
    base = None
    for rel in [0.0] + list(rels):
        c = rel * nd

        def smooth():
            return seq.smooth_packed_sequences(kp, layout, fresh, fixed_qpos=fixed, qpos_init=tape.qpos, accel_weight=c)

        t_smooth, _ = time_calls(smooth, seconds)
        _, q, status = smooth()
        vst = torch.empty(layout.num_frames, dtype=torch.int32, device=dev)

        def vjp():
            return seq.smooth_packed_sequences_vjp(kp, layout, q, fresh.last_qpos, fresh.projected, gq, grq,
                                                   fixed_qpos=fixed, status_out=vst, accel_weight=c)

        t_vjp, _ = time_calls(vjp, seconds)
        vjp()
        torch.cuda.synchronize()
        st, vs = status.cpu().numpy()[first], vst.cpu().numpy()[first]
        iters = st & 0xffff
        base = t_smooth if base is None else base
        rows[f"c={rel:g}"] = dict(
            accel_weight=c, smooth_ms=t_smooth * 1e3, smooth_over_c0=t_smooth / base, vjp_ms=t_vjp * 1e3,
            iters_mean=float(iters.mean()), iters_max=int(iters.max()),
            at_max_iters=float(((st & STATUS_MAXITER) != 0).mean()), not_pd=int(((vs & STATUS_NOT_PD) != 0).sum()),
            jitter=jitter(q.cpu().numpy(), offs), fidelity=fidelity(seq, kp, q, fixed, tape.projected))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accel", default="1,10,100", help="c in units of the robot's norm_delta, besides c = 0")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rels = [float(v) for v in args.accel.split(",")]
    result = dict(card=card(), workloads={})
    print(result["card"])
    for name, key, S in WORKLOADS:
        seq = W.build(key, device=0)
        kp, lengths = W.ragged_streams(S)
        rows = run_workload(seq, kp, lengths, rels, args.seconds, 1)
        result["workloads"][name] = dict(streams=S, frames=int(lengths.sum()),
                                         norm_delta=float(seq.optimizer.params().norm_delta), **rows)
        print(f"{name:16s} causal tape{'':39s}jitter {rows['causal']['jitter']:.5f}  fidelity "
              f"{rows['causal']['fidelity']:.6f}")
        for arm, r in rows.items():
            if arm == "causal":
                continue
            print(f"{name:16s} {arm:7s} smooth {r['smooth_ms']:8.2f} ms x{r['smooth_over_c0']:.2f}  vjp {r['vjp_ms']:7.2f} ms  "
                  f"iters {r['iters_mean']:.2f}/{r['iters_max']}  at max_iters {r['at_max_iters']:.4f}  "
                  f"NOT_PD {r['not_pd']}/{S}  jitter {r['jitter']:.5f}  fidelity {r['fidelity']:.6f}", flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
