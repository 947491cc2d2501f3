#!/usr/bin/env python
"""Objective evaluation throughput (`dexr_eval_objective` through Optimizer.objective_batch) on the seeded frames of
tools/workloads.py, against the solve of the same frames (`retarget_batch`) in the same run.

  python tools/bench_objective.py [--frames 65536,1048576] [--seconds 1.0] [--ctas 0,1,2] [--out result.json]

Workloads: Allegro vector (block-diagonal robot, 16 lanes), Shadow position (offline YAML: 24 + 6 free-flying-base joints =
30, shipped +-5 m / +-2 pi base range, 32 lanes), LEAP DexPilot (16 lanes).  The 65 536 seeded frames of each are tiled up to
the larger sizes.  Every frame is evaluated at its warm start, anchored at the warm start of the next frame.  Times are CUDA
events around back-to-back launches after warm-up, at least --seconds of launches per number.  `bytes_per_frame` is what one
frame's evaluation must move at least (inputs read once, flags read and written, outputs written), from the shapes;
`hbm_fraction` relates it to the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM.  --ctas: CTAs per SM of the evaluation
kernel (DEXR_EVAL_CTAS_PER_SM; 0 = as many as are resident, the library's choice), for the grid-size measurement.
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import workloads as W  # noqa: E402

HBM_PEAK = 3.35e12
WORKLOADS = [("allegro_vector", W.METRIC_KEY, W.METRIC_SEED), ("shadow_position", W.SHADOW_POS_KEY, W.SHADOW_SEED),
             ("leap_dexpilot", W.LEAP_DEXPILOT_KEY, W.STREAM_SEED)]


def card():
    """Name and enforced power limit of device 0, read in this run (nvidia-smi query; torch's name if that fails)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=limit)
    except Exception:
        return dict(name=torch.cuda.get_device_name(0), power_limit="unknown")


def time_it(fn, seconds):
    """Mean seconds per call over back-to-back calls covering at least `seconds`, after warm-up."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    once = max(a.elapsed_time(b) * 1e-3, 1e-6)
    n = max(5, int(np.ceil(seconds / once)))
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3 / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="65536,1048576")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--ctas", default="0")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    sizes = [int(s) for s in args.frames.split(",")]
    ctas = [int(s) for s in args.ctas.split(",")]
    result = dict(card=card(), hbm_peak_bytes_per_s=HBM_PEAK, seconds_per_number=args.seconds, workloads=[])
    for name, key, seed in WORKLOADS:
        seq = W.build(key, device=0)
        opt = seq.optimizer
        kp0, x00, fixed0, info = W.frames(seq, 65536, seed)
        n, nf, m = opt.opt_dof, len(opt.idx_pin2fixed), opt.num_residuals
        lp = len(opt.projected) if opt.retargeting_type == "DEXPILOT" else 0
        for B in sizes:
            reps = (B + 65535) // 65536
            kp = torch.from_numpy(np.tile(kp0, (reps, 1, 1))[:B].copy()).to(dev)
            x = torch.from_numpy(np.tile(x00, (reps, 1))[:B].copy()).to(dev)
            last = torch.roll(x, 1, 0).contiguous()
            fixed = None if fixed0 is None else torch.from_numpy(np.tile(fixed0, (reps, 1))[:B].copy()).to(dev)
            proj = torch.zeros((B, lp), dtype=torch.uint8, device=dev) if lp else None
            loss, cost = torch.empty(B, device=dev), torch.empty(B, device=dev)
            grad = torch.empty((B, n), device=dev)
            in_bytes = 4 * (3 * 21 + 2 * n + nf) + 2 * lp
            row = dict(workload=name, key=key, frames=B, n_var=n, n_res=m, dummy_range=info["dummy_range"], eval={}, grid={})
            for want in (True, False):
                bytes_pf = in_bytes + 8 + (4 * n if want else 0)
                for c in ctas:
                    if c:
                        os.environ["DEXR_EVAL_CTAS_PER_SM"] = str(c)
                    else:
                        os.environ.pop("DEXR_EVAL_CTAS_PER_SM", None)
                    fn = lambda: opt.objective_batch(x, None, fixed, last, keypoints=kp, projected=proj, loss_out=loss,  # noqa: E731
                                                     cost_out=cost, grad_out=grad if want else None, want_grad=want)
                    t, calls = time_it(fn, args.seconds)
                    li = opt.engine().launch_info()
                    rec = dict(ms=t * 1e3, calls=calls, frames_per_s=B / t, bytes_per_frame=bytes_pf,
                               hbm_fraction=bytes_pf * B / t / HBM_PEAK, grid=li["grid"], block=li["block"])
                    tag = ("grad" if want else "value") + (f"_ctas{c}" if c else "")
                    row["grid" if c else "eval"][tag] = rec
                    print(name, B, tag, "%.3f ms  %.3g frames/s  %.1f %% of HBM peak  grid %d" % (
                        rec["ms"], rec["frames_per_s"], 100 * rec["hbm_fraction"], rec["grid"]), flush=True)
            os.environ.pop("DEXR_EVAL_CTAS_PER_SM", None)
            qout = torch.empty((B, n), device=dev)
            pj = torch.zeros((B, lp), dtype=torch.uint8, device=dev) if lp else None
            t, calls = time_it(lambda: opt.retarget_batch(None, fixed, x, keypoints=kp, projected=pj, out=qout), args.seconds)
            row["solve"] = dict(ms=t * 1e3, calls=calls, frames_per_s=B / t)
            row["eval_grad_over_solve"] = row["eval"]["grad"]["ms"] / row["solve"]["ms"]
            print(name, B, "solve %.3f ms  eval/solve %.3f" % (row["solve"]["ms"], row["eval_grad_over_solve"]), flush=True)
            result["workloads"].append(row)
            del kp, x, last, fixed, proj, loss, cost, grad, qout, pj
            torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)
    print(json.dumps(dict(card=result["card"])))


if __name__ == "__main__":
    main()
