#!/usr/bin/env python
"""Backpropagation through the solve (`dexr_solve_vjp` through Optimizer.retarget_batch_vjp) against the forward solve of the
same frames (`retarget_batch`), on the seeded frames of tools/workloads.py.

  python tools/bench_vjp.py [--frames 65536,1048576] [--seconds 1.0] [--out result.json]

Workloads as in tools/bench_objective.py: Allegro vector (16 lanes), Shadow position (24 + 6 free-flying-base joints = 30,
32 lanes), LEAP DexPilot (16 lanes); the 65 536 seeded frames of each are tiled up to the larger sizes.  The forward solve
runs from the frames' warm starts (DexPilot flags from 0); the VJP runs at its answers with the flags it left and a seeded
cotangent, anchored at the warm starts, keypoints form.  Times are CUDA events around back-to-back launches after warm-up,
at least --seconds of launches per number.  `bytes_per_frame` is what one frame's VJP must move at least (keypoints, qpos,
anchor, cotangent, fixed joints and flags read once; keypoint, anchor and fixed-joint cotangents and the status written),
from the shapes; `hbm_fraction` relates it to the 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM.
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
import workloads as W  # noqa: E402
from bench_objective import HBM_PEAK, WORKLOADS, card, time_it  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="65536,1048576")
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    sizes = [int(s) for s in args.frames.split(",")]
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
            x0 = torch.from_numpy(np.tile(x00, (reps, 1))[:B].copy()).to(dev)
            fixed = None if fixed0 is None else torch.from_numpy(np.tile(fixed0, (reps, 1))[:B].copy()).to(dev)
            gbar = torch.from_numpy(np.random.RandomState(1).randn(B, n).astype(np.float32)).to(dev)
            qout = torch.empty((B, n), device=dev)
            proj = torch.zeros((B, lp), dtype=torch.uint8, device=dev) if lp else None

            def forward():
                if proj is not None:
                    proj.zero_()
                return opt.retarget_batch(None, fixed, x0, keypoints=kp, projected=proj, out=qout)

            t_fwd, calls_fwd = time_it(forward, args.seconds)
            forward()
            flags = None if proj is None else proj.clone()
            status = torch.empty(B, dtype=torch.int32, device=dev)
            g_kp, g_last = torch.empty((B, 21, 3), device=dev), torch.empty((B, n), device=dev)
            g_fixed = torch.empty((B, nf), device=dev) if nf else None

            def backward():
                return opt.retarget_batch_vjp(gbar, qout, None, fixed, x0, keypoints=kp, projected=flags, grad_keypoints_out=g_kp,
                                              grad_fixed_qpos_out=g_fixed, grad_last_qpos_out=g_last, status_out=status)

            t_vjp, calls_vjp = time_it(backward, args.seconds)
            li = opt.engine().launch_info()
            st = status.cpu().numpy()
            bytes_pf = 4 * (2 * 63 + 4 * n + 2 * nf + 1) + lp
            row = dict(workload=name, key=key, frames=B, n_var=n, n_res=m, dummy_range=info["dummy_range"],
                       forward=dict(ms=t_fwd * 1e3, calls=calls_fwd, frames_per_s=B / t_fwd),
                       vjp=dict(ms=t_vjp * 1e3, calls=calls_vjp, frames_per_s=B / t_vjp, bytes_per_frame=bytes_pf,
                                hbm_fraction=bytes_pf * B / t_vjp / HBM_PEAK, grid=li["grid"], block=li["block"],
                                smem_bytes=li["smem_bytes"]),
                       vjp_over_forward=t_vjp / t_fwd,
                       status=dict(ok=int((st == 0).sum()), not_pd=int(((st >> 26) & 1).sum()), nonfinite=int(((st >> 25) & 1).sum())))
            print(name, B, "forward %.3f ms  vjp %.3f ms  vjp/forward %.3f  %.1f %% of HBM peak  grid %d  status %s" % (
                row["forward"]["ms"], row["vjp"]["ms"], row["vjp_over_forward"], 100 * row["vjp"]["hbm_fraction"], li["grid"],
                row["status"]), flush=True)
            result["workloads"].append(row)
            del kp, x0, fixed, gbar, qout, proj, flags, status, g_kp, g_last, g_fixed
            torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)
    print(json.dumps(dict(card=result["card"])))


if __name__ == "__main__":
    main()
