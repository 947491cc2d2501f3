#!/usr/bin/env python
"""Per-frame Jacobians of the solve (`dexr_solve_jacobian` through Optimizer.retarget_batch_jacobian) against the forward
solve, one VJP and the loop of n = opt_dof `retarget_batch_vjp` launches with the unit cotangents e_i (what a caller had
to run for J before), on the seeded frames of tools/workloads.py.

  python tools/bench_jacobian.py [--frames 65536] [--seconds 1.0] [--out result.json]

Workloads as in tools/bench_vjp.py: Allegro vector (n = 16), Shadow position (n = 30), LEAP DexPilot (n = 16).  The forward
solve runs from the frames' warm starts (DexPilot flags from 0); the VJP, the Jacobian and the loop run at its answers with
the flags it left, anchored at the warm starts, keypoints form.  Times are CUDA events around back-to-back calls after
warm-up, at least --seconds of calls per number.  `bytes_per_frame` is what one frame's Jacobian must move at least: its
inputs read once (keypoints, qpos, anchor, fixed joints, flags), the n x 63 keypoint block, the n x n anchor block, the
n x n_fixed fixed-joint block and the status written.  `max_row_diff` is the worst |Jacobian row - VJP of e_i|_inf over all
frames and rows, relative to that row's |.|_inf.
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
    ap.add_argument("--frames", type=int, default=65536)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    B = args.frames
    result = dict(card=card(), hbm_peak_bytes_per_s=HBM_PEAK, seconds_per_number=args.seconds, frames=B, workloads=[])
    for name, key, seed in WORKLOADS:
        seq = W.build(key, device=0)
        opt = seq.optimizer
        kp0, x00, fixed0, info = W.frames(seq, 65536, seed)
        n, nf, m = opt.opt_dof, len(opt.idx_pin2fixed), opt.num_residuals
        lp = len(opt.projected) if opt.retargeting_type == "DEXPILOT" else 0
        reps = (B + 65535) // 65536
        kp = torch.from_numpy(np.tile(kp0, (reps, 1, 1))[:B].copy()).to(dev)
        x0 = torch.from_numpy(np.tile(x00, (reps, 1))[:B].copy()).to(dev)
        fixed = None if fixed0 is None else torch.from_numpy(np.tile(fixed0, (reps, 1))[:B].copy()).to(dev)
        qout = torch.empty((B, n), device=dev)
        proj = torch.zeros((B, lp), dtype=torch.uint8, device=dev) if lp else None

        def forward():
            if proj is not None:
                proj.zero_()
            return opt.retarget_batch(None, fixed, x0, keypoints=kp, projected=proj, out=qout)

        t_fwd, _ = time_it(forward, args.seconds)
        forward()
        flags = None if proj is None else proj.clone()
        status = torch.empty(B, dtype=torch.int32, device=dev)
        j_kp, j_last = torch.empty((B, n, 21, 3), device=dev), torch.empty((B, n, n), device=dev)
        j_fixed = torch.empty((B, n, nf), device=dev) if nf else None
        eye = torch.eye(n, device=dev)
        gbar = torch.from_numpy(np.random.RandomState(1).randn(B, n).astype(np.float32)).to(dev)
        units = [eye[i].expand(B, n).contiguous() for i in range(n)]
        g_kp, g_last = torch.empty((n, B, 21, 3), device=dev), torch.empty((n, B, n), device=dev)
        g_fixed = torch.empty((n, B, nf), device=dev) if nf else None
        vst = torch.empty(B, dtype=torch.int32, device=dev)

        def vjp(g, i=0):
            return opt.retarget_batch_vjp(g, qout, None, fixed, x0, keypoints=kp, projected=flags, grad_keypoints_out=g_kp[i],
                                          grad_fixed_qpos_out=None if g_fixed is None else g_fixed[i],
                                          grad_last_qpos_out=g_last[i], status_out=vst)

        def jacobian():
            return opt.retarget_batch_jacobian(qout, None, fixed, x0, keypoints=kp, projected=flags, jac_keypoints_out=j_kp,
                                               jac_fixed_qpos_out=j_fixed, jac_last_qpos_out=j_last, status_out=status)

        def vjp_loop():
            for i in range(n):
                vjp(units[i], i)

        t_vjp, _ = time_it(lambda: vjp(gbar), args.seconds)
        t_jac, calls_jac = time_it(jacobian, args.seconds)
        t_loop, _ = time_it(vjp_loop, args.seconds)
        jacobian()
        vjp_loop()
        torch.cuda.synchronize()
        # Jacobian rows against the loop, per frame and row, in units of the row's |.|_inf (one block at a time)
        worst = 0.0
        for a, b in ((j_kp, g_kp.transpose(0, 1)), (j_last, g_last.transpose(0, 1)),
                     (j_fixed, None if g_fixed is None else g_fixed.transpose(0, 1))):
            if a is None:
                continue
            d = (a - b).abs().flatten(2).amax(2)
            s = b.abs().flatten(2).amax(2)
            worst = max(worst, float(torch.where(s > 0, d / s.clamp_min(1e-30), d).max()))
        st = status.cpu().numpy()
        same_status = bool(np.array_equal(st, vst.cpu().numpy()))
        li = opt.engine().launch_info()
        bytes_pf = 4 * (63 + 2 * n + nf + 1) + lp + 4 * (n * 63 + n * n + n * nf)
        row = dict(workload=name, key=key, frames=B, n_var=n, n_res=m, dummy_range=info["dummy_range"],
                   forward_ms=t_fwd * 1e3, vjp_ms=t_vjp * 1e3, jacobian_ms=t_jac * 1e3, vjp_loop_ms=t_loop * 1e3,
                   jacobian_calls=calls_jac, loop_over_jacobian=t_loop / t_jac, jacobian_over_forward=t_jac / t_fwd,
                   bytes_per_frame=bytes_pf, hbm_fraction=bytes_pf * B / t_jac / HBM_PEAK, grid=li["grid"],
                   block=li["block"], smem_bytes=li["smem_bytes"], max_row_diff=worst, statuses_match_vjp=same_status,
                   status=dict(ok=int((st == 0).sum()), not_pd=int(((st >> 26) & 1).sum()),
                               nonfinite=int(((st >> 25) & 1).sum())))
        print(name, B, "forward %.3f ms  vjp %.3f ms  jacobian %.3f ms  loop of %d vjps %.3f ms  loop/jacobian %.2f  "
              "%.1f %% of HBM peak  max row diff %.2e  status %s" % (
                  row["forward_ms"], row["vjp_ms"], row["jacobian_ms"], n, row["vjp_loop_ms"], row["loop_over_jacobian"],
                  100 * row["hbm_fraction"], worst, row["status"]), flush=True)
        result["workloads"].append(row)
        del kp, x0, fixed, qout, proj, flags, status, j_kp, j_last, j_fixed, units, g_kp, g_last, g_fixed, vst, gbar
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)
    print(json.dumps(dict(card=result["card"])))


if __name__ == "__main__":
    main()
