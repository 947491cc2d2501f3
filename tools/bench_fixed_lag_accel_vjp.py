"""Backpropagation through fixed-lag smoothing with an acceleration penalty (`retarget_fixed_lag_accel_vjp`, one
`dexr_fixed_lag_step_accel_vjp` launch) on the three fixed-lag workloads: the cost of recording the tape (a K-tick
`retarget_fixed_lag` on an accelerated state with and without `tape=`, `dexr_fixed_lag_step_accel_tape` against
`dexr_fixed_lag_step_accel`) and the backward's time against the forward's (without a tape), for S streams, lag L, K ticks
and c in units of w = norm_delta.  CUDA events around single calls from the same state, after a warm-up call; `reps` calls
each (default 5), the median and the range reported.  The card's name and power limit are read in the same run.

  python tools/bench_fixed_lag_accel_vjp.py [--keys ...] [--streams 1,256,2048] [--lags 0,4,8] [--cw 1,10] [--ticks 300]
                                            [--reps 5] [--out f]
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
from bench_fixed_lag_vjp import STATUS_NONFINITE, STATUS_NOT_PD, STATUS_PENDING, WORKLOADS, copy_state, event_ms  # noqa: E402
from bench_objective import card  # noqa: E402


def run(seq, S, L, K, cw, reps):
    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    c = cw * float(opt.params().norm_delta)
    kp = torch.from_numpy(W.streams(S, K)).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((S, K, nf), device=dev) if nf else None
    st0 = seq.make_fixed_lag_state(S, L, accel_weight=c)
    tape = seq.make_fixed_lag_tape(S, K, L, accel_weight=c)
    # warm-up of every call at a few ticks
    w = min(K, 8)
    wt = seq.make_fixed_lag_tape(S, w, L, accel_weight=c)
    kw, fw = kp[:, :w].contiguous(), None if fixed is None else fixed[:, :w].contiguous()
    seq.retarget_fixed_lag(kw, copy_state(st0), fixed_qpos=fw)
    seq.retarget_fixed_lag(kw, copy_state(st0), fixed_qpos=fw, tape=wt)
    seq.retarget_fixed_lag_accel_vjp(kw, wt, st0, fixed_qpos=fw, grad_qpos=torch.ones((S, w, opt.opt_dof), device=dev))
    torch.cuda.synchronize()
    fwd, rec, bwd = [], [], []
    for _ in range(reps):
        st = copy_state(st0)
        torch.cuda.synchronize()
        fwd.append(event_ms(lambda: seq.retarget_fixed_lag(kp, st, fixed_qpos=fixed))[0])
        st = copy_state(st0)
        torch.cuda.synchronize()
        t, (_, q, status) = event_ms(lambda: seq.retarget_fixed_lag(kp, st, fixed_qpos=fixed, tape=tape))
        rec.append(t)
    gq = torch.ones_like(q)
    for _ in range(reps):
        t, out = event_ms(lambda: seq.retarget_fixed_lag_accel_vjp(kp, tape, st0, fixed_qpos=fixed, grad_qpos=gq))
        bwd.append(t)
    vstatus = out[6].cpu().numpy()
    emitted = (vstatus & STATUS_PENDING) == 0
    r = dict(S=S, L=L, K=K, c_over_w=cw, forward_ms=float(np.median(fwd)), forward_tape_ms=float(np.median(rec)),
             backward_ms=float(np.median(bwd)))
    r["backward_ms_range"] = [float(min(bwd)), float(max(bwd))]
    r["forward_ms_range"] = [float(min(fwd)), float(max(fwd))]
    r["forward_tape_ms_range"] = [float(min(rec)), float(max(rec))]
    r["tape_cost"] = r["forward_tape_ms"] / r["forward_ms"]
    r["backward_over_forward"] = r["backward_ms"] / r["forward_ms"]  # (the forward without a tape)
    r["tape_mb"] = (tape.qpos.numel() * 4 + (0 if tape.projected is None else tape.projected.numel())) / 1e6
    r["not_pd_ticks"] = int(((vstatus & STATUS_NOT_PD) != 0)[emitted].sum())
    r["nonfinite_ticks"] = int(((vstatus & STATUS_NONFINITE) != 0)[emitted].sum())
    r["emitting_ticks"] = int(emitted.sum())
    r["grad_finite"] = bool(torch.isfinite(out[0]).all())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default=",".join(WORKLOADS))
    ap.add_argument("--lags", default="0,4,8")
    ap.add_argument("--streams", default="1,256,2048")
    ap.add_argument("--cw", default="1,10")
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=card(), rows=[])
    print(json.dumps(res["card"]), flush=True)
    for name in args.keys.split(","):
        seq = W.build(WORKLOADS[name], device=0)
        for S in (int(x) for x in args.streams.split(",")):
            for L in (int(x) for x in args.lags.split(",")):
                for cw in (float(x) for x in args.cw.split(",")):
                    row = dict(workload=name, **run(seq, S, L, args.ticks, cw, args.reps))
                    res["rows"].append(row)
                    print(json.dumps(row), flush=True)
                    torch.cuda.empty_cache()
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
