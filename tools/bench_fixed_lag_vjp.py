"""Backpropagation through fixed-lag smoothing (`retarget_fixed_lag_vjp`, one `dexr_fixed_lag_step_vjp` launch) on the
three fixed-lag workloads: the cost of recording the tape (a K-tick `retarget_fixed_lag` with and without `tape=`) and the
backward's time against the forward's (without a tape), for S streams, lag L and K ticks.  CUDA events around single
calls from the same state, after a warm-up call; `reps` calls each (default 5), the median and the range reported.  The
card's name and power limit are read in the same run.

  python tools/bench_fixed_lag_vjp.py [--keys ...] [--streams 1,256,2048] [--lags 0,4,16] [--ticks 300] [--reps 5] [--out f]
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
from bench_objective import card  # noqa: E402

WORKLOADS = {"leap_dexpilot": W.LEAP_DEXPILOT_KEY, "allegro_vector": W.METRIC_KEY, "shadow_position": W.SHADOW_POS_KEY}
STATUS_NOT_PD, STATUS_NONFINITE, STATUS_PENDING = 1 << 26, 1 << 25, 1 << 28


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def copy_state(st):
    from dex_retargeting_b200.objective import _fixed_lag_copy

    return _fixed_lag_copy(st)


def run(seq, S, L, K, reps):
    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    kp = torch.from_numpy(W.streams(S, K)).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((S, K, nf), device=dev) if nf else None
    st0 = seq.make_fixed_lag_state(S, L)
    tape = seq.make_fixed_lag_tape(S, K, L)
    # warm-up of every call at a few ticks
    w = min(K, 8)
    wt = seq.make_fixed_lag_tape(S, w, L)
    ws0 = copy_state(st0)
    seq.retarget_fixed_lag(kp[:, :w].contiguous(), copy_state(st0), fixed_qpos=None if fixed is None else fixed[:, :w].contiguous())
    seq.retarget_fixed_lag(kp[:, :w].contiguous(), copy_state(st0), tape=wt,
                           fixed_qpos=None if fixed is None else fixed[:, :w].contiguous())
    seq.retarget_fixed_lag_vjp(kp[:, :w].contiguous(), wt, ws0, fixed_qpos=None if fixed is None else fixed[:, :w].contiguous(),
                               grad_qpos=torch.ones((S, w, opt.opt_dof), device=dev))
    torch.cuda.synchronize()
    fwd, rec, bwd = [], [], []  # (single calls; the median over `reps`, and the spread kept)
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
        t, out = event_ms(lambda: seq.retarget_fixed_lag_vjp(kp, tape, st0, fixed_qpos=fixed, grad_qpos=gq))
        bwd.append(t)
    vstatus = out[-1].cpu().numpy()
    emitted = (vstatus & STATUS_PENDING) == 0
    r = dict(S=S, L=L, K=K, forward_ms=float(np.median(fwd)), forward_tape_ms=float(np.median(rec)),
             backward_ms=float(np.median(bwd)))
    r["backward_ms_range"] = [float(min(bwd)), float(max(bwd))]
    r["forward_ms_range"] = [float(min(fwd)), float(max(fwd))]
    r["tape_cost"] = r["forward_tape_ms"] / r["forward_ms"]
    r["backward_over_forward"] = r["backward_ms"] / r["forward_ms"]  # (the forward without a tape)
    r["tape_mb"] = tape.qpos.numel() * 4 / 1e6
    r["not_pd_ticks"] = int(((vstatus & STATUS_NOT_PD) != 0)[emitted].sum())
    r["nonfinite_ticks"] = int(((vstatus & STATUS_NONFINITE) != 0)[emitted].sum())
    r["emitting_ticks"] = int(emitted.sum())
    r["grad_finite"] = bool(torch.isfinite(out[0]).all())
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default=",".join(WORKLOADS))
    ap.add_argument("--lags", default="0,4,16")
    ap.add_argument("--streams", default="1,256,2048")
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
                row = dict(workload=name, **run(seq, S, L, args.ticks, args.reps))
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
