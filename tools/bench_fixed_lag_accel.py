#!/usr/bin/env python
"""Fixed-lag smoothing with an acceleration penalty (`dexr_fixed_lag_step_accel` through SeqRetargeting.retarget_fixed_lag
on a state made with accel_weight = c) on the workloads of tools/bench_fixed_lag.py: S streams of the recorded trajectory,
K = --ticks frames each, fresh state.  c = 0 is the velocity-only path (`dexr_fixed_lag_step`).

  python tools/bench_fixed_lag_accel.py [--keys leap_dexpilot,allegro_vector,shadow_position] [--cw 0,1,10,100]
                                        [--lags 0,4,8] [--streams 1,256,2048] [--ticks 300] [--seconds 0.3] [--out r.json]

Per workload, c (in units of w = norm_delta), lag L and stream count S:
  tick_ms      per-tick latency: CUDA events around back-to-back K = 1 calls (at least --seconds of them)
  replay_ms    one call of K = --ticks ticks (CUDA events around it, after a warm-up call)
  iters        accepted outer iterations per emitting tick (mean, max) and the fraction of them at max_iters
  quality      from the replay plus a flush (every frame emitted): jitter (mean |second difference| of qpos), fidelity
               (mean per-frame data loss, tools/bench_smooth_accel.py), and mean / max |dq| to the offline accel
               smoother's whole-clip answer at the same c from the same anchor (smooth_packed_sequences)
The card's name and power limit are read in the same run.
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
from bench_fixed_lag import WORKLOADS, event_ms, jitter  # noqa: E402
from bench_objective import card  # noqa: E402
from bench_seq_vjp import time_calls  # noqa: E402
from bench_smooth_accel import fidelity  # noqa: E402

STATUS_MAXITER, STATUS_PENDING = 1 << 24, 1 << 28


def run(seq, S, L, T, cw, seconds):
    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    c = cw * float(opt.params().norm_delta)
    kp = torch.from_numpy(W.streams(S, T)).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((S, T, nf), device=dev) if nf else None
    sub = (lambda t, a, b: None if t is None else t[:, a:b].contiguous())
    r = dict(S=S, L=L, T=T, c_over_w=cw)

    st = seq.make_fixed_lag_state(S, L, accel_weight=c)
    i = [0]

    def tick():
        k = i[0] % T
        i[0] += 1
        seq.retarget_fixed_lag(kp[:, k:k + 1].contiguous(), st, fixed_qpos=sub(fixed, k, k + 1))

    r["tick_ms"] = time_calls(tick, seconds)[0] * 1e3

    seq.retarget_fixed_lag(kp[:, :8].contiguous(), seq.make_fixed_lag_state(S, L, accel_weight=c), fixed_qpos=sub(fixed, 0, 8))
    st = seq.make_fixed_lag_state(S, L, accel_weight=c)
    a0 = st.last_qpos.clone()
    torch.cuda.synchronize()
    r["replay_ms"], (_, q, status) = event_ms(lambda: seq.retarget_fixed_lag(kp, st, fixed_qpos=fixed))
    _, fq, count = seq.flush_fixed_lag(st)
    q, status, fq, count = (x.cpu().numpy() for x in (q, status, fq, count))
    emitted = (status & STATUS_PENDING) == 0
    it = status[emitted] & 0xffff
    r["iters_mean"], r["iters_max"] = float(it.mean()), int(it.max())
    r["maxiter_fraction"] = float(((status[emitted] & STATUS_MAXITER) != 0).mean())

    assert (count == min(L, T)).all()
    fl = np.concatenate([q[:, L:], fq[:, :min(L, T)]], axis=1) if L < T else fq[:, :T]
    layout = seq.pack_streams([T] * S)
    ss = seq.make_stream_state(S)
    ss.last_qpos.copy_(a0)
    tape = seq.make_packed_sequence_tape(layout)
    seq.retarget_packed_sequences(kp.reshape(-1, 21, 3), layout, seq.make_stream_state(S),
                                  fixed_qpos=None if fixed is None else fixed.reshape(-1, nf), tape=tape)
    _, off, _ = seq.smooth_packed_sequences(kp.reshape(-1, 21, 3), layout, ss, qpos_init=tape.qpos,
                                            fixed_qpos=None if fixed is None else fixed.reshape(-1, nf),
                                            accel_weight=c or None)
    off = off.cpu().numpy().reshape(S, T, -1)
    d = np.abs(fl - off)
    r.update(jitter=jitter(fl), offline_jitter=jitter(off), dq_mean=float(d.mean()), dq_max=float(d.max()),
             fidelity=fidelity(seq, kp.reshape(-1, 21, 3), torch.from_numpy(fl.reshape(S * T, -1)).to(dev),
                               None if fixed is None else fixed.reshape(-1, nf), tape.projected))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default=",".join(WORKLOADS))
    ap.add_argument("--cw", default="0,1,10,100")
    ap.add_argument("--lags", default="0,4,8")
    ap.add_argument("--streams", default="1,256,2048")
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=0.3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=card(), rows=[])
    print(json.dumps(res["card"]), flush=True)
    for name in args.keys.split(","):
        seq = W.build(WORKLOADS[name], device=0)
        for S in (int(x) for x in args.streams.split(",")):
            for L in (int(x) for x in args.lags.split(",")):
                for cw in (float(x) for x in args.cw.split(",")):
                    row = dict(workload=name, **run(seq, S, L, args.ticks, cw, args.seconds))
                    res["rows"].append(row)
                    print(json.dumps(row), flush=True)
                    if args.out:
                        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
