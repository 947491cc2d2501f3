#!/usr/bin/env python
"""Fixed-lag smoothing of live streams (`dexr_fixed_lag_step` through SeqRetargeting.retarget_fixed_lag) against the causal
stream solve (`retarget_sequences`) on the same frames: S streams of the recorded trajectory (tools/workloads.py `streams`,
each stream with its own 2 mm keypoint offsets), fresh state.

  python tools/bench_fixed_lag.py [--keys leap_dexpilot,allegro_vector,shadow_position] [--lags 0,4,8,16]
                                  [--streams 1,256,2048] [--ticks 300] [--seconds 0.5] [--out result.json]

Per workload, lag L and stream count S:
  tick_ms     per-tick latency: CUDA events around back-to-back K = 1 calls (at least --seconds of them), the streams
              running on through the recorded frames; causal_ms the same for retarget_sequences with T = 1
  replay_ms   one call of K = --ticks ticks (CUDA events around it, after a warm-up call), and causal_replay_ms for
              retarget_sequences over the same T = --ticks frames
  iters       accepted outer iterations per emitting tick (mean, max) and the fraction of ticks at max_iters, from the
              replay (its status words)
  quality     from the replay plus a flush (every frame emitted): mean and max |dq| to the offline smoother's answer on
              the whole clip from the same anchor (smooth_packed_sequences), and the jitter, the mean |second difference|
              of qpos; the same two figures for the causal path's unfiltered qpos (its tape).
The card's name and power limit are read in the same run.  Large S x L on Shadow position takes minutes per replay.
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
from bench_seq_vjp import time_calls  # noqa: E402

WORKLOADS = {"leap_dexpilot": W.LEAP_DEXPILOT_KEY, "allegro_vector": W.METRIC_KEY, "shadow_position": W.SHADOW_POS_KEY}
STATUS_MAXITER, STATUS_PENDING = 1 << 24, 1 << 28


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def jitter(q):
    """Mean |x_{t+1} - 2 x_t + x_{t-1}| over streams, frames and joints: q [S,T,n]."""
    return float(np.abs(q[:, 2:] - 2 * q[:, 1:-1] + q[:, :-2]).mean())


def run(seq, S, L, T, seconds):
    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    kp_np = W.streams(S, T)
    kp = torch.from_numpy(kp_np).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((S, T, nf), device=dev) if nf else None
    r = dict(S=S, L=L, T=T)

    # per-tick latency: the streams run on through the frames, one tick per call
    st = seq.make_fixed_lag_state(S, L)
    i = [0]

    def tick():
        k = i[0] % T
        i[0] += 1
        seq.retarget_fixed_lag(kp[:, k:k + 1].contiguous(), st,
                               fixed_qpos=None if fixed is None else fixed[:, k:k + 1].contiguous())

    r["tick_ms"] = time_calls(tick, seconds)[0] * 1e3
    cs = seq.make_stream_state(S)
    j = [0]

    def causal_tick():
        k = j[0] % T
        j[0] += 1
        seq.retarget_sequences(kp[:, k:k + 1].contiguous(), cs,
                               fixed_qpos=None if fixed is None else fixed[:, k:k + 1].contiguous())

    r["causal_ms"] = time_calls(causal_tick, seconds)[0] * 1e3

    # replay: K = T ticks in one launch, from a fresh state (after a warm-up call)
    seq.retarget_fixed_lag(kp[:, :8].contiguous(), seq.make_fixed_lag_state(S, L),
                           fixed_qpos=None if fixed is None else fixed[:, :8].contiguous())
    st = seq.make_fixed_lag_state(S, L)
    torch.cuda.synchronize()
    r["replay_ms"], (_, q, status) = event_ms(lambda: seq.retarget_fixed_lag(kp, st, fixed_qpos=fixed))
    _, fq, count = seq.flush_fixed_lag(st)
    tape = seq.make_sequence_tape(S, T)
    seq.retarget_sequences(kp[:, :8].contiguous(), seq.make_stream_state(S),
                           fixed_qpos=None if fixed is None else fixed[:, :8].contiguous())
    cs = seq.make_stream_state(S)
    torch.cuda.synchronize()
    r["causal_replay_ms"], _ = event_ms(lambda: seq.retarget_sequences(kp, cs, fixed_qpos=fixed, tape=tape))
    q, status, fq, count = (x.cpu().numpy() for x in (q, status, fq, count))
    emitted = (status & STATUS_PENDING) == 0
    it = status[emitted] & 0xffff
    r["iters_mean"], r["iters_max"] = float(it.mean()), int(it.max())
    r["maxiter_fraction"] = float(((status[emitted] & STATUS_MAXITER) != 0).mean())

    # quality against the offline smoother on the whole clip, from the same (fresh) anchor
    assert (count == min(L, T)).all()
    fl = np.concatenate([q[:, L:], fq[:, :min(L, T)]], axis=1) if L < T else fq[:, :T]
    layout = seq.pack_streams([T] * S)
    _, off, _ = seq.smooth_packed_sequences(kp.reshape(-1, 21, 3), layout, seq.make_stream_state(S),
                                            fixed_qpos=None if fixed is None else fixed.reshape(-1, nf))
    off = off.cpu().numpy().reshape(S, T, -1)
    causal = tape.qpos.cpu().numpy()
    d, dc = np.abs(fl - off), np.abs(causal - off)
    r.update(dq_mean=float(d.mean()), dq_max=float(d.max()), jitter=jitter(fl), causal_dq_mean=float(dc.mean()),
             causal_dq_max=float(dc.max()), causal_jitter=jitter(causal), offline_jitter=jitter(off))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default=",".join(WORKLOADS))
    ap.add_argument("--lags", default="0,4,8,16")
    ap.add_argument("--streams", default="1,256,2048")
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = dict(card=card(), rows=[])
    print(json.dumps(res["card"]), flush=True)
    for name in args.keys.split(","):
        seq = W.build(WORKLOADS[name], device=0)
        for S in (int(x) for x in args.streams.split(",")):
            for L in (int(x) for x in args.lags.split(",")):
                row = dict(workload=name, **run(seq, S, L, args.ticks, args.seconds))
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
