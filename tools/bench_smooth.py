#!/usr/bin/env python
"""Offline smoothing of recorded clips (`dexr_smooth_sequences_packed` through SeqRetargeting.smooth_packed_sequences) against
the causal taped solve it starts from, on the packed-stream workloads (tools/workloads.py `ragged_streams`: clip lengths
uniform over [60, 300], fresh state).

  python tools/bench_smooth.py [--seconds 1.0] [--polish 6] [--out result.json]

Per workload and arm, CUDA events around back-to-back calls after warm-up (at least --seconds of calls per number):
  causal   the taped packed solve (dexr_solve_sequences_packed with a tape), the smoother's usual starting point
  smooth   the smoother from that tape
and from one smoothing call: outer iterations (mean, max), rejected trials, streams at max_iters, the relative drop of
F = sum of the per-frame costs + the smoothness terms from the causal trajectory to the smoothed one (float64), and the
float64 polish displacement (tests/smooth_cases.py) on --polish sampled clips.  Arm "dropped" repeats it with 5 % of the
frames set to NaN in bursts of 1-10 frames.  Workloads: LEAP DexPilot and Allegro vector with 2048 clips, Shadow position with
512.  The card's name and power limit are read in the same run.
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

WORKLOADS = [("leap_dexpilot", W.LEAP_DEXPILOT_KEY, 2048), ("allegro_vector", W.METRIC_KEY, 2048),
             ("shadow_position", W.SHADOW_POS_KEY, 512)]
STATUS_MAXITER = 1 << 24


def drop_bursts(lengths, frac, seed):
    """Frame indices (packed) dropped in bursts of 1-10 frames until `frac` of the frames are gone."""
    rng = np.random.RandomState(seed)
    N = int(lengths.sum())
    mask = np.zeros(N, bool)
    while mask.mean() < frac:
        start, n = rng.randint(0, N), rng.randint(1, 11)
        mask[start:start + n] = True
    return np.flatnonzero(mask)


def run_arm(seq, o, kp_np, lengths, seconds, n_polish, seed):
    import smooth_cases as SMC

    dev = torch.device("cuda", 0)
    opt = seq.optimizer
    layout = seq.pack_streams(lengths)
    S = len(lengths)
    kp = torch.from_numpy(kp_np).to(dev)
    nf = len(opt.idx_pin2fixed)
    fixed = torch.zeros((layout.num_frames, nf), device=dev) if nf else None
    fresh = seq.make_stream_state(S)
    tape = seq.make_packed_sequence_tape(layout)

    def causal():
        st = seq.make_stream_state(S)
        return seq.retarget_packed_sequences(kp, layout, st, fixed_qpos=fixed, tape=tape)

    def smooth():
        return seq.smooth_packed_sequences(kp, layout, fresh, fixed_qpos=fixed, qpos_init=tape.qpos)

    t_causal, _ = time_calls(causal, seconds)
    causal()
    t_smooth, calls = time_calls(smooth, seconds)
    rq, q, status = smooth()
    torch.cuda.synchronize()
    q, status, tq = q.cpu().numpy(), status.cpu().numpy(), tape.qpos.cpu().numpy()
    tp = None if tape.projected is None else tape.projected.cpu().numpy()
    offs = np.concatenate([[0], np.cumsum(lengths)])
    first = status[offs[:-1][lengths > 0]]
    iters, rejects = first & 0xffff, (first >> 16) & 0x7f
    rng = np.random.RandomState(seed)
    anch = SMC.clipped_anchor(o, fresh.last_qpos.cpu().numpy())
    nd = float(opt.params().norm_delta)
    drops, moves = [], []
    for s in rng.choice(S, n_polish, replace=False):
        a, b = offs[s], offs[s + 1]
        m = SMC.Model(o, kp_np[a:b], None if fixed is None else np.zeros((b - a, nf)), None if tp is None else tp[a:b],
                      anch[s], nd)
        f0, f1 = m.value(tq[a:b]), m.value(q[a:b])
        drops.append((f0 - f1) / f0)
        moves.append(float(np.abs(m.polish(q[a:b]) - q[a:b]).max()))
    return dict(causal_ms=t_causal * 1e3, smooth_ms=t_smooth * 1e3, smooth_over_causal=t_smooth / t_causal, calls=calls,
                iters_mean=float(iters.mean()), iters_max=int(iters.max()), rejects_mean=float(rejects.mean()),
                at_max_iters=int(((first & STATUS_MAXITER) != 0).sum()), sampled_F_drop=drops,
                polish_move_max=max(moves) if moves else None, missing_frames=int(((status >> 27) & 1).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--polish", type=int, default=6)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from helpers import build_oracle

    result = dict(card=card(), workloads={})
    print(result["card"])
    for name, key, S in WORKLOADS:
        seq, o = W.build(key, device=0), build_oracle(key)
        kp, lengths = W.ragged_streams(S)
        rows = dict(clean=run_arm(seq, o, kp, lengths, args.seconds, args.polish, 1))
        kp_d = kp.copy()
        kp_d[drop_bursts(lengths, 0.05, 2)] = np.nan
        rows["dropped"] = run_arm(seq, o, kp_d, lengths, args.seconds, args.polish, 3)
        result["workloads"][name] = dict(streams=S, frames=int(lengths.sum()), **rows)
        for arm, r in rows.items():
            print(f"{name:16s} {arm:8s} causal {r['causal_ms']:8.2f} ms  smooth {r['smooth_ms']:8.2f} ms  "
                  f"x{r['smooth_over_causal']:.2f}  iters {r['iters_mean']:.2f}/{r['iters_max']}  rejects "
                  f"{r['rejects_mean']:.2f}  at max_iters {r['at_max_iters']}  F drop "
                  f"{np.mean(r['sampled_F_drop']) if r['sampled_F_drop'] else float('nan'):.4f}  polish move {r['polish_move_max']}  "
                  f"missing {r['missing_frames']}",
                  flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
