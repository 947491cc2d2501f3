#!/usr/bin/env python
"""Packed streams of different lengths (`dexr_solve_sequences_packed`, `dexr_solve_sequences_packed_vjp`) against the ways
the rectangular calls can serve the same clips, on seeded ragged workloads (tools/workloads.py `ragged_streams`: clip lengths
uniform over [60, 300], each clip the first frames of the recorded trajectory with a 2 mm per-stream offset, fresh state).

  python tools/bench_packed_streams.py [--seconds 1.0] [--equal-steps 180] [--out result.json]

Per workload, CUDA events around back-to-back calls after warm-up, at least --seconds of calls per number; the stream
state is reset before every call.  Arms:
  1 packed        one packed launch, the clips in the workload's order (streams are dealt to warps in index order)
  2 longest_first the same clips packed longest first (the dealing order a load balancer would pick; the digest is taken
                  after putting the rows back in the workload's order)
  3 equal         packed with every length = --equal-steps, against dexr_solve_sequences on the same [S,T] data
  4 padded        one rectangular launch padded to the longest clip (the last frame repeated)
  5 per_length    one rectangular launch per distinct clip length
  6 taped / vjp   taped packed forward and packed backward against the rectangular ones at equal lengths
Every arm prints a digest of the frames it solved (packed order; padding dropped), so equal digests mean equal bits.
Workloads: LEAP DexPilot and Allegro vector with 2048 clips, Shadow position with 512.
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

WORKLOADS = [("leap_dexpilot", W.LEAP_DEXPILOT_KEY, 2048), ("allegro_vector", W.METRIC_KEY, 2048),
             ("shadow_position", W.SHADOW_POS_KEY, 512)]


class Resettable:
    """A stream state and the fresh copy it is reset from before every timed call."""

    def __init__(self, seq, S):
        self.fresh, self.state = seq.make_stream_state(S), seq.make_stream_state(S)

    def reset(self):
        for k in ("last_qpos", "filter_state", "filter_init", "projected", "damping"):
            if getattr(self.state, k) is not None:
                getattr(self.state, k).copy_(getattr(self.fresh, k))


def digest(t):
    return W.digest(t.detach().cpu().numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--equal-steps", type=int, default=180)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    result = dict(card=card(), seconds_per_number=args.seconds, equal_steps=args.equal_steps, workloads=[])
    print(json.dumps(dict(card=result["card"])), flush=True)
    for name, key, S in WORKLOADS:
        seq = W.build(key, device=0)
        opt = seq.optimizer
        dof = opt.robot.dof
        kp_np, lengths = W.ragged_streams(S)
        kp = torch.from_numpy(kp_np).to(dev)
        layout = seq.pack_streams(lengths)
        N_ = layout.num_frames
        offsets = np.concatenate([[0], np.cumsum(lengths)])
        row = dict(workload=name, key=key, streams=S, frames=N_, mean_len=float(lengths.mean()), max_len=int(lengths.max()))
        st = Resettable(seq, S)
        out = torch.empty((N_, dof), device=dev)
        perm = np.argsort(-lengths, kind="stable")
        rows_lf = torch.from_numpy(np.concatenate([offsets[s] + np.arange(lengths[s]) for s in perm])).to(dev)
        kp_lf = kp[rows_lf].contiguous()
        layout_lf = seq.pack_streams(lengths[perm])
        st_lf = Resettable(seq, S)
        out_lf = torch.empty_like(out)

        def packed():
            st.reset()
            seq.retarget_packed_sequences(kp, layout, st.state, out=out)

        def longest_first():
            st_lf.reset()
            seq.retarget_packed_sequences(kp_lf, layout_lf, st_lf.state, out=out_lf)

        arms = {}
        t, n = time_calls(packed, args.seconds)
        packed()
        arms["1_packed"] = dict(ms=t * 1e3, calls=n, digest=digest(out))
        t, n = time_calls(longest_first, args.seconds)
        longest_first()
        back = torch.empty_like(out_lf)
        back[rows_lf] = out_lf
        arms["2_longest_first"] = dict(ms=t * 1e3, calls=n, digest=digest(back))

        # 4: padded to the longest clip (last frame repeated), outputs cut back to each clip
        Tm = int(lengths.max())
        idx = np.concatenate([offsets[s] + np.minimum(np.arange(Tm), lengths[s] - 1) for s in range(S)])
        kp_pad = kp[torch.from_numpy(idx).to(dev)].reshape(S, Tm, 21, 3).contiguous()
        out_pad = torch.empty((S, Tm, dof), device=dev)

        def padded():
            st.reset()
            seq.retarget_sequences(kp_pad, st.state, out=out_pad)

        t, n = time_calls(padded, args.seconds)
        padded()
        keep = torch.from_numpy(np.concatenate([s * Tm + np.arange(lengths[s]) for s in range(S)])).to(dev)
        arms["4_padded"] = dict(ms=t * 1e3, calls=n, digest=digest(out_pad.reshape(-1, dof)[keep]))

        # 5: one rectangular call per distinct length
        groups = []
        for L in np.unique(lengths):
            ss = np.nonzero(lengths == L)[0]
            rows = np.concatenate([offsets[s] + np.arange(L) for s in ss])
            groups.append((ss, torch.from_numpy(rows).to(dev), kp[torch.from_numpy(rows).to(dev)].reshape(len(ss), int(L), 21, 3)
                           .contiguous(), Resettable(seq, len(ss)), torch.empty((len(ss), int(L), dof), device=dev)))

        def per_length():
            for _, _, k, r, o in groups:
                r.reset()
                seq.retarget_sequences(k, r.state, out=o)

        t, n = time_calls(per_length, args.seconds)
        per_length()
        gathered = torch.empty_like(out)
        for _, rows, _, _, o in groups:
            gathered[rows] = o.reshape(-1, dof)
        arms["5_per_length"] = dict(ms=t * 1e3, calls=n, launches=len(groups), digest=digest(gathered))

        # 3 and 6: every clip T frames, packed against rectangular
        T = args.equal_steps
        kp_eq = torch.from_numpy(W.streams(S, T)).to(dev)
        eq_layout = seq.pack_streams(np.full(S, T))
        kp_eq_p = kp_eq.reshape(S * T, 21, 3)
        out_eq = torch.empty((S, T, dof), device=dev)
        out_eq_p = torch.empty((S * T, dof), device=dev)

        def rect():
            st.reset()
            seq.retarget_sequences(kp_eq, st.state, out=out_eq)

        def rect_packed():
            st.reset()
            seq.retarget_packed_sequences(kp_eq_p, eq_layout, st.state, out=out_eq_p)

        t_r, n_r = time_calls(rect, args.seconds)
        rect()
        d_r = digest(out_eq)
        t_p, n_p = time_calls(rect_packed, args.seconds)
        rect_packed()
        arms["3_equal"] = dict(rect_ms=t_r * 1e3, packed_ms=t_p * 1e3, packed_over_rect=t_p / t_r, rect_digest=d_r,
                               packed_digest=digest(out_eq_p), calls=(n_r, n_p))

        tape = seq.make_sequence_tape(S, T)
        tape_p = seq.make_packed_sequence_tape(eq_layout)

        def rect_taped():
            st.reset()
            seq.retarget_sequences(kp_eq, st.state, out=out_eq, tape=tape)

        def packed_taped():
            st.reset()
            seq.retarget_packed_sequences(kp_eq_p, eq_layout, st.state, out=out_eq_p, tape=tape_p)

        t_rt, _ = time_calls(rect_taped, args.seconds)
        t_pt, _ = time_calls(packed_taped, args.seconds)
        g_out = torch.from_numpy(np.random.RandomState(3).randn(S, T, dof).astype(np.float32)).to(dev)
        g_kp, g_kp_p = torch.empty((S, T, 21, 3), device=dev), torch.empty((S * T, 21, 3), device=dev)
        f = st.fresh

        def rect_vjp():
            seq.retarget_sequences_vjp(kp_eq, tape, f.last_qpos, f.filter_init, grad_robot_qpos=g_out, grad_keypoints_out=g_kp)

        def packed_vjp():
            seq.retarget_packed_sequences_vjp(kp_eq_p, eq_layout, tape_p, f.last_qpos, f.filter_init,
                                              grad_robot_qpos=g_out.reshape(S * T, dof), grad_keypoints_out=g_kp_p)

        t_rv, _ = time_calls(rect_vjp, args.seconds)
        t_pv, _ = time_calls(packed_vjp, args.seconds)
        rect_vjp()
        packed_vjp()
        arms["6_taped_and_vjp"] = dict(rect_taped_ms=t_rt * 1e3, packed_taped_ms=t_pt * 1e3, rect_vjp_ms=t_rv * 1e3,
                                       packed_vjp_ms=t_pv * 1e3, tape_digests=(digest(tape.qpos), digest(tape_p.qpos)),
                                       vjp_digests=(digest(g_kp), digest(g_kp_p)))
        row["arms"] = arms
        row["longest_first_over_packed"] = arms["2_longest_first"]["ms"] / arms["1_packed"]["ms"]
        row["padded_over_packed"] = arms["4_padded"]["ms"] / arms["1_packed"]["ms"]
        row["per_length_over_packed"] = arms["5_per_length"]["ms"] / arms["1_packed"]["ms"]
        print(json.dumps(row), flush=True)
        result["workloads"].append(row)
        del kp, out, kp_lf, out_lf, back, kp_pad, out_pad, groups, gathered, kp_eq, out_eq, out_eq_p, tape, tape_p, g_out, g_kp, g_kp_p
        torch.cuda.empty_cache()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
