"""Warp sweep of the block-diagonal frames kernel (`dexr_frames_kernel<16, 4, NCW>`, Allegro / LEAP vector retargeting).

    python tools/block_warps_sweep.py [--warps 16,20,24,28] [--repeats 3] [--seconds 1.0]

For every warp count (consumers + producer, passed to the library as DEXR_FRAMES_WARPS, which is read once per process)
a fresh subprocess times the headline shape of bench.py: Vector Allegro, 65 536 frames per launch, 8 rotating seeded input
batches, CUDA events around back-to-back launches for at least `--seconds`.  It also times 4 096 frames (config 2) and
the 0.5-sigma cold start.  The warp counts are run in turn, `--repeats` times, so that slow drift of the clocks shows up as
spread instead of as a difference.  Prints one JSON line per run and a median table; also checks that every warp count
returns the same bits as the first.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

CHILD = r"""
import hashlib, json, os, sys
import torch
sys.path.insert(0, os.path.join(sys.argv[1], "tools"))
sys.path.insert(0, sys.argv[1])
import workloads as W
seconds = float(sys.argv[2])
dev = torch.device("cuda", 0)
seq = W.build(W.METRIC_KEY, device=0)
opt = seq.optimizer
res = {"warps": os.environ["DEXR_FRAMES_WARPS"].split(",")[0]}

def timed(name, n, sigma, sets):
    data = [W.frames(seq, n, W.METRIC_SEED + 1000 * s, sigma=sigma) for s in range(sets)]
    kp = [torch.from_numpy(d[0]).to(dev) for d in data]
    x0 = [torch.from_numpy(d[1]).to(dev) for d in data]
    out = torch.empty((n, opt.opt_dof), dtype=torch.float32, device=dev)
    status = torch.zeros((n,), dtype=torch.int32, device=dev)
    run = lambda s: opt.retarget_batch(keypoints=kp[s % sets], last_qpos=x0[s % sets], out=out, status_out=status)
    for s in range(2 * sets):
        run(s)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(0); e1.record(); torch.cuda.synchronize()
    reps = max(8 * sets, int(seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for s in range(reps):
        run(s)
    e1.record(); torch.cuda.synchronize()
    res[name + "_ms"] = e0.elapsed_time(e1) / reps
    run(0); torch.cuda.synchronize()
    res[name + "_digest"] = hashlib.sha256(out.cpu().numpy().tobytes() + status.cpu().numpy().tobytes()).hexdigest()[:16]
    info = opt.engine().launch_info()
    res[name + "_launch"] = {k: info[k] for k in ("grid", "block", "smem_bytes", "frames_per_tile", "consumer_warps") if k in info}

timed("headline", 65536, 0.05, 8)
timed("config2", 4096, 0.05, 8)
timed("cold", 65536, 0.5, 2)
print(json.dumps(res), flush=True)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warps", default="16,20,24,28")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    warps = [int(w) for w in args.warps.split(",")]
    runs = []
    for _ in range(args.repeats):
        for w in warps:
            env = dict(os.environ, DEXR_FRAMES_WARPS=f"{w},16,16,16")
            p = subprocess.run([sys.executable, "-c", CHILD, str(ROOT), str(args.seconds)], env=env, capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"warps {w}: exit code {p.returncode}")
            rec = json.loads(p.stdout.strip().splitlines()[-1])
            print(json.dumps(rec), flush=True)
            runs.append(rec)
    if args.out:
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in runs))
    print(f"{'warps':>5} {'headline ms':>22} {'4096 ms':>22} {'cold 0.5 ms':>22}  same bits")
    first = {k: v for k, v in runs[0].items() if k.endswith("_digest")}
    for w in warps:
        rs = [r for r in runs if int(r["warps"]) == w]
        cells = []
        for name in ("headline", "config2", "cold"):
            v = [r[name + "_ms"] for r in rs]
            cells.append(f"{statistics.median(v):.4f} ({min(v):.4f}-{max(v):.4f})")
        same = all(r[k] == first[k] for r in rs for k in first)
        print(f"{w:>5} " + " ".join(f"{c:>22}" for c in cells) + f"  {same}")


if __name__ == "__main__":
    main()
