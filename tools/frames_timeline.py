"""Where the frames kernel's warp-time goes: a timeline of one launch of the headline (and of its cold-start arm).

    python tools/frames_timeline.py [--configs static2,queue2,queue3,queue4] [--launches 5] [--out timeline.json]

Runs the experiment library `variants/libdexr_timeline.so` (`python -m dex_retargeting_b200.build --variants`; built here
if missing), whose frames kernel records %globaltimer events into a buffer given with `dexr_exp_timeline()` (layout:
`Timeline` in csrc/dexr.cu).  For each schedule it times `--launches` launches of bench.py's headline shape (Vector
Allegro, 65 536 frames, warm start sigma 0.05) and of the sigma 0.5 cold start, and reports the median launch of:

  launch_us       first warp entry to last warp exit, over the grid
  cta_end_spread  last minus first CTA end (a CTA ends with its last warp), and its share of the launch
  stage_wait      consumer warp-time spent waiting for a stage of the input ring (after the first tile), share
  tail_idle       consumer warp-time from each warp's last frame to the end of the launch, share
  head_idle       consumer warp-time from the launch's start to each warp's first frame, share
  bound           1 - busy / (consumer warps x launch): the share of the launch that no schedule of the same frames on
                  the same warps could beat (time spent solving frames is fixed; everything else is scheduling)
  issued_per_frame  outer iterations the consumer warps ran per frame and group: a warp's iteration count times its
                  groups (32 / lanes per frame) over the frames it solved.  The two frames of a warp run until both are
                  done, so this is the mean over frame pairs of the larger of the two frames' iteration counts.  A frame
                  runs one iteration more than its status word counts when it converges (the iteration whose step meets
                  the tolerance is not counted): compare it with iterations_mean + 1, the frames' own mean.

Schedules (environment switches of the library, read per call): `static<S>` = tiles strided over the CTAs
(DEXR_FRAMES_QUEUE=0), `queue<S>` = the grid-wide queue with shrinking tail tiles; S = input ring stages
(DEXR_FRAMES_STAGES).  `static2` is the schedule before the queue.  The recording adds a few stores per frame pair, so
compare schedules with each other rather than with bench.py's times.  Prints the card, its power limit and SM clock.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

KINDS = {"span": 0, "claim": 1, "stage_wait": 2, "producer_wait": 3, "tile": 4}


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        return {"error": str(e)}


def decode(buf: np.ndarray, ctas: int, events: int) -> list[dict]:
    """Per (CTA, warp) with events: {cta, warp, ev: [n, 4] uint64}."""
    counts = buf[: ctas * 32]
    body = buf[ctas * 32:].reshape(ctas * 32, events, 4)
    out = []
    for slot in np.nonzero(counts)[0]:
        n = int(min(counts[slot], events))
        out.append({"cta": int(slot // 32), "warp": int(slot % 32), "ev": body[slot, :n]})
    return out


def analyse(warps: list[dict], ncw: int, groups: int = 2) -> dict:
    """groups: frames a consumer warp solves at a time (32 / lanes per frame)"""
    spans, cta_end = [], {}
    busy = stage_wait = tail = head = 0
    t_start = min(int(w["ev"][w["ev"][:, 0] >> 32 == 0][0, 2]) for w in warps)
    t_end = max(int(w["ev"][w["ev"][:, 0] >> 32 == 0][0, 3]) for w in warps)
    n_cons = 0
    issued = solved = 0
    for w in warps:
        ev = w["ev"]
        kind = ev[:, 0] >> 32
        span = ev[kind == 0][0]
        cta_end[w["cta"]] = max(cta_end.get(w["cta"], 0), int(span[3]))
        if w["warp"] == ncw:  # the producer
            continue
        n_cons += 1
        claims = ev[kind == 1]
        waits = ev[kind == 2]
        totals = ev[kind == 6]
        if len(totals):
            issued += int(totals[0, 0] & 0xFFFFFFFF) * groups
            solved += int(totals[0, 1])
        busy += int((claims[:, 3] - claims[:, 2]).sum())
        if len(waits) > 1:
            stage_wait += int((waits[1:, 3] - waits[1:, 2]).sum())  # the first wait is the launch's start-up
        if len(claims):
            tail += t_end - int(claims[-1, 3])
            head += int(claims[0, 2]) - t_start
        else:
            tail += t_end - t_start
        spans.append(span)
    launch = t_end - t_start
    total = n_cons * launch
    ends = np.array(sorted(cta_end.values()), dtype=np.float64)
    return {
        "launch_us": launch / 1e3,
        "ctas": len(cta_end),
        "consumer_warps": n_cons,
        "cta_end_spread_us": (ends[-1] - ends[0]) / 1e3,
        "cta_end_spread": (ends[-1] - ends[0]) / launch,
        "stage_wait": stage_wait / total,
        "tail_idle": tail / total,
        "head_idle": head / total,
        "bound": 1.0 - busy / total,
        "issued_per_frame": issued / max(solved, 1),
    }


CHILD = r"""
import ctypes as C, json, os, statistics, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tools"))
import workloads as W
from frames_timeline import decode, analyse
from dex_retargeting_b200 import _native as N
launches, configs = int(sys.argv[2]), sys.argv[3].split(",")
lib = N.load()
lib.dexr_exp_timeline.restype = C.c_int64
lib.dexr_exp_timeline.argtypes = [C.c_void_p]
nbytes = lib.dexr_exp_timeline(None)
CTAS, EVENTS = 256, 128
assert nbytes == CTAS * 32 * (1 + 4 * EVENTS) * 8
dev = torch.device("cuda", 0)
seq = W.build(W.METRIC_KEY, device=0)
opt = seq.optimizer
buf = torch.zeros(nbytes // 8, dtype=torch.int64, device=dev)
B = 65536
arms = {"headline": W.frames(seq, B, W.METRIC_SEED, sigma=0.05), "cold_start": W.frames(seq, B, W.METRIC_SEED, sigma=0.5)}
out = torch.empty((B, opt.opt_dof), dtype=torch.float32, device=dev)
status = torch.zeros((B,), dtype=torch.int32, device=dev)
res = []
for cfg in configs:
    os.environ["DEXR_FRAMES_QUEUE"] = "0" if cfg.startswith("static") else "1"
    os.environ["DEXR_FRAMES_STAGES"] = cfg[-1]
    for arm, d in arms.items():
        kp, x0 = torch.from_numpy(d[0]).to(dev), torch.from_numpy(d[1]).to(dev)
        run = lambda: opt.retarget_batch(keypoints=kp, last_qpos=x0, out=out, status_out=status)
        lib.dexr_exp_timeline(None)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        stats = []
        for _ in range(launches):
            buf.zero_()
            lib.dexr_exp_timeline(C.c_void_p(buf.data_ptr()))
            run()
            torch.cuda.synchronize()
            lib.dexr_exp_timeline(None)
            info = opt.engine().launch_info()
            stats.append(analyse(decode(buf.cpu().numpy().view(np.uint64), CTAS, EVENTS), info["consumer_warps"],
                                 32 // info["lanes_per_frame"]))
        med = sorted(stats, key=lambda s: s["launch_us"])[len(stats) // 2]
        med["launch_us_all"] = [round(s["launch_us"], 2) for s in stats]
        med.update(config=cfg, arm=arm, iterations_mean=float((status.cpu().numpy() & 0xffff).mean()),
                   smem_bytes=info["smem_bytes"], frames_per_tile=info["frames_per_tile"])
        res.append(med)
        print(json.dumps(med), flush=True)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="static2,queue2,queue3,queue4")
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    from dex_retargeting_b200.build import build_library

    lib = build_library(variant="timeline", verbose=False)
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    env = dict(os.environ, DEXR_LIBRARY=str(lib))
    p = subprocess.run([sys.executable, "-c", CHILD, str(ROOT), str(args.launches), args.configs], env=env,
                       capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout + p.stderr)
        raise SystemExit(f"exit code {p.returncode}")
    recs = [json.loads(line) for line in p.stdout.splitlines() if line.startswith("{")]
    for r in recs:
        print(json.dumps(r), flush=True)
    if args.out:
        Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in [{"gpu": info}] + recs))
    print(f"\n{info.get('name', '?')}, power limit {info.get('power.limit', '?')}, SM clock {info.get('clocks.sm', '?')} "
          f"(max {info.get('clocks.max.sm', '?')})")
    print(f"{'arm':<11} {'schedule':<8} {'launch us':>9} {'CTA end spread':>18} {'stage wait':>10} {'tail idle':>9} "
          f"{'head idle':>9} {'bound':>6} {'issued/frame':>12} {'iters/frame + 1':>15}")
    for r in recs:
        print(f"{r['arm']:<11} {r['config']:<8} {r['launch_us']:>9.1f} {r['cta_end_spread_us']:>8.1f} us {100 * r['cta_end_spread']:>5.1f} % "
              f"{100 * r['stage_wait']:>9.1f}% {100 * r['tail_idle']:>8.1f}% {100 * r['head_idle']:>8.1f}% {100 * r['bound']:>5.1f}% {r['issued_per_frame']:>12.2f} {r['iterations_mean'] + 1:>15.2f}")


if __name__ == "__main__":
    main()
