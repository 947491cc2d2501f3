#!/usr/bin/env bash
# One gpurun call: GPU suite, bench line, launch list + full ncu captures, status dumps.  Writes gpurun_out/job/.
#   gpurun --timeout 1500 -- 'bash tools/gpu_job.sh [suite] [bench] [final] [sanitize] [multisweep] [multitune] [streams256] [tiles] [abprev] ...'
# `final` = the record run (captures, traffic file of this build, bench line, reference arm); then `python tools/collect_profiles.py`.
# `abprev` / `tiles` / `ncuab` / `g16d` / `warps` compare against dex_retargeting_b200/variants/libdexr_prev.so (a library built from the
# previous commit's sources; single-robot entry points only, see _native.py).
set -u
out=gpurun_out/job
mkdir -p "$out"
want() { [ $# -eq 0 ] && return 0; for a in "${ARGS[@]}"; do [ "$a" = "$1" ] && return 0; done; return 1; }
ARGS=("$@"); [ ${#ARGS[@]} -eq 0 ] && ARGS=(suite bench ncu ncu2 dump)
M="smsp__sass_thread_inst_executed_op_ffma_pred_on.sum,smsp__sass_thread_inst_executed_op_fadd_pred_on.sum,smsp__sass_thread_inst_executed_op_fmul_pred_on.sum,smsp__thread_inst_executed.sum"
if want suite; then
  timeout 1500 python -m pytest tests -x -q -m gpu > "$out/pytest_gpu.log" 2>&1; echo "GPU suite: exit $?"; tail -4 "$out/pytest_gpu.log"
fi
if want bench; then
  python bench.py > "$out/bench.json" 2> "$out/bench.err"; echo "bench exit $?"; tail -c 1500 "$out/bench.json"
fi
if want ncu; then
  ncu --metrics gpu__time_duration.sum --clock-control none -c 60 --csv --log-file "$out/launches_bench.csv" \
      python bench.py --steps 5 --warmup 3 --no-cpu-baseline > "$out/ncu_launches.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_frames_kernel -s 4 -c 1 -f -o "$out/prof_frames_allegro" \
      python bench.py --steps 5 --warmup 3 --no-cpu-baseline > "$out/ncu_full.log" 2>&1
  python -c "from dex_retargeting_b200 import _native as N; print(N.build_id())" > "$out/build_id.txt"
fi
if want ncu2; then
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_frames_shadowpos" \
      python tools/profile_targets.py shadow > "$out/ncu_shadow.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_frames_leapdp" \
      python tools/profile_targets.py leapdp > "$out/ncu_leapdp.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_streams_256x300" \
      python tools/profile_targets.py streams > "$out/ncu_streams.log" 2>&1
fi
if want sanitize; then
  for tool in memcheck synccheck; do
    timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tests/tools/sanitize_run.py > "$out/sanitize_$tool.log" 2>&1
    echo "$tool exit $?"; grep -E "ERROR SUMMARY|ok " "$out/sanitize_$tool.log" | tail -24
  done
fi
du -sh "$out" 2>/dev/null
if want dump; then
  python tests/tools/dump_status.py "$out/status_default.npz" 2>&1 | tee "$out/dump_default.log"
fi
if want streams256; then
  python - <<'PY'
import sys, torch
sys.path.insert(0, "tools")
import workloads as W
dev = torch.device("cuda", 0)
seq = W.build(W.LEAP_DEXPILOT_KEY, device=0)
for S in (64, 256, 1024, 2048, 4096):
    tk = torch.from_numpy(W.streams(max(S, 2048), 300)[:S] if S <= 2048 else __import__("numpy").concatenate([W.streams(2048, 300)] * 2)).to(dev)
    seq.retarget_sequences(tk)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        seq.retarget_sequences(tk)
    e1.record(); torch.cuda.synchronize()
    print(f"streams {S:5d} x 300: {e0.elapsed_time(e1) / 3:.3f} ms  launch {seq.optimizer.engine().launch_info()}")
PY
fi
if want multisweep; then
  python tools/multi_sweep.py 2>&1 | tee "$out/multi_sweep.txt"
fi
if want multitune; then
  python tools/multi_tune.py 2>&1 | tee "$out/multi_tune.txt"
fi
if want final; then
  # the record run: captures first, then the traffic file of THIS build, then the bench line that reads it
  BID=$(python -c "from dex_retargeting_b200 import _native as N; print(N.build_id())")
  ncu --metrics gpu__time_duration.sum --clock-control none -c 80 --csv --log-file "$out/launches_bench.csv" \
      python bench.py --steps 5 --warmup 3 --no-cpu-baseline > "$out/ncu_launches.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_frames_kernel -s 4 -c 1 -f -o "$out/prof_frames_allegro" \
      python bench.py --steps 5 --warmup 3 --no-cpu-baseline --no-configs > "$out/ncu_full.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_frames_shadowpos" python tools/profile_targets.py shadow > "$out/ncu_shadow.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_frames_leapdp" python tools/profile_targets.py leapdp > "$out/ncu_leapdp.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_streams_256x300" python tools/profile_targets.py streams > "$out/ncu_streams.log" 2>&1
  ncu --set full --metrics "$M" --clock-control none --import-source on -k regex:dexr_ -s 1 -c 1 -f -o "$out/prof_streams_2048x300" python tools/profile_targets.py streams2048 > "$out/ncu_streams2048.log" 2>&1
  python tools/make_traffic.py "$out" profiles/roofline_traffic.json "$BID" && cp profiles/roofline_traffic.json "$out/roofline_traffic.json"
  nvidia-smi --query-gpu=index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap --format=csv -lms 200 > "$out/clocks.csv" &
  SMI=$!
  python bench.py > "$out/bench.json" 2> "$out/bench.err"; echo "bench exit $?"
  python bench.py --impl reference > "$out/bench_reference.json" 2> "$out/bench_reference.err"; echo "reference arm exit $?"
  kill $SMI
  du -sh "$out"
fi
if want abprev; then
  for n in default prev; do
    if [ $n = prev ]; then export DEXR_LIBRARY=$PWD/dex_retargeting_b200/variants/libdexr_prev.so; else unset DEXR_LIBRARY; fi
    python bench.py --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_$n.json" 2> "$out/bench_$n.err"
  done
  unset DEXR_LIBRARY
  python - <<'PY'
import json
for n in ("default", "prev"):
    try:
        d = json.loads(open(f"gpurun_out/job/bench_{n}.json").read().strip().splitlines()[-1])
        print(f"{n:8s} headline {d['value']:.4e} sustained {d['sustained']['value']:.4e} | " + " | ".join(f"{r['name'][:22]} {r['ms_per_step']:.4f}" for r in d["configs"]))
    except Exception as e:
        print(n, "FAILED", e)
PY
fi
if want ncuab; then
  for n in default prev; do
    if [ $n = prev ]; then export DEXR_LIBRARY=$PWD/dex_retargeting_b200/variants/libdexr_prev.so; else unset DEXR_LIBRARY; fi
    ncu --set full --clock-control none -k regex:dexr_ -s 1 -c 1 -f -o "$out/ab_leapdp_$n" python tools/profile_targets.py leapdp > "$out/ncu_ab_$n.log" 2>&1
    python tools/ncu_summary.py "$out/ab_leapdp_$n.ncu-rep" "$out/ab_leapdp_$n.md" "$n" > /dev/null 2>&1
    grep -E "time_duration|inst_executed.sum |issue_active|bank_conflicts|wavefronts_mem_shared" "$out/ab_leapdp_$n.md" | sed "s/^/$n /"
    sed -n '/warp stall/,/instructions by pipe/p' "$out/ab_leapdp_$n.md" | head -16 | sed "s/^/$n /"
  done
  unset DEXR_LIBRARY
fi
if want g16d; then
  for w in 16 12; do
    DEXR_G16D_WARPS=$w python - <<'PY'
import os, sys, torch
sys.path.insert(0, "tools")
import workloads as W
dev = torch.device("cuda", 0)
for key, seed in ((W.LEAP_DEXPILOT_KEY, W.SHADOW_SEED), ("teleop/ability_hand_right", 303), ("teleop/inspire_hand_right", 305)):
    seq = W.build(key, device=0)
    kp, x0, f, _ = W.frames(seq, 65536, seed)
    k, x = torch.from_numpy(kp).to(dev), torch.from_numpy(x0).to(dev)
    ff = torch.from_numpy(f).to(dev) if f is not None else None
    out = torch.empty((65536, seq.optimizer.opt_dof), dtype=torch.float32, device=dev)
    for _ in range(3):
        seq.optimizer.retarget_batch(keypoints=k, last_qpos=x, fixed_qpos=ff, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        seq.optimizer.retarget_batch(keypoints=k, last_qpos=x, fixed_qpos=ff, out=out)
    e1.record(); torch.cuda.synchronize()
    print(f"warps {os.environ['DEXR_G16D_WARPS']}  {key:36s} {e0.elapsed_time(e1) / 10:.4f} ms  {seq.optimizer.engine().launch_info()['block']} threads")
PY
  done
fi
if want warps; then
  for cfg in 16,16,16,16 20,14,14,14 24,12,12,12; do  # (block diagonal: 16 | 20 | 24, the other kinds 16 | 14 | 12)
    DEXR_FRAMES_WARPS=$cfg python - <<'PY'
import os, sys, torch
sys.path.insert(0, "tools")
import workloads as W
dev = torch.device("cuda", 0)
cases = [("block16 allegro vector", W.METRIC_KEY, W.METRIC_SEED, {}), ("dense16 leap dexpilot", W.LEAP_DEXPILOT_KEY, W.SHADOW_SEED, {}),
         ("dense16 ability (mimic)", "teleop/ability_hand_right", 303, {}), ("arrow32 shadow position", W.SHADOW_POS_KEY, W.SHADOW_SEED, dict(narrow_dummy=True)),
         ("arrow32 shadow vector", "teleop/shadow_hand_right", 301, {}), ("dense32 svh (mimic)", "teleop/schunk_svh_hand_right", 304, {})]
for name, key, seed, kw in cases:
    seq = W.build(key, device=0)
    sets = []
    for s in range(4):
        kp, x0, f, _ = W.frames(seq, 65536, seed + 1000 * s, **kw)
        sets.append((torch.from_numpy(kp).to(dev), torch.from_numpy(x0).to(dev), torch.from_numpy(f).to(dev) if f is not None else None))
    out = torch.empty((65536, seq.optimizer.opt_dof), dtype=torch.float32, device=dev)
    for i in range(4):
        seq.optimizer.retarget_batch(keypoints=sets[i][0], last_qpos=sets[i][1], fixed_qpos=sets[i][2], out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(12):
        k, x, f = sets[i % 4]
        seq.optimizer.retarget_batch(keypoints=k, last_qpos=x, fixed_qpos=f, out=out)
    e1.record(); torch.cuda.synchronize()
    print(f"warps {os.environ['DEXR_FRAMES_WARPS']:12s} {name:28s} {e0.elapsed_time(e1) / 12:.4f} ms  ({seq.optimizer.engine().launch_info()['block']} threads)")
PY
  done 2>&1 | tee "$out/warps_sweep.txt"
fi
if want tiles; then
  for n in default prev; do
    if [ $n = prev ]; then export DEXR_LIBRARY=$PWD/dex_retargeting_b200/variants/libdexr_prev.so; else unset DEXR_LIBRARY; fi
    python - <<'PY'
import os, sys, torch
sys.path.insert(0, "tools")
import workloads as W
dev = torch.device("cuda", 0)
tag = "prev" if os.environ.get("DEXR_LIBRARY") else "new "
for key, seed, kw in ((W.SHADOW_POS_KEY, W.SHADOW_SEED, dict(narrow_dummy=True)), (W.METRIC_KEY, W.METRIC_SEED, {}), (W.LEAP_DEXPILOT_KEY, W.SHADOW_SEED, {})):
    seq = W.build(key, device=0)
    for B in (int(x) for x in os.environ.get("DEXR_TILE_SIZES", "2048,8192,16384,32768").split(",")):
        kp, x0, f, _ = W.frames(seq, B, seed, **kw)
        k, x = torch.from_numpy(kp).to(dev), torch.from_numpy(x0).to(dev)
        out = torch.empty((B, seq.optimizer.opt_dof), dtype=torch.float32, device=dev)
        for _ in range(3):
            seq.optimizer.retarget_batch(keypoints=k, last_qpos=x, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            seq.optimizer.retarget_batch(keypoints=k, last_qpos=x, out=out)
        e1.record(); torch.cuda.synchronize()
        print(f"{tag} {key:34s} B {B:6d}: {e0.elapsed_time(e1) / 20:.4f} ms  tile {seq.optimizer.engine().launch_info()['frames_per_tile']}")
PY
  done
  unset DEXR_LIBRARY
fi
