#!/usr/bin/env python
"""Small end-to-end exercise of every kernel for compute-sanitizer (memcheck / racecheck / synccheck):
frames kernel (G=16 dense, G=16 block, G=32 arrow / dense, mimic), fused preprocessing, sequences kernel (two half-warps per
stream, one half-warp per stream, several streams per warp), the mixed-robot call (fork-join and persistent), the host-buffer
call (pinned zero-copy and pageable staged), the preprocessing kernel, ragged batch sizes; and the evaluation, VJP,
Jacobian, sequence-VJP, packed-stream and smoothing calls on a robot with fixed joints (fixed_dense16) and on the largest
32-lane robot (dof31_vector) of tests/structure_cases.py.

  compute-sanitizer --tool memcheck python tests/tools/sanitize_run.py [--derivatives-only]"""
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from helpers import build_product, keypoint_trajectory  # noqa: E402
from dex_retargeting_b200.preprocess import preprocess_keypoints  # noqa: E402

dev = torch.device("cuda", 0)
kp = keypoint_trajectory()


def derivative_calls(cid):
    """One call of every derivative, evaluation and smoothing entry point on structure case `cid`."""
    import tempfile

    import structure_cases as SC

    seq, _ = SC.build(SC.BY_ID[cid], Path(tempfile.mkdtemp()))
    opt = seq.optimizer
    n, nf, dof = opt.opt_dof, len(opt.idx_pin2fixed), opt.robot.dof
    mid = seq.joint_limits.mean(1).astype(np.float32)

    def fixed(*shape):
        return torch.zeros(shape + (nf,), device=dev) if nf else None

    B = 37
    k = torch.from_numpy(kp[:B * 3:3].copy()).to(dev)
    x0 = torch.from_numpy(np.tile(mid, (B, 1))).to(dev)
    q = opt.retarget_batch(keypoints=k, last_qpos=x0, fixed_qpos=fixed(B), clip_init=True)
    loss, cost, grad = opt.objective_batch(q, None, fixed(B), x0, keypoints=k)
    vjp = opt.retarget_batch_vjp(torch.ones((B, n), device=dev), q, fixed_qpos=fixed(B), last_qpos=x0, keypoints=k)
    jac = opt.retarget_batch_jacobian(q, fixed_qpos=fixed(B), last_qpos=x0, keypoints=k)
    S, T = 3, 5
    tk = torch.from_numpy(np.stack([kp[40 * s:40 * s + T] for s in range(S)]).copy()).to(dev)
    st = seq.make_stream_state(S)
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    tape = seq.make_sequence_tape(S, T)
    out, _ = seq.retarget_sequences(tk, st, fixed_qpos=fixed(S, T), tape=tape)
    svjp = seq.retarget_sequences_vjp(tk, tape, last0, finit0, grad_robot_qpos=torch.ones((S, T, dof), device=dev),
                                      fixed_qpos=fixed(S, T))
    lengths = [4, 0, 1, 6]
    N = sum(lengths)
    layout = seq.pack_streams(lengths)
    pk = torch.from_numpy(kp[:N].copy()).to(dev)
    st = seq.make_stream_state(len(lengths))
    last0, finit0 = st.last_qpos.clone(), st.filter_init.clone()
    ptape = seq.make_packed_sequence_tape(layout)
    pout, _ = seq.retarget_packed_sequences(pk, layout, st, fixed_qpos=fixed(N), tape=ptape)
    pvjp = seq.retarget_packed_sequences_vjp(pk, layout, ptape, last0, finit0, grad_robot_qpos=torch.ones((N, dof), device=dev),
                                             fixed_qpos=fixed(N))
    rq, qs, status = seq.smooth_packed_sequences(pk, layout, seq.make_stream_state(len(lengths)), fixed_qpos=fixed(N))
    torch.cuda.synchronize()
    sums = [float(t.abs().sum()) for t in (q, loss, cost, grad, *vjp, *jac, out, *svjp, pout, *pvjp, rq, qs)
            if t is not None]
    print(cid, "derivative calls ok", sum(sums))


if "--derivatives-only" in sys.argv:
    for cid in ("fixed_dense16", "dof31_vector"):
        derivative_calls(cid)
    sys.exit(0)

for key, B in (("teleop/allegro_hand_right", 37), ("teleop/leap_hand_right_dexpilot", 64), ("offline/shadow_hand_right", 21),
               ("teleop/schunk_svh_hand_right", 33), ("offline/panda_gripper", 9)):
    seq = build_product(key)
    opt = seq.optimizer
    k = torch.from_numpy(kp[:B * 3:3].copy()).to(dev)
    x0 = torch.from_numpy(np.tile(seq.joint_limits.mean(1).astype(np.float32), (B, 1))).to(dev)
    proj = torch.zeros((B, opt._objective_spec().len_proj), dtype=torch.uint8, device=dev) if opt.retargeting_type == "DEXPILOT" else None
    q = opt.retarget_batch(keypoints=k, last_qpos=x0, projected=proj, clip_init=True)
    torch.cuda.synchronize()
    print(key, "frames ok", float(q.abs().sum()))
for key in ("teleop/allegro_hand_right", "teleop/shadow_hand_right_dexpilot"):
    seq = build_product(key)
    tk = torch.from_numpy(np.stack([kp[0:16], kp[100:116], kp[300:316]]).copy()).to(dev)
    out, st = seq.retarget_sequences(tk)
    torch.cuda.synchronize()
    print(key, "sequences ok", float(out.abs().sum()))
raw = torch.from_numpy(kp[:300].copy()).to(dev) + 0.1
out = preprocess_keypoints(raw)
torch.cuda.synchronize()
print("preprocess ok", float(out.abs().sum()))

# ---- round 2 additions -------------------------------------------------------------------------------------------------
from dex_retargeting_b200.optimizer import retarget_batch_mixed  # noqa: E402

seq = build_product("teleop/allegro_hand_right")
opt = seq.optimizer
B = 45
rawk = torch.from_numpy(kp[:B].copy()).to(dev) + 0.05
x0 = torch.from_numpy(np.tile(seq.joint_limits.mean(1).astype(np.float32), (B, 1))).to(dev)
q = opt.retarget_batch(keypoints=rawk, last_qpos=x0, raw_hand="Right")
torch.cuda.synchronize()
print("fused preprocess ok", float(q.abs().sum()))

seq = build_product("teleop/leap_hand_right_dexpilot")
for duo, S, T in (("1", 5, 12), ("0", 5, 12), ("1", 132 * 8 + 37, 3)):
    os.environ["DEXR_SEQ_DUO"] = duo
    tk = torch.from_numpy(np.stack([kp[(7 * s) % 400:(7 * s) % 400 + T] for s in range(S)]).copy()).to(dev)
    out, st = seq.retarget_sequences(tk)
    torch.cuda.synchronize()
    print(f"sequences duo={duo} S={S} ok", float(out.abs().sum()))
os.environ.pop("DEXR_SEQ_DUO")

for mode in ("streams", "persistent"):
    os.environ["DEXR_MULTI_MODE"] = mode
    jobs = []
    for i, key in enumerate(("teleop/allegro_hand_right", "offline/shadow_hand_right", "teleop/leap_hand_right_dexpilot",
                             "teleop/schunk_svh_hand_right")):
        s_ = build_product(key)
        o_ = s_.optimizer
        n = 19 + 7 * i
        job = dict(keypoints=torch.from_numpy(kp[i:i + n].copy()).to(dev),
                   last_qpos=torch.from_numpy(np.tile(s_.joint_limits.mean(1).astype(np.float32), (n, 1))).to(dev), clip_init=True)
        if o_.retargeting_type == "DEXPILOT":
            job["projected"] = torch.zeros((n, o_._objective_spec().len_proj), dtype=torch.uint8, device=dev)
        jobs.append((o_, job))
    outs = retarget_batch_mixed(jobs)
    torch.cuda.synchronize()
    print(f"mixed {mode} ok", sum(float(o.abs().sum()) for o in outs))
os.environ.pop("DEXR_MULTI_MODE")

seq = build_product("teleop/allegro_hand_right")
opt = seq.optimizer
B = 300
x0h = np.tile(seq.joint_limits.mean(1).astype(np.float32), (B, 1))
o1 = opt.retarget_batch_host(keypoints=torch.from_numpy(kp[:B].copy()).pin_memory(), last_qpos=torch.from_numpy(x0h).pin_memory(),
                             out=torch.empty((B, opt.opt_dof)).pin_memory())
o2 = opt.retarget_batch_host(keypoints=kp[:B].copy(), last_qpos=x0h)
torch.cuda.synchronize()
print("host call ok", float(np.abs(np.asarray(o1) - np.asarray(o2)).max()))

for cid in ("fixed_dense16", "dof31_vector"):
    derivative_calls(cid)
