"""The frames kernel's grid-wide tile queue and input ring (DESIGN.md 3.1): where a frame is solved -- which CTA, which tile,
how large the tile, how deep the ring, static striding or the queue -- must not change a bit of its answer or status.
Every check compares a launch against the same frames solved in small batches (2 048 frames: every CTA's first tile
covers the batch, so those launches never touch a queue)."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import workloads as W  # noqa: E402

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SMALL = 2048


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


def _inputs(seq, n, seed, sigma=0.05):
    dev = _dev()
    kp, x0, fixed, _ = W.frames(seq, n, seed, sigma=sigma)
    return (torch.from_numpy(kp).to(dev), torch.from_numpy(x0).to(dev),
            torch.from_numpy(fixed).to(dev) if fixed is not None else None)


def _solve(opt, kp, x0, fixed, stream=None):
    dev = _dev()
    B = kp.shape[0]
    out = torch.empty((B, opt.opt_dof), dtype=torch.float32, device=dev)
    status = torch.zeros((B,), dtype=torch.int32, device=dev)
    kw = {}
    if opt.retargeting_type == "DEXPILOT":
        kw["projected"] = torch.zeros((B, opt._objective_spec().len_proj), dtype=torch.uint8, device=dev)
    opt.retarget_batch(keypoints=kp, last_qpos=x0, fixed_qpos=fixed, out=out, status_out=status, stream=stream, **kw)
    return out, status


def _reference(opt, kp, x0, fixed):
    qs, ss = [], []
    for i in range(0, kp.shape[0], SMALL):
        q, s = _solve(opt, kp[i:i + SMALL], x0[i:i + SMALL], None if fixed is None else fixed[i:i + SMALL])
        qs.append(q)
        ss.append(s)
    torch.cuda.synchronize()
    return torch.cat(qs), torch.cat(ss)


def _assert_same(got, ref):
    q, s = got
    q_ref, s_ref = ref
    assert torch.equal(q, q_ref)
    assert torch.equal(s, s_ref)


@pytest.fixture(scope="module")
def metric():
    seq = W.build(W.METRIC_KEY, device=0)
    kp, x0, fixed = _inputs(seq, 65537, W.METRIC_SEED)
    return seq.optimizer, kp, x0, fixed, _reference(seq.optimizer, kp, x0, fixed)


@pytest.mark.parametrize("schedule", ["queue", "queue-3", "queue-2", "static-2"])
@pytest.mark.parametrize("B", [1, 3, 4095, 4096, 65536, 65537])
def test_batch_sizes(metric, B, schedule, monkeypatch):
    """Headline robot (block-diagonal 16-lane kernel) at batch sizes around the tile and grid boundaries, with the queue
    at every ring depth and with static striding over the parent's two-stage ring."""
    if schedule.startswith("static"):
        monkeypatch.setenv("DEXR_FRAMES_QUEUE", "0")
    if "-" in schedule:
        monkeypatch.setenv("DEXR_FRAMES_STAGES", schedule.split("-")[1])
    opt, kp, x0, fixed, (q_ref, s_ref) = metric
    got = _solve(opt, kp[:B], x0[:B], fixed)
    torch.cuda.synchronize()
    _assert_same(got, (q_ref[:B], s_ref[:B]))


def test_cold_start(monkeypatch):
    """Cold starts (sigma 0.5: more iterations and a wider spread of them per frame) through the queue."""
    seq = W.build(W.METRIC_KEY, device=0)
    kp, x0, fixed = _inputs(seq, 40000, W.METRIC_SEED + 7, sigma=0.5)
    ref = _reference(seq.optimizer, kp, x0, fixed)
    got = _solve(seq.optimizer, kp, x0, fixed)
    torch.cuda.synchronize()
    _assert_same(got, ref)


@pytest.mark.parametrize("key", [W.LEAP_DEXPILOT_KEY, W.SHADOW_POS_KEY, "offline/schunk_svh_hand_right",
                                 "teleop/ability_hand_right"])
def test_other_solver_kinds(key):
    """Dense 16-lane (DexPilot flags), arrow 32-lane, dense 32-lane and mimic robots: batches large enough for the queue,
    with a ragged end."""
    seq = W.build(key, device=0)
    kp, x0, fixed = _inputs(seq, 20001, 900)
    opt = seq.optimizer
    ref = _reference(opt, kp, x0, fixed)
    got = _solve(opt, kp, x0, fixed)
    torch.cuda.synchronize()
    _assert_same(got, ref)


def test_unaligned_pointers(metric):
    """Inputs offset by one float: no tile is 16-byte aligned, the producer stages every tile with plain loads."""
    opt, kp, x0, fixed, (q_ref, s_ref) = metric
    dev = _dev()
    B = 65537
    big_kp = torch.zeros(B * 63 + 1, dtype=torch.float32, device=dev)
    big_x0 = torch.zeros(B * opt.opt_dof + 1, dtype=torch.float32, device=dev)
    big_kp[1:] = kp.reshape(-1)
    big_x0[1:] = x0.reshape(-1)
    got = _solve(opt, big_kp[1:].view(B, 21, 3), big_x0[1:].view(B, opt.opt_dof), fixed)
    torch.cuda.synchronize()
    _assert_same(got, (q_ref, s_ref))


def test_concurrent_streams(metric):
    """One robot launched on three streams at once, eight launches each: more launches in flight than the robot has queue
    slots, so slots are shared over time, and launches that overlap must each get their own."""
    opt, kp, x0, fixed, (q_ref, s_ref) = metric
    streams = [torch.cuda.Stream() for _ in range(3)]
    B = 65536
    cuts = [0, 1000, 30000]  # different batches per stream: a mix-up of two launches' tiles shows
    torch.cuda.synchronize()
    results = []
    for rep in range(8):
        for si, st in enumerate(streams):
            c = cuts[si]
            n = B - c - rep
            with torch.cuda.stream(st):
                results.append((c, n, _solve(opt, kp[c:c + n], x0[c:c + n], fixed, stream=st)))
    torch.cuda.synchronize()
    for c, n, got in results:
        _assert_same(got, (q_ref[c:c + n], s_ref[c:c + n]))


@pytest.mark.parametrize("mode", ["streams", "persistent"])
def test_mixed_call_same_robot_twice(metric, mode, monkeypatch):
    """dexr_solve_frames_multi with the headline robot in two large groups (fork-join: two concurrent queue launches of one
    robot on two side streams; persistent: static striding inside one kernel) next to two other solver kinds."""
    from dex_retargeting_b200.optimizer import retarget_batch_mixed

    monkeypatch.setenv("DEXR_MULTI_MODE", mode)
    opt, kp, x0, fixed, (q_ref, s_ref) = metric
    dev = _dev()
    others = []
    for key, n, seed in ((W.SHADOW_POS_KEY, 3001, 901), (W.LEAP_DEXPILOT_KEY, 12000, 902)):
        seq = W.build(key, device=0)
        k, x, f = _inputs(seq, n, seed)
        others.append((seq.optimizer, k, x, f, _reference(seq.optimizer, k, x, f)))
    jobs, refs = [], []
    for c, n in ((0, 40000), (25000, 40537)):
        jobs.append((opt, dict(keypoints=kp[c:c + n], last_qpos=x0[c:c + n],
                               status_out=torch.zeros((n,), dtype=torch.int32, device=dev))))
        refs.append((q_ref[c:c + n], s_ref[c:c + n]))
    for o, k, x, f, ref in others:
        kw = dict(keypoints=k, last_qpos=x, fixed_qpos=f, status_out=torch.zeros((k.shape[0],), dtype=torch.int32, device=dev))
        if o.retargeting_type == "DEXPILOT":
            kw["projected"] = torch.zeros((k.shape[0], o._objective_spec().len_proj), dtype=torch.uint8, device=dev)
        jobs.append((o, kw))
        refs.append(ref)
    outs = retarget_batch_mixed(jobs)
    torch.cuda.synchronize()
    for q, (_, kw), ref in zip(outs, jobs, refs):
        _assert_same((q, kw["status_out"]), ref)


def test_host_entry(metric):
    """dexr_solve_frames_host: chunks of one call solved on the library's two streams at once."""
    opt, kp, x0, fixed, (q_ref, _) = metric
    out = opt.retarget_batch_host(keypoints=kp.cpu().numpy(), last_qpos=x0.cpu().numpy())
    np.testing.assert_array_equal(out, q_ref.cpu().numpy())
