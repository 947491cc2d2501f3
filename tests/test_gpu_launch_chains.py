"""Chains of frames launches, each reading what the launch before it wrote, with nothing between them on the stream -- how a
batched teleop loop calls retarget_batch once per tick: the previous tick's `out` is the next `last_qpos`, the carried
damping and the DexPilot flags are updated in place.

The single-robot frames kernel is launched with programmatic dependent launch (dexr.cu, grid_dep_launch): the next launch
on the stream may start while this one still solves, and is correct only because it reads its inputs, the damping, the
flags and the queue after grid_dep_wait().  So every chain here is built to expose a read that moves in front of that wait:
  - every output buffer is allocated before the chain and poisoned (NaN answers, zero statuses): a read of q_(t-1) before
    launch t-1 wrote it is a non-finite start (status bit 25) and a NaN answer;
  - tail links: a CTA's first tile is its own static tile, so launch t+1's first tiles read what launch t solved first,
    long ago.  A link that takes the next launch's streams as the LAST B' of the previous launch's (views: no kernel
    between the calls) makes it read what the previous launch wrote last, in the tail of its tile queue;
  - batches large enough that the grid-wide queue is in use, under the queue, static striding and a two-stage ring.
The references: the same calls serialised (DEXR_FRAMES_PDL=0 and a synchronise after every call) bit for bit, the
sequences kernel (the same recurrence in registers) bit for bit, and the float64 oracle on teacher-forced frames."""
import sys
from pathlib import Path

import numpy as np
import pytest

import structure_cases as SC
from helpers import build_oracle

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import workloads as W  # noqa: E402

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

TOL = 1e-4  # rad, BASELINE.json north_star tolerance
NONFINITE = 1 << 25
HEADLINE_B = 65537
OTHER_B = 20001
# every chain: full links, then a link into the tail of a queue launch, and tail links of the no-queue launches after it
HEADLINE_LINKS = [HEADLINE_B, HEADLINE_B, 40000, 4096, 4096, 1000, 3]
OTHER_LINKS = [OTHER_B, OTHER_B, 12000, 4096, 1000, 1000, 3]
# test_chain_matches_sequences_kernel / test_chain_matches_oracle_teacher_forced: streams and steps per robot
SEQ_S, SEQ_T = 20001, 8
ORACLE_S = {W.METRIC_KEY: HEADLINE_B, W.LEAP_DEXPILOT_KEY: OTHER_B}
ORACLE_T = 60


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


class Inputs:
    """Per-step targets of S streams, [T,S,...] on the device (so that a step's tail of streams is a contiguous slice), the
    fixed joints [T,S,n_fixed] or None, and the mid-range start [S,opt_dof]."""

    def __init__(self, opt, targets, arg, fixed, mid):
        dev = _dev()
        self.opt, self.arg = opt, arg
        self.targets = torch.from_numpy(np.ascontiguousarray(targets, dtype=np.float32)).to(dev)
        self.fixed = None if fixed is None else torch.from_numpy(np.ascontiguousarray(fixed, dtype=np.float32)).to(dev)
        self.x0 = torch.from_numpy(np.tile(np.asarray(mid, np.float32), (self.targets.shape[1], 1))).to(dev)

    def step(self, t, first):
        kw = {self.arg: self.targets[t, first:]}
        if self.fixed is not None:
            kw["fixed_qpos"] = self.fixed[t, first:]
        return kw


def _fixed(opt, shape, seed):
    lim = opt.robot.kin.joint_limits[opt.idx_pin2fixed]
    return np.random.RandomState(seed).uniform(lim[:, 0], lim[:, 1], size=shape + (len(lim),))


def stream_inputs(seq, S, T, seed=W.STREAM_SEED):
    """The first T recorded frames, every stream with its own offsets (workloads.streams), as keypoints."""
    opt = seq.optimizer
    kp = W.streams(S, T, seed).transpose(1, 0, 2, 3)
    fixed = _fixed(opt, (T, S), seed) if len(opt.idx_pin2fixed) else None
    return Inputs(opt, kp, "keypoints", fixed, seq.joint_limits.mean(1))


def case_inputs(case, tmp_path, S, T, seed=11):
    """A synthetic robot of tests/structure_cases.py: every step of every stream draws one of 256 warm-start problems
    (targets and fixed joints), so consecutive steps of a stream are unrelated targets."""
    seq, o = SC.build(case, tmp_path)
    refs, fixed, _ = SC.problems(o, 256, seed=seed)
    pick = np.random.RandomState(seed).randint(0, 256, size=(T, S))
    nf = fixed.shape[1]
    return Inputs(seq.optimizer, refs[pick], "ref_value", fixed[pick] if nf else None, seq.joint_limits.mean(1))


def _poisoned(opt, sizes):
    dev = _dev()
    qs = [torch.full((b, opt.opt_dof), float("nan"), dtype=torch.float32, device=dev) for b in sizes]
    ss = [torch.zeros((b,), dtype=torch.int32, device=dev) for b in sizes]
    return qs, ss


def _state(opt, S):
    dev = _dev()
    lp = opt._objective_spec().len_proj if opt.retargeting_type == "DEXPILOT" else 0
    return (torch.zeros((S,), dtype=torch.float32, device=dev),
            torch.zeros((S, lp), dtype=torch.uint8, device=dev) if lp else None)


class ChainRun:
    """One chain of retarget_batch calls: step t solves the last sizes[t] streams, starting from the previous step's answer
    (step 0: the mid-range pose), with the streams' damping and flags carried in place.  A step smaller than the one before
    is a tail link: its inputs are views of the last sizes[t] rows of the previous step's buffers."""

    def __init__(self, inp, sizes):
        self.inp, self.sizes = inp, list(sizes)
        self.S = inp.targets.shape[1]
        assert self.sizes[0] == self.S and all(a >= b for a, b in zip(self.sizes, self.sizes[1:]))
        self.qs, self.ss = _poisoned(inp.opt, self.sizes)
        self.damping, self.projected = _state(inp.opt, self.S)
        self.t = 0
        self.last, self.d, self.p = inp.x0, self.damping, self.projected

    def step(self, stream=None):
        t, b = self.t, self.sizes[self.t]
        cut = self.last.shape[0] - b
        if cut:
            self.last, self.d = self.last[cut:], self.d[cut:]
            self.p = None if self.p is None else self.p[cut:]
        self.inp.opt.retarget_batch(last_qpos=self.last, damping=self.d, projected=self.p, out=self.qs[t],
                                    status_out=self.ss[t], clip_init=True, stream=stream, **self.inp.step(t, self.S - b))
        self.last = self.qs[t]
        self.t += 1

    def run(self, barrier):
        torch.cuda.synchronize()  # (the poison and the inputs are in place before the chain)
        while self.t < len(self.sizes):
            self.step()
            barrier()
        torch.cuda.synchronize()
        return self

    def tensors(self):
        return self.qs + self.ss + [self.damping] + ([] if self.projected is None else [self.projected])


def _serialised(monkeypatch):
    monkeypatch.setenv("DEXR_FRAMES_PDL", "0")


def _as_shipped(monkeypatch):
    monkeypatch.delenv("DEXR_FRAMES_PDL", raising=False)


def _assert_equal(got, ref, what):
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.shape == b.shape and torch.equal(a, b), f"{what}: tensor {i} differs from the serialised calls"


def _assert_clean(statuses, qs, what):
    for t, (s, q) in enumerate(zip(statuses, qs)):
        assert int(((s & NONFINITE) != 0).sum()) == 0, f"{what}: step {t} has non-finite frames"
        assert bool(torch.isfinite(q).all()), f"{what}: step {t} has non-finite answers"


def twin(monkeypatch, make, what):
    """`make()` -> a fresh object with run(barrier) -> self and tensors(): run once serialised (DEXR_FRAMES_PDL=0, a
    synchronise after every call), once as shipped with nothing between the calls; every tensor equal bit for bit."""
    _serialised(monkeypatch)
    ref = make().run(torch.cuda.synchronize).tensors()
    _as_shipped(monkeypatch)
    got = make().run(lambda: None).tensors()
    _assert_equal(got, ref, what)
    return got


# ------------------------------------------------------------------------------------------------ 1. serialised twin
KINDS = [  # (id, config key or structure case, solver instantiation, links)
    ("block16_allegro", W.METRIC_KEY, "<16,4>", HEADLINE_LINKS),
    ("dense16_leap_dexpilot", W.LEAP_DEXPILOT_KEY, "<16,0>", OTHER_LINKS),
    ("arrow32_shadow_position", W.SHADOW_POS_KEY, "<32,-1>", OTHER_LINKS),
    ("dense32_svh_offline", "offline/schunk_svh_hand_right", "<32,0>", OTHER_LINKS),
    ("mimic_ability", "teleop/ability_hand_right", "<16,0>", OTHER_LINKS),
    ("fixed_mimic_dense32", "mimic_fixed_dense32", "<32,0>", OTHER_LINKS),
]
SCHEDULES = {"queue": {}, "static": {"DEXR_FRAMES_QUEUE": "0"}, "stages2": {"DEXR_FRAMES_STAGES": "2"}}
CHAIN_CASES = [(c, s) for c in KINDS for s in (SCHEDULES if c is KINDS[0] else ["queue"])]


@pytest.mark.parametrize("case,schedule", CHAIN_CASES, ids=[f"{c[0]}-{s}" for c, s in CHAIN_CASES])
def test_chain_matches_serialised_calls(case, schedule, tmp_path, monkeypatch):
    """A chain of 7 calls with PDL as shipped == the same calls serialised, at every step: answers, statuses, the final
    damping and flags.  No frame is non-finite (a read of a poisoned answer would be)."""
    kind, key, solver, links = case
    for k, v in SCHEDULES[schedule].items():
        monkeypatch.setenv(k, v)
    T = len(links)
    if key in SC.BY_ID:
        inp = case_inputs(SC.BY_ID[key], tmp_path, links[0], T)
    else:
        inp = stream_inputs(W.build(key, device=0), links[0], T)
    assert SC.solver_kind(inp.opt.build_table()) == solver
    got = twin(monkeypatch, lambda: ChainRun(inp, links), kind)
    _assert_clean(got[T:2 * T], got[:T], kind)


# ------------------------------------------------------------------------------------------------ 2. sequences kernel
@pytest.mark.parametrize("key", [W.METRIC_KEY, W.LEAP_DEXPILOT_KEY, W.SHADOW_POS_KEY])
def test_chain_matches_sequences_kernel(key, monkeypatch):
    """The chain (full-batch links: a tail slice would change the streams) is the recurrence retarget_sequences runs in
    registers -- clip, solve, carry the damping, advance the flags.  The sequences kernel's recorded per-frame answers equal
    every step's answers and its final state the chain's, bit for bit.  DEXR_SEQ_DUO=0: one group per stream, the
    summation order of the frames kernel."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "0")
    dev = _dev()
    seq = W.build(key, device=0)
    S, T = SEQ_S, SEQ_T
    inp = stream_inputs(seq, S, T)
    chain = ChainRun(inp, [S] * T).run(lambda: None)
    _assert_clean(chain.ss, chain.qs, key)

    state = seq.make_stream_state(S)
    tape = seq.make_sequence_tape(S, T)
    status = torch.zeros((S, T), dtype=torch.int32, device=dev)
    kp = inp.targets.transpose(0, 1).contiguous()
    fixed = None if inp.fixed is None else inp.fixed.transpose(0, 1).contiguous()
    seq.retarget_sequences(kp, state=state, fixed_qpos=fixed, status_out=status, tape=tape)
    torch.cuda.synchronize()
    for t in range(T):
        assert torch.equal(tape.qpos[:, t], chain.qs[t]), f"{key}: step {t}"
        assert torch.equal(status[:, t], chain.ss[t]), f"{key}: status of step {t}"
    assert torch.equal(state.last_qpos, chain.qs[-1])
    assert torch.equal(state.damping, chain.damping)
    if chain.projected is not None:
        assert torch.equal(state.projected, chain.projected)
        assert torch.equal(tape.projected[:, -1], chain.projected)


# ------------------------------------------------------------------------------------------------ 3. float64 oracle
@pytest.mark.parametrize("key,floor", [(W.LEAP_DEXPILOT_KEY, 0.985), (W.METRIC_KEY, 0.995)])
def test_chain_matches_oracle_teacher_forced(key, floor):
    """Four streams of a chain (the first, one inside, the last two: solved in the last tiles of the queue), every frame
    re-solved by the float64 oracle (mode B) from the chain's own previous answer, with the DexPilot flags advanced along
    the stream.  |dq|_inf < 1e-4 rad on frames in the same basin, median < 5e-6, and the same-basin fraction at the floors
    of test_gpu_bench_parity's teacher-forced stream test (the rest: other local minima entered at a flag switch)."""
    from oracle.solvers import solve_converged

    seq = W.build(key, device=0)
    S, T = ORACLE_S[key], ORACLE_T
    inp = stream_inputs(seq, S, T)
    chain = ChainRun(inp, [S] * T).run(lambda: None)
    _assert_clean(chain.ss, chain.qs, key)
    picks = [0, S // 3, S - 2, S - 1]
    q = torch.stack([qt[picks] for qt in chain.qs], 1).cpu().numpy().astype(np.float64)  # [4,T,n]
    kp = inp.targets[:, picks].transpose(0, 1).cpu().numpy()
    o = build_oracle(key)
    lim = seq.joint_limits
    dq = np.zeros((len(picks), T))
    for i in range(len(picks)):
        if o.type == "dexpilot":
            o.projected[:] = False
        last = lim.mean(1).astype(np.float32)
        for t in range(T):
            start = np.clip(last, lim[:, 0], lim[:, 1])
            xb, kkt, _ = solve_converged(o, o.ref_from_keypoints(kp[i, t]).astype(np.float32), np.zeros(0), start,
                                         update_state=True)
            assert kkt < 1e-6
            dq[i, t] = np.abs(xb - q[i, t]).max()
            last = q[i, t].astype(np.float32)
    same = dq < TOL
    print(f"{key}: same basin {same.mean():.4f} of {same.size} frames (floor {floor}), |dq| median {np.median(dq):.1e}, "
          f"max inside {dq[same].max() if same.any() else float('nan'):.1e}")
    assert dq[same].max() < TOL and np.median(dq) < 5e-6
    assert same.mean() >= floor, same.mean()


# ------------------------------------------------------------------------------------------------ 4. neighbours
class Calls:
    """A sequence of calls for `twin`: `body(barrier)` allocates and poisons its buffers, synchronises once, issues the calls
    (barrier() between them) and returns the tensors."""

    def __init__(self, body):
        self.body, self.out = body, None

    def run(self, barrier):
        self.out = self.body(barrier)
        torch.cuda.synchronize()
        return self

    def tensors(self):
        return self.out


def test_torch_kernel_writes_the_keypoints(monkeypatch):
    """torch.add (a kernel, not a copy engine memcpy) writes the keypoints the next frames launch reads, and overwrites
    them right after that launch for the next step."""
    inp = stream_inputs(W.build(W.METRIC_KEY, device=0), HEADLINE_B, len(HEADLINE_LINKS))

    def body(barrier):
        buf = torch.empty_like(inp.targets[0])
        ch = ChainRun(inp, HEADLINE_LINKS)
        torch.cuda.synchronize()
        for t, b in enumerate(HEADLINE_LINKS):
            dst = buf[HEADLINE_B - b:]
            torch.add(inp.targets[t, HEADLINE_B - b:], 0.0, out=dst)
            barrier()
            cut = ch.last.shape[0] - b
            ch.last, ch.d = ch.last[cut:], ch.d[cut:]
            inp.opt.retarget_batch(keypoints=dst, last_qpos=ch.last, damping=ch.d, out=ch.qs[t], status_out=ch.ss[t],
                                   clip_init=True)
            ch.last = ch.qs[t]
            barrier()
        return ch.tensors()

    got = twin(monkeypatch, lambda: Calls(body), "torch.add -> retarget_batch")
    T = len(HEADLINE_LINKS)
    _assert_clean(got[T:2 * T], got[:T], "torch.add -> retarget_batch")


def _rotations(n, rng):
    q, r = np.linalg.qr(rng.randn(n, 3, 3))
    q *= np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def test_preprocessing_writes_the_keypoints(monkeypatch):
    """preprocess_keypoints turns raw landmarks (recorded frames under random camera poses) into the keypoints the next
    frames launch reads, into one buffer reused every step."""
    from dex_retargeting_b200.constants import HandType
    from dex_retargeting_b200.preprocess import preprocess_keypoints

    seq = W.build(W.LEAP_DEXPILOT_KEY, device=0)
    links = OTHER_LINKS
    inp = stream_inputs(seq, OTHER_B, len(links))
    rng = np.random.RandomState(3)
    raw = np.einsum("sij,tskj->tski", _rotations(OTHER_B, rng), inp.targets.cpu().numpy().astype(np.float64))
    raw = torch.from_numpy((raw + rng.randn(1, OTHER_B, 1, 3) * 0.3).astype(np.float32)).to(_dev())

    def body(barrier):
        buf = torch.empty_like(raw[0])
        ch = ChainRun(inp, links)
        torch.cuda.synchronize()
        for t, b in enumerate(links):
            preprocess_keypoints(raw[t, OTHER_B - b:], HandType.right, out=buf[OTHER_B - b:])
            barrier()
            cut = ch.last.shape[0] - b
            ch.last, ch.d, ch.p = ch.last[cut:], ch.d[cut:], ch.p[cut:]
            inp.opt.retarget_batch(keypoints=buf[OTHER_B - b:], last_qpos=ch.last, damping=ch.d, projected=ch.p,
                                   out=ch.qs[t], status_out=ch.ss[t], clip_init=True)
            ch.last = ch.qs[t]
            barrier()
        return ch.tensors() + [buf]

    got = twin(monkeypatch, lambda: Calls(body), "preprocess_keypoints -> retarget_batch")
    T = len(links)
    _assert_clean(got[T:2 * T], got[:T], "preprocess_keypoints -> retarget_batch")


def test_derivative_kernels_after_a_solve(monkeypatch):
    """objective_batch, retarget_batch_vjp and retarget_batch_jacobian (not launched as dependents) each directly after a
    solve, at its answer, with the flags it left."""
    seq = W.build(W.LEAP_DEXPILOT_KEY, device=0)
    opt = seq.optimizer
    B = OTHER_B
    inp = stream_inputs(seq, B, 6)
    dev = _dev()
    grad = torch.from_numpy(np.random.RandomState(4).randn(B, opt.opt_dof).astype(np.float32)).to(dev)

    def body(barrier):
        ch = ChainRun(inp, [B] * 6)
        sts = [torch.full((B,), -1, dtype=torch.int32, device=dev) for _ in range(6)]
        outs = []
        torch.cuda.synchronize()
        for t in range(6):
            ch.step()
            barrier()
            kw = dict(keypoints=inp.targets[t], last_qpos=inp.x0 if t == 0 else ch.qs[t - 1])
            st = sts[t]
            if t % 3 == 0:  # (no flags: the evaluation updates the ones it is given)
                outs += list(opt.objective_batch(ch.qs[t], **kw))
            elif t % 3 == 1:
                outs += list(opt.retarget_batch_vjp(grad, ch.qs[t], projected=ch.projected, status_out=st, **kw)) + [st]
            else:
                outs += list(opt.retarget_batch_jacobian(ch.qs[t], projected=ch.projected, status_out=st, **kw)) + [st]
            barrier()
        return ch.tensors() + [x for x in outs if x is not None]

    got = twin(monkeypatch, lambda: Calls(body), "retarget_batch -> derivative kernels")
    _assert_clean(got[6:12], got[:6], "retarget_batch -> derivative kernels")
    assert len(got) == 14 + 6 * 3  # per step (loss, cost, grad) or (targets, last_qpos, status)
    assert all(bool(torch.isfinite(x).all()) for x in got[14:] if x.dtype == torch.float32)


@pytest.mark.parametrize("mode", ["streams", "persistent"])
def test_mixed_launch_then_single_robot(mode, monkeypatch):
    """retarget_batch_mixed (headline robot and LEAP DexPilot), then single-robot launches that continue the headline
    group's streams from the tail of its output, damping carried."""
    from dex_retargeting_b200.optimizer import retarget_batch_mixed

    monkeypatch.setenv("DEXR_MULTI_MODE", mode)
    dev = _dev()
    head = stream_inputs(W.build(W.METRIC_KEY, device=0), 40000, 4)
    leap = stream_inputs(W.build(W.LEAP_DEXPILOT_KEY, device=0), 12000, 1)

    def body(barrier):
        q0, s0 = _poisoned(head.opt, [40000])
        d0, _ = _state(head.opt, 40000)
        q1, s1 = _poisoned(leap.opt, [12000])
        d1, p1 = _state(leap.opt, 12000)
        sizes = [4096, 1000, 3]
        qs, ss = _poisoned(head.opt, sizes)
        torch.cuda.synchronize()
        retarget_batch_mixed([(head.opt, dict(keypoints=head.targets[0], last_qpos=head.x0, damping=d0, out=q0[0],
                                              status_out=s0[0], clip_init=True)),
                              (leap.opt, dict(keypoints=leap.targets[0], last_qpos=leap.x0, damping=d1, projected=p1,
                                              out=q1[0], status_out=s1[0], clip_init=True))])
        barrier()
        last, d = q0[0], d0
        for t, b in enumerate(sizes):
            last, d = last[last.shape[0] - b:], d[d.shape[0] - b:]
            head.opt.retarget_batch(keypoints=head.targets[t + 1, 40000 - b:], last_qpos=last, damping=d, out=qs[t],
                                    status_out=ss[t], clip_init=True)
            last = qs[t]
            barrier()
        return q0 + s0 + q1 + s1 + qs + ss + [d0, d1, p1]

    got = twin(monkeypatch, lambda: Calls(body), f"mixed ({mode}) -> retarget_batch")
    _assert_clean([got[1], got[3]] + got[7:10], [got[0], got[2]] + got[4:7], f"mixed ({mode}) -> retarget_batch")


def test_two_robots_alternate_on_one_stream(monkeypatch):
    """Bimanual teleop: Allegro left and right take turns on one stream, each carrying its own chain with tail links, so
    every launch directly follows one of the other robot."""
    left = stream_inputs(W.build("teleop/allegro_hand_left", device=0), HEADLINE_B, len(HEADLINE_LINKS), seed=21)
    right = stream_inputs(W.build(W.METRIC_KEY, device=0), HEADLINE_B, len(HEADLINE_LINKS), seed=22)

    class Pair:
        def run(self, barrier):
            self.a, self.b = ChainRun(left, HEADLINE_LINKS), ChainRun(right, HEADLINE_LINKS)
            torch.cuda.synchronize()
            for _ in HEADLINE_LINKS:
                self.a.step()
                barrier()
                self.b.step()
                barrier()
            torch.cuda.synchronize()
            return self

        def tensors(self):
            return self.a.tensors() + self.b.tensors()

    got = twin(monkeypatch, Pair, "Allegro left / right")
    T = len(HEADLINE_LINKS)
    n = 2 * T + 1
    _assert_clean(got[T:2 * T] + got[n + T:n + 2 * T], got[:T] + got[n:n + T], "Allegro left / right")


def test_chain_across_two_streams_joined_by_events(monkeypatch):
    """The chain alternates between two streams: each launch is followed by an event recorded on its stream that the other
    stream waits for before the next launch reads its output."""
    inp = stream_inputs(W.build(W.METRIC_KEY, device=0), HEADLINE_B, len(HEADLINE_LINKS))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]

    class TwoStreams(ChainRun):
        def run(self, barrier):
            torch.cuda.synchronize()
            for t in range(len(self.sizes)):
                st, other = streams[t % 2], streams[1 - t % 2]
                with torch.cuda.stream(st):
                    self.step(stream=st)
                ev = torch.cuda.Event()
                ev.record(st)
                other.wait_event(ev)
                barrier()
            torch.cuda.synchronize()
            return self

    got = twin(monkeypatch, lambda: TwoStreams(inp, HEADLINE_LINKS), "two streams")
    T = len(HEADLINE_LINKS)
    _assert_clean(got[T:2 * T], got[:T], "two streams")


def test_joint_limits_changed_mid_chain(monkeypatch):
    """set_joint_limit after the third call: the next call rebuilds the engine and its device table, and the chain goes on
    from the previous answers inside the narrowed limits."""
    links = HEADLINE_LINKS

    class Narrowed(ChainRun):
        def run(self, barrier):
            opt = self.inp.opt
            lim = opt._limits.copy()
            torch.cuda.synchronize()
            for t in range(len(self.sizes)):
                if t == 3:
                    mid, half = lim.mean(1), 0.35 * (lim[:, 1] - lim[:, 0])
                    opt.set_joint_limit(np.stack([mid - half, mid + half], 1))
                self.step()
                barrier()
            torch.cuda.synchronize()
            opt.set_joint_limit(lim)
            self.narrow = (mid - half - 2e-3, mid + half + 2e-3)
            return self

    inp = stream_inputs(W.build(W.METRIC_KEY, device=0), HEADLINE_B, len(links))
    chains = []

    def make():
        chains.append(Narrowed(inp, links))
        return chains[-1]

    got = twin(monkeypatch, make, "set_joint_limit mid-chain")
    T = len(links)
    _assert_clean(got[T:2 * T], got[:T], "set_joint_limit mid-chain")
    lo, hi = (torch.from_numpy(v.astype(np.float32)).to(_dev()) for v in chains[-1].narrow)
    for q in got[3:T]:
        assert bool(((q >= lo) & (q <= hi)).all()), "answers after set_joint_limit leave the new limits"
    assert not bool(((got[0] >= lo) & (got[0] <= hi)).all()), "the narrowed limits bind nothing"
