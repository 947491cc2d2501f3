"""Backpropagation through the sequence solve (`dexr_solve_sequences_tape` / `dexr_solve_sequences_vjp`,
SeqRetargeting.retarget_sequences_vjp, objective.differentiable_retarget_sequences) through the host emulation of the
kernels' own drivers (tests/emu runs solve_stream<G, BW, true> and vjp_stream of dexr_kernels.cuh): against the float64
reverse-time model of tests/seq_vjp_cases.py on 16- and 32-lane robots, DexPilot with flags that switch mid-stream, mimic
and fixed-joint hands, with and without the low-pass filter and the final-state cotangents; the recurrence itself against
central differences of whole float64 oracle streams; the recorded forward against the unrecorded one; NaN isolation; the
argument checks; the kernels' register budget.  The GPU test file tests/test_gpu_seq_vjp.py is dry-run here as well."""
import ctypes as C
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_host
import emu_seq_vjp_host as H
import seq_vjp_cases as SV
import structure_cases as SC
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID
NO_FILTER = {"low_pass_alpha": -1.0}


def _problem(seq, o, S, T, seed, pinch=False, filter_init=0, band=0.0):
    """Inputs, the oracle's streams (the tape) and seeded cotangents."""
    kp, fixed = SV.stream_inputs(o, S, T, seed, pinch=pinch)
    rng = np.random.RandomState(seed + 1)
    n, dof = o.opt_dof, o.robot.dof
    mid = o.joint_limits.mean(1)
    last0 = np.clip(mid + 0.1 * rng.randn(S, n), o.joint_limits[:, 0], o.joint_limits[:, 1]).astype(np.float32)
    if band:  # warm starts `band` outside clip_lo / clip_hi
        side = rng.rand(S, n) < 0.5
        last0 = np.where(side, np.float32(o.joint_limits[:, 0]) - np.float32(band),
                         np.float32(o.joint_limits[:, 1]) + np.float32(band)).astype(np.float32)
    y0 = rng.uniform(-0.3, 0.3, size=(S, dof)).astype(np.float32)
    finit = np.full(S, filter_init, np.uint8)
    ref = SV.oracle_streams(o, kp, fixed, last0, y0, finit)
    return dict(kp=kp, fixed=fixed, last0=last0, y0=y0, finit=finit, X=ref["qpos"], F=ref["flags"],
                g_out=rng.randn(S, T, dof).astype(np.float32), g_last=rng.randn(S, n).astype(np.float32),
                g_filter=rng.randn(S, dof).astype(np.float32))


def _emu(seq, p, state_grads=True, spw=0, **kw):
    return H.solve_sequences_vjp(seq, p["kp"], p["X"], p["last0"], p["finit"], p["F"], grad_robot_qpos=p["g_out"],
                                 grad_last_qpos=p["g_last"] if state_grads else None,
                                 grad_filter_state=p["g_filter"] if state_grads else None, fixed_qpos=p["fixed"], spw=spw,
                                 **kw)


def _against_model(seq, o, p, state_grads=True, spw=0):
    got = _emu(seq, p, state_grads, spw)
    worst = 0.0
    for s in range(p["kp"].shape[0]):
        m = SV.model_stream(o, p["kp"][s], None if p["fixed"] is None else p["fixed"][s], p["last0"][s], p["finit"][s],
                            p["X"][s], None if p["F"] is None else p["F"][s], g_out=p["g_out"][s],
                            g_last=p["g_last"][s] if state_grads else None,
                            g_filter=p["g_filter"][s] if state_grads else None)
        one = tuple(None if g is None else g[s] for g in got)
        worst = max(worst, SV.compare_stream(one, m))
    return worst, got


# (config, override, streams, steps, pinch): 16 lanes (Allegro vector, LEAP DexPilot with pinches), 32 lanes (Shadow
# position); S = 3 is not a multiple of the two 16-lane streams of a warp
PACKAGED = [
    ("teleop/allegro_hand_right", None, 3, 3, False),
    ("teleop/allegro_hand_right", NO_FILTER, 2, 3, False),
    ("offline/shadow_hand_right", None, 1, 3, False),
    ("teleop/leap_hand_right_dexpilot", None, 3, 4, True),
]


@pytest.mark.parametrize("filter_init", [0, 1])
@pytest.mark.parametrize("state_grads", [True, False])
@pytest.mark.parametrize("key,override,S,T,pinch", PACKAGED, ids=lambda v: str(v) if not isinstance(v, dict) else "nofilter")
def test_packaged_streams_match_model(key, override, S, T, pinch, state_grads, filter_init):
    seq, o = build_product(key, override), build_oracle(key, override)
    p = _problem(seq, o, S, T, seed=11 + filter_init, pinch=pinch, filter_init=filter_init)
    if pinch:  # the flags switch on and off again inside the streams
        on = p["F"].any(axis=2)
        assert on.any() and (~on).any(), on
    worst, _ = _against_model(seq, o, p, state_grads)
    print(key, "worst error / tau %.3f" % worst)


@pytest.mark.parametrize("case", ["mimic_dense16", "fixed_dense32", "mimic_fixed_dense16"])
def test_mimic_and_fixed_joint_streams_match_model(case, tmp_path):
    """The mimic fold of gq into its source variable, the direct fixed-joint term and the fixed joints' H-term."""
    seq, o = SC.build(SC.BY_ID[case], tmp_path)
    p = _problem(seq, o, 2, 3, seed=21)
    worst, _ = _against_model(seq, o, p)
    print(case, "worst error / tau %.3f" % worst)


@pytest.mark.parametrize("band", [5e-4, 0.3])
def test_warm_start_outside_the_limits_is_clipped(band):
    """Warm starts 0.5 mrad outside clip_lo / clip_hi (the widened band the solver's bounds can leave a solution in) and
    0.3 rad outside (a caller's state): the anchor is the clipped value and no cotangent reaches those entries of the
    initial last_qpos."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    p = _problem(seq, o, 2, 2, seed=23, band=band)
    worst, got = _against_model(seq, o, p)
    np.testing.assert_array_equal(got[2], 0.0)
    print("worst error / tau %.3f" % worst)


@pytest.mark.parametrize("spw", [0, 1])
def test_single_frame_streams_and_launch_shapes(spw):
    """T = 1, and the one-stream-per-warp launch shape gives the same bits as two streams per warp."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    p = _problem(seq, o, 3, 1, seed=25, filter_init=1)
    worst, got = _against_model(seq, o, p, spw=spw)
    if spw == 1:
        ref = _emu(seq, p)
        for a, b in zip(got, ref):
            if a is not None:
                np.testing.assert_array_equal(a, b)


def test_recurrence_against_central_differences_of_oracle_streams():
    """The recurrence itself, independently of model_vjp: l = sum(w * robot_qpos) of whole float64 oracle streams (T = 4)
    re-solved under central differences in keypoint coordinates of the first and last frame, in the initial last_qpos and
    in the initial filter state, for a filtered vector robot and an unfiltered position robot.  The streams' solutions are
    rounded to float32 as the oracle stream keeps them, so the differences carry about 1e-4 / h of rounding noise."""
    h = 1e-3
    for key, override in (("teleop/allegro_hand_right", None), ("offline/allegro_hand_right", NO_FILTER)):
        seq, o = build_product(key, override), build_oracle(key, override)
        p = _problem(seq, o, 1, 4, seed=27, filter_init=1)
        g_out = p["g_out"][0].astype(np.float64)

        def loss(kp=p["kp"][0], last0=p["last0"][0], y0=p["y0"][0]):
            r = SV.oracle_stream(o, kp, None, last0, y0, 1)
            return float((g_out * r["robot_qpos"]).sum())

        got = _emu(seq, p, state_grads=False)
        used = int(np.asarray(o.target_link_human_indices).reshape(-1)[-1])
        checks = [("keypoints", (0, used, 1)), ("keypoints", (3, used, 0)), ("last0", (2,)), ("last0", (5,))]
        if 0 <= o.low_pass_alpha <= 1:
            checks += [("y0", (1,)), ("y0", (7,))]
        for name, at in checks:
            base = dict(kp=p["kp"][0], last0=p["last0"][0], y0=p["y0"][0])[{"keypoints": "kp"}.get(name, name)]
            plus, minus = base.astype(np.float64).copy(), base.astype(np.float64).copy()
            plus[at] += h
            minus[at] -= h
            arg = {"keypoints": "kp"}.get(name, name)
            fd = (loss(**{arg: plus.astype(np.float32) if arg != "y0" else plus}) -
                  loss(**{arg: minus.astype(np.float32) if arg != "y0" else minus})) / (2 * h)
            an = {"keypoints": got[0][0], "last0": got[2][0], "y0": got[3][0]}[name][at]
            assert abs(an - fd) <= 2e-2 * max(abs(fd), 2e-2), (key, name, at, an, fd)


@pytest.mark.parametrize("key", ["teleop/leap_hand_right_dexpilot", "offline/shadow_hand_right", "teleop/allegro_hand_right"])
def test_recorded_forward_is_the_unrecorded_forward(key):
    """The taped call's outputs, status and final state are bit-identical to dexr_solve_sequences; tape.qpos[:, -1] is the
    final last_qpos and the flag tape ends at the final flags."""
    seq = build_product(key)
    o = build_oracle(key)
    kp, _ = SV.stream_inputs(o, 3, 3, seed=29, pinch=True)
    st_a, st_b = H.fresh_state(seq, 3), H.fresh_state(seq, 3)
    out_a, status_a, _ = emu_host.solve_sequences(seq, kp, state=st_a)
    out_b, status_b, _, tape = H.solve_sequences_tape(seq, kp, state=st_b)
    np.testing.assert_array_equal(out_a, out_b)
    np.testing.assert_array_equal(status_a, status_b)
    for k in st_a:
        if st_a[k] is not None:
            np.testing.assert_array_equal(st_a[k], st_b[k])
    np.testing.assert_array_equal(tape["qpos"][:, -1], st_b["last_qpos"])
    if tape["projected"] is not None:
        np.testing.assert_array_equal(tape["projected"][:, -1], st_b["projected"])
        # the flags after every frame: a stream cut after frame t ends with the tape's row t
        for t in range(2):
            st_c = H.fresh_state(seq, 3)
            H.solve_sequences_tape(seq, kp[:, :t + 1], state=st_c)
            np.testing.assert_array_equal(tape["projected"][:, t], st_c["projected"])


def test_non_finite_frame_poisons_its_stream_only():
    """A NaN keypoint in stream 1, frame 2: that frame and every earlier frame of stream 1 get NaN cotangents and
    DEXR_STATUS_NONFINITE, later frames of stream 1 and every other stream are bit-identical to a clean run."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    p = _problem(seq, o, 3, 4, seed=31)
    clean = _emu(seq, p)
    bad = dict(p, kp=p["kp"].copy())
    used = int(np.asarray(o.target_link_human_indices).reshape(-1)[-1])
    bad["kp"][1, 2, used, 0] = np.nan
    got = _emu(seq, bad)
    assert np.all(got[4][1, :3] == V_NONFINITE) and np.array_equal(got[4][1, 3:], clean[4][1, 3:])
    assert np.all(np.isnan(got[0][1, :3])) and np.all(np.isnan(got[2][1]))
    np.testing.assert_array_equal(got[0][1, 3:], clean[0][1, 3:])
    for g_clean, g in zip(clean, got):
        if g is not None:
            np.testing.assert_array_equal(g[[0, 2]], g_clean[[0, 2]])


V_NONFINITE = 1 << 25


def test_abi_layout_and_argument_checks(tmp_path):
    """dexr_sequences_tape_t / dexr_sequences_vjp_t agree with their bindings; the library rejects null arguments without a
    GPU, and seq_vjp_io_error (shared by the library and the emulation) rejects every malformed buffer set."""
    from dex_retargeting_b200 import _native as N

    lib = N.load()
    assert lib.dexr_sequences_tape_sizeof() == C.sizeof(N.DexrSequencesTape) == 16
    assert lib.dexr_sequences_vjp_sizeof() == C.sizeof(N.DexrSequencesVjp) == 112
    assert lib.dexr_sequences_sizeof() == 72
    p, io, tp = N.default_params(), N.DexrSequencesVjp(), N.DexrSequencesTape()
    assert lib.dexr_solve_sequences_vjp(None, C.byref(p), C.byref(io), 1, 1, None) == N_INVALID
    assert b"null" in lib.dexr_last_error()
    assert lib.dexr_solve_sequences_tape(None, C.byref(p), C.byref(N.DexrSequences()), C.byref(tp), 1, 1, None) == N_INVALID
    assert b"null" in lib.dexr_last_error()

    key = "teleop/leap_hand_right_dexpilot"
    seq, o = build_product(key), build_oracle(key)
    kp = np.zeros((1, 2, 21, 3), np.float32)
    X = np.zeros((1, 2, o.opt_dof), np.float32)
    F = np.zeros((1, 2, len(o.projected)), np.uint8)
    last0, finit = np.zeros((1, o.opt_dof), np.float32), np.zeros(1, np.uint8)
    for kw, msg in [(dict(raw_hand="right"), "pre-processing is not differentiated"),
                    (dict(null=("qpos",)), "qpos (the tape of the forward call) is required"),
                    (dict(null=("last_qpos",)), "last_qpos (the warm start before the forward call) is required"),
                    (dict(null=("keypoints",)), "keypoints are required"),
                    (dict(null=("filter_init",)), "the low-pass filter needs filter_init"),
                    (dict(null=("projected",)), "DexPilot needs the flag tape")]:
        with pytest.raises(H.EmulationError) as e:
            H.solve_sequences_vjp(seq, kp, X, last0, finit, F, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg, (kw, e.value.msg)
    seq2, o2 = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    with pytest.raises(H.EmulationError, match="fixed joints but fixed_qpos is NULL"):
        H.solve_sequences_vjp(seq2, kp, np.zeros((1, 2, o2.opt_dof), np.float32), np.zeros((1, o2.opt_dof), np.float32),
                              finit, fixed_qpos=np.zeros((1, 2, 2), np.float32), null=("fixed_qpos",))


def test_differentiable_retarget_sequences_refuses_to_differentiate_raw_landmarks():
    torch = pytest.importorskip("torch")
    from dex_retargeting_b200.objective import differentiable_retarget_sequences
    from dex_retargeting_b200.seq_retarget import StreamState

    seq = build_product("teleop/allegro_hand_right")
    n, dof = seq.optimizer.opt_dof, seq.optimizer.robot.dof
    state = StreamState(last_qpos=torch.zeros((2, n)), filter_state=torch.zeros((2, dof)),
                        filter_init=torch.zeros(2, dtype=torch.uint8), projected=None)
    kp = torch.zeros((2, 3, 21, 3), requires_grad=True)
    with pytest.raises(ValueError, match="raw-landmark pre-processing is not differentiated"):
        differentiable_retarget_sequences(seq, kp, state, raw_hand="right")


def test_recording_raw_landmarks_is_refused():
    """A tape is for the backward, and raw-landmark pre-processing is not differentiated: retarget_sequences refuses
    raw_hand together with tape= before it touches the device."""
    torch = pytest.importorskip("torch")
    from dex_retargeting_b200.seq_retarget import SequenceTape

    seq = build_product("teleop/allegro_hand_right")
    tape = SequenceTape(qpos=torch.zeros((2, 3, seq.optimizer.opt_dof)), projected=None)
    with pytest.raises(ValueError, match="raw-landmark pre-processing is not differentiated"):
        seq.retarget_sequences(torch.zeros((2, 3, 21, 3)), raw_hand="right", tape=tape)


def test_seq_vjp_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v`: dexr_seq_vjp_kernel<16> and <32> spill nothing, and each recorded sequences kernel spills no more than
    its unrecorded twin."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    for g in (16, 32):
        name = f"_ZN4dexr19dexr_seq_vjp_kernelILi{g}EEEvNS_10SeqVjpArgsE"
        assert stores.get(name) == 0, (name, stores.get(name))
    for inst in ("ILi16ELi0ELi8E", "ILi16ELi4ELi8E", "ILi32ELi0ELi8E", "ILi32ELin1ELi8E"):
        plain = stores[f"_ZN4dexr21dexr_sequences_kernel{inst}EEvNS_7SeqArgsE"]
        taped = stores[f"_ZN4dexr26dexr_sequences_tape_kernel{inst}EEvNS_7SeqArgsE19dexr_sequences_tape"]
        assert taped <= plain, (inst, taped, plain)


def test_gpu_seq_vjp_file_passes_against_the_emulation():
    """tests/test_gpu_seq_vjp.py dry-run on the CPU (tests/tools/emu_gpu_seq_vjp.py: the recorded forward, the sequence VJP
    and retarget_batch_vjp served by the emulation)."""
    count = 12
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_seq_vjp.py")], capture_output=True,
                         text=True, timeout=1800)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
