"""Packed streams (`dexr_solve_sequences_packed`, `dexr_solve_sequences_packed_vjp`) through the host emulation of the
kernels' own drivers (tests/emu runs solve_packed_stream<G, BW, REC> and vjp_packed_stream of dexr_kernels.cuh) on the
four solver instantiations (block 16, dense 16, arrow 32, dense 32): equal lengths bit for bit against the rectangular
drivers, in paired and duo mode; ragged lengths (0 and 1 included) bit for bit against each stream solved alone; the
float64 oracle streams and the reverse-time model of tests/seq_vjp_cases.py; chained chunks; the streams' positions in
the batch and both VJP launch shapes; malformed
layouts inside guard words; the argument checks; the new kernels' register budget; and a dry run of
tests/test_gpu_packed_streams.py."""
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import emu_host
import emu_packed_host as P
import emu_seq_vjp_host as H
import seq_vjp_cases as SV
import structure_cases as SC
from emu_eval_host import EmulationError
from helpers import build_oracle, build_product

ROOT = Path(__file__).resolve().parent.parent
N_INVALID = -1  # DEXR_E_INVALID
NO_FILTER = {"low_pass_alpha": -1.0}

# (name, kind the table is solved on, how to build it): the four instantiations, with and without the filter, DexPilot,
# fixed joints and mimic joints
CASES = [
    ("allegro_vector", "<16,4>", ("teleop/allegro_hand_right", None)),
    ("leap_dexpilot", "<16,0>", ("teleop/leap_hand_right_dexpilot", None)),
    ("mimic_fixed_dense16", "<16,0>", "mimic_fixed_dense16"),
    ("shadow_position_nofilter", "<32,-1>", ("offline/shadow_hand_right", NO_FILTER)),
    ("prismatic_arrow", "<32,-1>", "prismatic_arrow"),
    ("mimic_fixed_dense32", "<32,0>", "mimic_fixed_dense32"),
]
IDS = [c[0] for c in CASES]


def _build(spec, tmp_path):
    if isinstance(spec, str):
        return SC.build(SC.BY_ID[spec], tmp_path)
    return build_product(*spec), build_oracle(*spec)


def _setup(case, tmp_path):
    name, kind, spec = case
    seq, o = _build(spec, tmp_path)
    assert SC.solver_kind(seq.optimizer.build_table()) == kind, (name, kind)
    return seq, o


def _inputs(o, lengths, seed, pinch=False):
    """Packed keypoints [N,21,3] and fixed joints [N,n_fixed] (or None): stream s is a stream_inputs stream cut to lengths[s]."""
    T = max(int(max(lengths)), 1)
    kp, fixed = SV.stream_inputs(o, len(lengths), T, seed, pinch=pinch)
    pk = np.concatenate([kp[s, :n] for s, n in enumerate(lengths)]).reshape(-1, 21, 3)
    pf = None if fixed is None else np.concatenate([fixed[s, :n] for s, n in enumerate(lengths)]).reshape(-1, fixed.shape[2])
    return kp, fixed, pk, pf


def _start(seq, o, S, seed):
    """A seeded initial state (warm starts near mid-range, filter state set and initialised)."""
    rng = np.random.RandomState(seed)
    st = H.fresh_state(seq, S)
    st["last_qpos"][...] = np.clip(o.joint_limits.mean(1) + 0.1 * rng.randn(S, o.opt_dof), o.joint_limits[:, 0],
                                   o.joint_limits[:, 1])
    st["filter_state"][...] = rng.uniform(-0.3, 0.3, size=st["filter_state"].shape)
    st["filter_init"][...] = 1
    return st


def _copy(st):
    return {k: None if v is None else v.copy() for k, v in st.items()}


def _same_state(a, b, what=""):
    for k in a:
        if a[k] is None:
            assert b[k] is None
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{what} {k}")


def _cotangents(seq, S, Nf, seed):
    rng = np.random.RandomState(seed)
    opt = seq.optimizer
    return (rng.randn(Nf, opt.robot.dof).astype(np.float32), rng.randn(S, opt.opt_dof).astype(np.float32),
            rng.randn(S, opt.robot.dof).astype(np.float32))


def _packed_all(seq, pk, pf, lengths, st0, cot, duo=False, spw=0, offsets=None):
    """Unrecorded and recorded packed forward and the packed VJP from state st0 (not modified)."""
    offsets = P.offsets_of(lengths) if offsets is None else offsets
    st_u, st_r = _copy(st0), _copy(st0)
    out_u, status_u, _, _ = P.solve_packed(seq, pk, offsets, state=st_u, fixed_qpos=pf, duo=duo)
    out, status, _, tape = P.solve_packed(seq, pk, offsets, state=st_r, fixed_qpos=pf, record=True, duo=duo)
    np.testing.assert_array_equal(out_u, out)
    np.testing.assert_array_equal(status_u, status)
    _same_state(st_u, st_r, "recorded vs unrecorded")
    g_out, g_last, g_filter = cot
    grads = P.solve_packed_vjp(seq, pk, offsets, tape["qpos"], st0["last_qpos"], st0["filter_init"], tape["projected"],
                               grad_robot_qpos=g_out, grad_last_qpos=g_last, grad_filter_state=g_filter, fixed_qpos=pf,
                               spw=spw)
    return dict(out=out, status=status, state=st_r, tape=tape, grads=grads)


def _rect_all(seq, kp, fixed, st0, cot_rows, duo=False):
    """The rectangular drivers on [S,T] streams from st0: the same three calls."""
    st_u, st_r = _copy(st0), _copy(st0)
    out_u, status_u, _ = emu_host.solve_sequences(seq, kp, state=st_u, duo=duo, fixed_qpos=fixed)
    out, status, _, tape = H.solve_sequences_tape(seq, kp, state=st_r, fixed_qpos=fixed, duo=duo)
    np.testing.assert_array_equal(out_u, out)
    g_out, g_last, g_filter = cot_rows
    grads = H.solve_sequences_vjp(seq, kp, tape["qpos"], st0["last_qpos"], st0["filter_init"], tape["projected"],
                                  grad_robot_qpos=g_out, grad_last_qpos=g_last, grad_filter_state=g_filter, fixed_qpos=fixed)
    return dict(out=out, status=status, state=st_r, tape=tape, grads=grads)


@pytest.mark.parametrize("duo", [False, True])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_equal_lengths_are_the_rectangular_calls(case, duo, tmp_path):
    """Every stream T frames: outputs, status, state, tape and gradients equal the rectangular drivers bit for bit."""
    if duo and case[1].startswith("<32"):
        pytest.skip("duo mode is a 16-lane mode")
    seq, o = _setup(case, tmp_path)
    S, T = 3, 3
    kp, fixed, pk, pf = _inputs(o, [T] * S, seed=81, pinch=True)
    st0 = _start(seq, o, S, seed=82)
    cot = _cotangents(seq, S, S * T, seed=83)
    got = _packed_all(seq, pk, pf, [T] * S, st0, cot, duo=duo)
    ref = _rect_all(seq, kp, fixed, st0, (cot[0].reshape(S, T, -1), cot[1], cot[2]), duo=duo)
    np.testing.assert_array_equal(got["out"], ref["out"].reshape(S * T, -1))
    np.testing.assert_array_equal(got["status"], ref["status"].reshape(-1))
    _same_state(got["state"], ref["state"])
    np.testing.assert_array_equal(got["tape"]["qpos"], ref["tape"]["qpos"].reshape(S * T, -1))
    if ref["tape"]["projected"] is not None:
        np.testing.assert_array_equal(got["tape"]["projected"], ref["tape"]["projected"].reshape(S * T, -1))
    for a, b in zip(got["grads"], ref["grads"]):
        if b is not None:
            np.testing.assert_array_equal(a, b.reshape(a.shape))


@pytest.mark.parametrize("duo", [False, True])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_ragged_streams_are_each_stream_alone(case, duo, tmp_path):
    """Lengths 3, 0, 1, 2, 0 (a warp of two 16-lane streams pairs 3 with 0 and 1 with 2): each stream's outputs, final
    state, tape and gradients equal a rectangular call on that stream alone; a stream of length 0 keeps its state and
    passes its cotangents through."""
    if duo and case[1].startswith("<32"):
        pytest.skip("duo mode is a 16-lane mode")
    seq, o = _setup(case, tmp_path)
    lengths = [3, 0, 1, 2, 0]
    S = len(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=84, pinch=True)
    st0 = _start(seq, o, S, seed=85)
    cot = _cotangents(seq, S, sum(lengths), seed=86)
    got = _packed_all(seq, pk, pf, lengths, st0, cot, duo=duo)
    offs = P.offsets_of(lengths)
    for s, n in enumerate(lengths):
        a, b = offs[s], offs[s + 1]
        one = {k: None if v is None else v[s:s + 1].copy() for k, v in st0.items()}
        mine = {k: None if v is None else v[s:s + 1] for k, v in got["state"].items()}
        if n == 0:
            _same_state(mine, one, f"empty stream {s}")
            np.testing.assert_array_equal(got["grads"][2][s], cot[1][s])
            np.testing.assert_array_equal(got["grads"][3][s], cot[2][s])
            continue
        ref = _rect_all(seq, kp[s:s + 1, :n], None if fixed is None else fixed[s:s + 1, :n], one,
                        (cot[0][None, a:b], cot[1][s:s + 1], cot[2][s:s + 1]), duo=duo)
        np.testing.assert_array_equal(got["out"][a:b], ref["out"][0])
        np.testing.assert_array_equal(got["status"][a:b], ref["status"][0])
        _same_state(mine, ref["state"], f"stream {s}")
        np.testing.assert_array_equal(got["tape"]["qpos"][a:b], ref["tape"]["qpos"][0])
        g_kp, g_fixed, g_last, g_filter, status = got["grads"]
        np.testing.assert_array_equal(g_kp[a:b], ref["grads"][0][0])
        if g_fixed is not None:
            np.testing.assert_array_equal(g_fixed[a:b], ref["grads"][1][0])
        np.testing.assert_array_equal(g_last[s], ref["grads"][2][0])
        np.testing.assert_array_equal(g_filter[s], ref["grads"][3][0])
        np.testing.assert_array_equal(status[a:b], ref["grads"][4][0])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_ragged_streams_match_the_float64_model(case, tmp_path):
    """The packed VJP at the oracle streams' tape against model_stream at compare_stream's tau, and, for the packaged
    robots, every forward frame against the float64 oracle streams (|dq| < 1e-4 rad)."""
    seq, o = _setup(case, tmp_path)
    lengths = [3, 1, 0, 2]
    S = len(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=87, pinch=True)
    st0 = _start(seq, o, S, seed=88)
    cot = _cotangents(seq, S, sum(lengths), seed=89)
    offs = P.offsets_of(lengths)
    refs = [None if n == 0 else SV.oracle_stream(o, kp[s, :n], None if fixed is None else fixed[s, :n], st0["last_qpos"][s],
                                                 st0["filter_state"][s], 1) for s, n in enumerate(lengths)]
    X = np.concatenate([r["qpos"] for r in refs if r is not None]).astype(np.float32)
    F = None if refs[0]["flags"] is None else np.concatenate([r["flags"] for r in refs if r is not None])
    grads = P.solve_packed_vjp(seq, pk, offs, X, st0["last_qpos"], st0["filter_init"], F, grad_robot_qpos=cot[0],
                               grad_last_qpos=cot[1], grad_filter_state=cot[2], fixed_qpos=pf)
    if not isinstance(case[2], str):
        st = _copy(st0)
        out, _, _, _ = P.solve_packed(seq, pk, offs, state=st, fixed_qpos=pf)
    worst = 0.0
    for s, n in enumerate(lengths):
        if n == 0:
            continue
        a, b = offs[s], offs[s + 1]
        r = refs[s]
        if not isinstance(case[2], str):
            assert np.abs(out[a:b] - r["robot_qpos"]).max() < 1e-4, (s, np.abs(out[a:b] - r["robot_qpos"]).max())
        m = SV.model_stream(o, kp[s, :n], None if fixed is None else fixed[s, :n], st0["last_qpos"][s], 1, r["qpos"],
                            r["flags"], g_out=cot[0][a:b], g_last=cot[1][s], g_filter=cot[2][s])
        one = (grads[0][a:b], None if grads[1] is None else grads[1][a:b], grads[2][s], grads[3][s], grads[4][a:b])
        worst = max(worst, SV.compare_stream(one, m))
    print(case[0], "worst error / tau %.3f" % worst)


@pytest.mark.parametrize("case", [CASES[1], CASES[2], CASES[5]], ids=[CASES[1][0], CASES[2][0], CASES[5][0]])
def test_chained_calls_are_one_call(case, tmp_path):
    """packed(L1) then packed(L2) on the returned state equals packed(L1 + L2) bit for bit; the backward of the two chunks,
    the second's initial-state gradients fed to the first, equals the backward of the one call."""
    seq, o = _setup(case, tmp_path)
    l1, l2 = np.array([2, 0, 1, 3]), np.array([1, 2, 0, 1])
    lengths = l1 + l2
    S = len(lengths)
    kp, fixed, pk, pf = _inputs(o, lengths, seed=90, pinch=True)
    st0 = _start(seq, o, S, seed=91)
    cot = _cotangents(seq, S, int(lengths.sum()), seed=92)
    whole = _packed_all(seq, pk, pf, lengths, st0, cot)
    offs = P.offsets_of(lengths)
    r1 = np.concatenate([offs[s] + np.arange(l1[s]) for s in range(S)]).astype(int)
    r2 = np.concatenate([offs[s] + l1[s] + np.arange(l2[s]) for s in range(S)]).astype(int)
    sub = (lambda a, r: None if a is None else a[r])
    st1 = _copy(st0)
    out1, _, _, tape1 = P.solve_packed(seq, pk[r1], P.offsets_of(l1), state=st1, fixed_qpos=sub(pf, r1), record=True)
    mid = _copy(st1)
    out2, _, _, tape2 = P.solve_packed(seq, pk[r2], P.offsets_of(l2), state=st1, fixed_qpos=sub(pf, r2), record=True)
    np.testing.assert_array_equal(out1, whole["out"][r1])
    np.testing.assert_array_equal(out2, whole["out"][r2])
    _same_state(st1, whole["state"])
    g2 = P.solve_packed_vjp(seq, pk[r2], P.offsets_of(l2), tape2["qpos"], mid["last_qpos"], mid["filter_init"],
                            tape2["projected"], grad_robot_qpos=cot[0][r2], grad_last_qpos=cot[1], grad_filter_state=cot[2],
                            fixed_qpos=sub(pf, r2))
    g1 = P.solve_packed_vjp(seq, pk[r1], P.offsets_of(l1), tape1["qpos"], st0["last_qpos"], st0["filter_init"],
                            tape1["projected"], grad_robot_qpos=cot[0][r1], grad_last_qpos=g2[2], grad_filter_state=g2[3],
                            fixed_qpos=sub(pf, r1))
    np.testing.assert_array_equal(g1[0], whole["grads"][0][r1])
    np.testing.assert_array_equal(g2[0], whole["grads"][0][r2])
    np.testing.assert_array_equal(g1[2], whole["grads"][2])
    np.testing.assert_array_equal(g1[3], whole["grads"][3])


@pytest.mark.parametrize("case", [CASES[0], CASES[3]], ids=[CASES[0][0], CASES[3][0]])
def test_results_do_not_depend_on_the_position_in_the_batch(case, tmp_path):
    """The same streams packed longest first or in a random order, and the VJP with one stream per warp: every stream's
    bits are the same (the cotangents follow their streams)."""
    seq, o = _setup(case, tmp_path)
    lengths = np.array([2, 0, 3, 1, 2])
    S = len(lengths)
    _, _, pk, pf = _inputs(o, lengths, seed=93)
    st0 = _start(seq, o, S, seed=94)
    cot = _cotangents(seq, S, int(lengths.sum()), seed=95)
    a = _packed_all(seq, pk, pf, lengths, st0, cot)
    offs = P.offsets_of(lengths)
    for perm in (np.argsort(-lengths, kind="stable"), np.random.RandomState(96).permutation(S)):
        rows = np.concatenate([offs[s] + np.arange(lengths[s]) for s in perm]).astype(int)
        for spw in (0, 1):
            b = _packed_all(seq, pk[rows], None if pf is None else pf[rows], lengths[perm],
                            {k: None if v is None else v[perm] for k, v in st0.items()},
                            (cot[0][rows], cot[1][perm], cot[2][perm]), spw=spw)
            np.testing.assert_array_equal(a["out"][rows], b["out"])
            _same_state({k: None if v is None else v[perm] for k, v in a["state"].items()}, b["state"])
            np.testing.assert_array_equal(a["grads"][0][rows], b["grads"][0])
            np.testing.assert_array_equal(a["grads"][2][perm], b["grads"][2])
            np.testing.assert_array_equal(a["grads"][3][perm], b["grads"][3])


def test_malformed_layouts_touch_nothing_outside_their_buffers():
    """Ranges with offsets[s] < 0, offsets[s] > offsets[s+1] or offsets[s+1] > N: those streams are empty (state untouched, cotangents passed through), the well-formed ones are solved as usual, and no guard
    word around any buffer is written."""
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    lengths = [2, 2, 2, 2]
    _, _, pk, _ = _inputs(o, lengths, seed=97)
    good = P.offsets_of(lengths)
    S, Nf = 4, 8
    st0 = _start(seq, o, S, seed=98)
    cot = _cotangents(seq, S, Nf, seed=99)
    ref = _packed_all(seq, pk, None, lengths, st0, cot)
    for offsets, bad in (([0, 2, -3, 6, 8], {1, 2}), ([0, 2, 9, 6, 8], {1, 2}), ([0, 2, 4, 6, 99], {3}), ([-1, 2, 4, 6, 8], {0})):
        got = _packed_all(seq, pk, None, lengths, st0, cot, offsets=np.array(offsets, np.int64))
        for s in range(S):
            if s in bad:
                for k, v in st0.items():
                    if v is not None:
                        np.testing.assert_array_equal(got["state"][k][s], v[s], err_msg=f"{offsets} stream {s} {k}")
                np.testing.assert_array_equal(got["grads"][2][s], cot[1][s])
                np.testing.assert_array_equal(got["grads"][3][s], cot[2][s])
            else:
                a, b = good[s], good[s + 1]
                np.testing.assert_array_equal(got["out"][a:b], ref["out"][a:b])
                np.testing.assert_array_equal(got["grads"][2][s], ref["grads"][2][s])


def test_zero_frames_do_nothing():
    key = "teleop/allegro_hand_right"
    seq = build_product(key)
    st0 = H.fresh_state(seq, 2)
    st = _copy(st0)
    out, _, _, _ = P.solve_packed(seq, np.zeros((0, 21, 3), np.float32), P.offsets_of([0, 0]), state=st, record=True)
    assert out.shape == (0, seq.optimizer.robot.dof)
    _same_state(st, st0)


def test_raw_landmarks_are_accepted_by_the_unrecorded_forward_only():
    key = "teleop/allegro_hand_right"
    seq, o = build_product(key), build_oracle(key)
    kp, _, pk, _ = _inputs(o, [2, 2], seed=100)
    rot = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], np.float32)  # raw frames: a rotated, shifted hand
    raw = (kp @ rot.T + np.float32(0.3)).astype(np.float32)
    st_a, st_b = H.fresh_state(seq, 2), H.fresh_state(seq, 2)
    out_a, _, _ = emu_host.solve_sequences(seq, raw, state=st_a, raw_hand="right")
    out_b, _, _, _ = P.solve_packed(seq, raw.reshape(-1, 21, 3), P.offsets_of([2, 2]), state=st_b, raw_hand="right")
    np.testing.assert_array_equal(out_a.reshape(4, -1), out_b)
    with pytest.raises(EmulationError, match="pre-processing is not recorded"):
        P.solve_packed(seq, raw.reshape(-1, 21, 3), P.offsets_of([2, 2]), record=True, raw_hand="right")


def test_argument_checks(tmp_path):
    """packed_io_error (shared by the library and the emulation) rejects every malformed buffer set with its message."""
    key = "teleop/leap_hand_right_dexpilot"
    seq, o = build_product(key), build_oracle(key)
    kp = np.zeros((3, 21, 3), np.float32)
    offs = P.offsets_of([1, 2])
    for kw, msg in [(dict(null=("offsets",)), "offsets (device [S+1]) are required"),
                    (dict(num_streams=-1), "bad sizes"),
                    (dict(null=("keypoints",)), "keypoints, last_qpos, robot_qpos_out required"),
                    (dict(null=("last_qpos",)), "keypoints, last_qpos, robot_qpos_out required"),
                    (dict(null=("filter_init",)), "low-pass filter needs filter_state and filter_init"),
                    (dict(record=True, null=("tape_qpos",)), "tape->qpos is required"),
                    (dict(record=True, null=("tape_projected",)), "DexPilot: the flag tape needs"),
                    (dict(record=True, null=("projected",)), "DexPilot: the flag tape needs"),
                    (dict(record=True, raw_hand="right"), "pre-processing is not recorded")]:
        with pytest.raises(EmulationError) as e:
            P.solve_packed(seq, kp, offs, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg, (kw, e.value.msg)
    X, F = np.zeros((3, o.opt_dof), np.float32), np.zeros((3, len(o.projected)), np.uint8)
    last0, finit = np.zeros((2, o.opt_dof), np.float32), np.zeros(2, np.uint8)
    for kw, msg in [(dict(null=("offsets",)), "offsets (device [S+1]) are required"),
                    (dict(num_streams=-1), "bad sizes"),
                    (dict(raw_hand="right"), "pre-processing is not differentiated"),
                    (dict(null=("qpos",)), "qpos (the tape of the forward call) is required"),
                    (dict(null=("projected",)), "DexPilot needs the flag tape")]:
        with pytest.raises(EmulationError) as e:
            P.solve_packed_vjp(seq, kp, offs, X, last0, finit, F, **kw)
        assert e.value.code == N_INVALID and msg in e.value.msg, (kw, e.value.msg)
    seq2, o2 = SC.build(SC.BY_ID["fixed_dense16"], tmp_path)
    with pytest.raises(EmulationError, match="fixed joints but fixed_qpos is NULL"):
        P.solve_packed(seq2, kp, offs, fixed_qpos=np.zeros((3, 2), np.float32), null=("fixed_qpos",))


def test_python_layout_validation():
    torch = pytest.importorskip("torch")  # noqa: F841
    seq = build_product("teleop/allegro_hand_right")
    for bad in ([2, -1], [[1, 2]], [1.5, 2.0]):
        with pytest.raises(ValueError):
            seq.pack_streams(bad)


def test_packed_kernels_do_not_spill(tmp_path):
    """`-Xptxas -v`: every dexr_packed_sequences_kernel and dexr_packed_seq_vjp_kernel instantiation spills nothing."""
    from test_block_kernel_budget import ptxas_log, spill_stores

    if shutil.which("nvcc") is None and not Path("/usr/local/cuda/bin/nvcc").exists():
        pytest.skip("needs nvcc")
    stores = spill_stores(ptxas_log(tmp_path))
    packed = {k: v for k, v in stores.items() if "dexr_packed_" in k}
    assert len(packed) == 10, sorted(packed)
    assert all(v == 0 for v in packed.values()), packed


def test_gpu_packed_file_passes_against_the_emulation():
    """tests/test_gpu_packed_streams.py dry-run on the CPU (tests/tools/emu_gpu_packed.py)."""
    count = 10
    res = subprocess.run([sys.executable, str(ROOT / "tests" / "tools" / "emu_gpu_packed.py")], capture_output=True,
                         text=True, timeout=1800)
    tail = "\n".join(res.stdout.strip().splitlines()[-15:])
    assert res.returncode == 0 and f"{count}/{count} passed" in res.stdout, tail + res.stderr[-2000:]
