"""The solver's first damped Newton step (host emulation of the solver source, tests/emu) against the float64 model of
tests/newton_model.py, on every solver instantiation and mode.

With max_iters = 1 and the starting damping given per frame (damping_io), the returned point is the first trial's
clip(x + s, lo, hi).  On every qualifying frame (no rejected trial, A_ff clear of the positive-definite fallback, no bound
variable near the active-set threshold) it must equal the model's step to tau of the step's length; active variables
stay where they started bit for bit; the status counts one iteration; the reported cost is the consistent objective at
the returned point (away from a minimiser); the full joint vector is the mimic map of the returned point.  These pin
the Newton system itself -- loss curvature, kinematic curvature, mimic fold, factorisations, damping shift, active set --
which the converged-minimiser tests cannot see: a wrong term there only costs iterations."""
import numpy as np
import pytest

import emu_host
import newton_model as NM
import structure_cases as SC
from helpers import build_oracle, build_product


def _solve(opt, fr, use_arrow):
    opt.max_iters = 1
    proj = None if fr.flags is None else fr.flags.copy()
    return emu_host.solve_frames(opt, fr.last, ref_value=fr.refs, fixed_qpos=fr.fixed if fr.fixed.size else None, projected=proj,
                                 use_arrow=use_arrow, clip_init=fr.clip_init, want_robot_qpos=True, damping=fr.lam.copy())


def _run(opt, o, regime, use_arrow, label):
    fr = NM.make_frames(o, regime, NM.N[regime], NM.SEEDS[regime])
    q, status, cost, full = _solve(opt, fr, use_arrow)
    NM.assert_regime(o, fr, q, status, cost, full, label)


@pytest.mark.parametrize("key,use_arrow,regime", NM.SHIPPED_RUNS)
def test_first_step_shipped(key, use_arrow, regime):
    _run(build_product(key).optimizer, build_oracle(key), regime, use_arrow, key)


@pytest.mark.parametrize("cid,regime", NM.STRUCT_RUNS)
def test_first_step_structure_cases(cid, regime, tmp_path):
    seq, o = SC.build(SC.BY_ID[cid], tmp_path)
    _run(seq.optimizer, o, regime, True, cid)


@pytest.mark.parametrize("key,duo", NM.STREAM_RUNS)
def test_first_step_sequences(key, duo):
    """dexr_sequences_kernel with T = 1: the warm start comes from the stream state (clipped), the damping from
    damping_state; the low-pass filter of a fresh stream passes its first output through unchanged.  `duo`: the
    scarce-streams mode of the 16-lane solver, both half-warps on one stream and g / H summed across them."""
    seq, o = build_product(key), build_oracle(key)
    seq.optimizer.max_iters = 1
    S = 6
    kps, fr = NM.stream_frames(o, S)
    state = dict(last_qpos=fr.last.copy(), filter_state=np.zeros((S, o.robot.dof), np.float32), filter_init=np.zeros(S, np.uint8),
                 projected=None if fr.flags is None else fr.flags.copy(), damping=fr.lam.copy())
    out, status, state = emu_host.solve_sequences(seq, kps, state=state, duo=duo)
    NM.assert_regime(o, fr, state["last_qpos"], status[:, 0], None, out[:, 0], f"{key} sequences duo={duo}")
