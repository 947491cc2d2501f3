"""The CUDA solver's first damped Newton step against the float64 model of tests/newton_model.py, through the public entry
points: retarget_batch with max_iters = 1 and the starting damping per frame (damping), and retarget_sequences with
T = 1 and damping_state, once per sequences mode (one group per stream, and the scarce-streams mode with both 16-lane
half-warps on one stream).  The same frames, qualification and assertions as tests/test_newton_step_emulation.py."""
import numpy as np
import pytest

import newton_model as NM
import structure_cases as SC
from helpers import build_oracle, build_product

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _solve(opt, fr):
    opt.max_iters = 1
    B = len(fr.lam)
    dev = _dev()
    status = torch.zeros(B, dtype=torch.int32, device=dev)
    cost = torch.zeros(B, dtype=torch.float32, device=dev)
    rq = torch.zeros((B, opt.robot.dof), dtype=torch.float32, device=dev)
    proj = None if fr.flags is None else _t(fr.flags.copy())
    q = opt.retarget_batch(ref_value=_t(fr.refs), fixed_qpos=_t(fr.fixed) if fr.fixed.shape[1] else None, last_qpos=_t(fr.last),
                           projected=proj, robot_qpos_out=rq, status_out=status, cost_out=cost, clip_init=fr.clip_init,
                           damping=_t(fr.lam.copy()))
    torch.cuda.synchronize()
    return q.cpu().numpy(), status.cpu().numpy(), cost.cpu().numpy(), rq.cpu().numpy()


def _run(opt, o, regime, label):
    fr = NM.make_frames(o, regime, NM.N[regime], NM.SEEDS[regime])
    q, status, cost, full = _solve(opt, fr)
    NM.assert_regime(o, fr, q, status, cost, full, label)


@pytest.mark.parametrize("key,use_arrow,regime", NM.SHIPPED_RUNS)
def test_gpu_first_step_shipped(key, use_arrow, regime, monkeypatch):
    monkeypatch.setenv("DEXR_ARROW", "1" if use_arrow else "0")
    _run(build_product(key).optimizer, build_oracle(key), regime, key)


@pytest.mark.parametrize("cid,regime", NM.STRUCT_RUNS)
def test_gpu_first_step_structure_cases(cid, regime, tmp_path, monkeypatch):
    monkeypatch.setenv("DEXR_ARROW", "1")
    seq, o = SC.build(SC.BY_ID[cid], tmp_path)
    _run(seq.optimizer, o, regime, cid)


@pytest.mark.parametrize("key,duo", NM.STREAM_RUNS)
def test_gpu_first_step_sequences(key, duo, monkeypatch):
    """T = 1 from a fresh stream state (its low-pass filter passes the first output through), warm starts and damping set
    per stream.  Six streams take one warp each, so DEXR_SEQ_DUO selects the mode of the 16-lane solver."""
    monkeypatch.setenv("DEXR_SEQ_DUO", "1" if duo else "0")
    seq, o = build_product(key), build_oracle(key)
    seq.optimizer.max_iters = 1
    S = 6
    kps, fr = NM.stream_frames(o, S)
    state = seq.make_stream_state(S)
    state.last_qpos = _t(fr.last.copy())
    state.damping = _t(fr.lam.copy())
    if fr.flags is not None:
        state.projected = _t(fr.flags.copy())
    status = torch.zeros((S, 1), dtype=torch.int32, device=_dev())
    out, state = seq.retarget_sequences(_t(kps), state=state, status_out=status)
    torch.cuda.synchronize()
    NM.assert_regime(o, fr, state.last_qpos.cpu().numpy(), status.cpu().numpy()[:, 0], None, out.cpu().numpy()[:, 0],
                     f"{key} sequences duo={duo}")
