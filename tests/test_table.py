"""Robot-table compiler: every reference config compiles; the table's pointer-jumping FK, ancestor masks,
mimic groups and index maps reproduce the float64 model."""
import ctypes as C

import numpy as np
import pytest

from helpers import build_oracle, build_product, configs
from dex_retargeting_b200 import _native as N
from dex_retargeting_b200.table import table_bytes, table_from_bytes

ALL_KEYS = sorted(configs())


def emulate_table_fk(t, q):
    """What the kernel does (dexr_kernels.cuh Solver::fk), in float64 numpy, driven ONLY by the table."""
    dof = t.dof
    R, p = [], []
    for c in range(dof):
        R0, RA, RB = (np.array(x[c][:]).reshape(3, 3) for x in (t.R0, t.RA, t.RB))
        p0, d0 = np.array(t.p0[c][:]), np.array(t.d0[c][:])
        if t.jtype[c] == 0:
            R.append(R0 + np.sin(q[c]) * RA + (1 - np.cos(q[c])) * RB)
            p.append(p0.copy())
        else:
            R.append(R0.copy())
            p.append(p0 + q[c] * d0)
    for r in range(t.n_rounds):
        Rn, pn = [x.copy() for x in R], [x.copy() for x in p]
        for c in range(dof):
            src = (t.jump[c] >> (6 * r)) & 63
            if src != 63:
                Rn[c] = R[src] @ R[c]
                pn[c] = R[src] @ p[c] + p[src]
        R, p = Rn, pn
    return np.array(R), np.array(p)


@pytest.mark.parametrize("key", ALL_KEYS)
def test_every_reference_config_compiles(key):
    seq = build_product(key)
    opt = seq.optimizer
    t = opt.build_table()
    assert t.magic == N.TABLE_MAGIC and t.nbytes == C.sizeof(N.DexrTable) == 8192
    assert t.dof == opt.robot.dof and t.n_var == opt.opt_dof and t.n_fixed == len(opt.idx_pin2fixed)
    # index maps: lane <-> target position
    for k, lane in enumerate(opt.idx_pin2target):
        assert t.var_index[lane] == k
    for k, lane in enumerate(opt.idx_pin2fixed):
        assert t.fixed_index[lane] == k
    # bounds: limits widened by 1e-3 (optimizer.py:59-60), clip limits un-widened
    for k, lane in enumerate(opt.idx_pin2target):
        assert t.lower[lane] == pytest.approx(seq.joint_limits[k, 0] - 1e-3, abs=1e-6)
        assert t.upper[lane] == pytest.approx(seq.joint_limits[k, 1] + 1e-3, abs=1e-6)
        assert t.clip_lo[lane] == pytest.approx(seq.joint_limits[k, 0], abs=1e-6)
    assert table_bytes(table_from_bytes(table_bytes(t))) == table_bytes(t)


@pytest.mark.parametrize("key", ["teleop/allegro_hand_right", "offline/shadow_hand_right", "teleop/schunk_svh_hand_right",
                                 "offline/schunk_svh_hand_left", "teleop/shadow_hand_left_dexpilot", "offline/panda_gripper",
                                 "teleop/inspire_hand_right"])
def test_table_fk_matches_model(key):
    seq = build_product(key)
    opt = seq.optimizer
    t = opt.build_table()
    kin = opt.robot.kin
    rng = np.random.RandomState(2)
    q = rng.uniform(kin.joint_limits[:, 0], kin.joint_limits[:, 1])
    R, p = emulate_table_fk(t, q)
    Rw, pw = kin.forward_kinematics(q)
    np.testing.assert_allclose(R, Rw, atol=2e-6)  # table is float32
    np.testing.assert_allclose(p, pw, atol=2e-6)
    # link slots: parent lane + offset reproduce link positions; ancestor masks match the tree
    anc = kin.is_ancestor_table()
    spec = opt._objective_spec()
    for k, name in enumerate(spec.link_names):
        li = kin.link_index(name)
        par = t.link_parent[k]
        assert par == kin.link_parent[li]
        pos = R[par] @ np.array(t.link_off[k][:]) + p[par] if par >= 0 else np.array(t.link_off[k][:])
        np.testing.assert_allclose(pos, kin.link_pose(Rw, pw, li)[1], atol=3e-6)
        mask = t.link_anc_mask[k]
        for j in range(kin.dof):
            assert bool((mask >> j) & 1) == (par >= 0 and bool(anc[par, j]))
    for c in range(kin.dof):
        for j in range(kin.dof):
            assert bool((t.anc_mask[c] >> j) & 1) == bool(anc[c, j])
            assert bool((t.desc_mask[c] >> j) & 1) == bool(anc[j, c])


@pytest.mark.parametrize("key", ["teleop/schunk_svh_hand_right", "teleop/ability_hand_left", "offline/inspire_hand_right",
                                 "teleop/panda_gripper"])
def test_mimic_tables_match_adaptor(key):
    seq = build_product(key)
    opt = seq.optimizer
    t = opt.build_table()
    a = opt.adaptor
    assert t.has_mimic == 1
    o = build_oracle(key)
    np.testing.assert_array_equal(a.idx_pin2mimic, o.adaptor.idx_pin2mimic)
    np.testing.assert_array_equal(a.idx_pin2source, o.adaptor.idx_pin2source)
    for i, lane in enumerate(a.idx_pin2mimic):
        assert t.mimic_src[lane] == a.idx_pin2source[i]
        assert t.mimic_mult[lane] == pytest.approx(a.multipliers[i])
        assert t.mimic_off[lane] == pytest.approx(a.offsets[i])
        assert t.var_index[lane] == -1 and t.fixed_index[lane] == -1
    # groups: every variable lane lists itself first, then exactly its mimic joints
    for lane in opt.idx_pin2target:
        cnt = t.group_count[lane]
        lanes = [t.group_lane[lane][f] for f in range(cnt)]
        assert lanes[0] == lane and t.group_mult[lane][0] == 1.0
        assert sorted(lanes[1:]) == sorted(int(m) for m, s in zip(a.idx_pin2mimic, a.idx_pin2source) if s == lane)
    # host adaptor == oracle adaptor on qpos and Jacobian folding
    rng = np.random.RandomState(0)
    q = rng.randn(opt.robot.dof)
    np.testing.assert_allclose(a.forward_qpos(q.copy()), o.adaptor.forward_qpos(q.copy()))
    J = rng.randn(3, 3, opt.robot.dof)
    np.testing.assert_allclose(a.backward_jacobian(J.copy()), o.adaptor.backward_jacobian(J.copy()))


def test_objective_spec_indices():
    seq = build_product("teleop/leap_hand_right_dexpilot")
    opt = seq.optimizer
    t = opt.build_table()
    assert (t.loss, t.n_res, t.n_links, t.num_fingers, t.len_proj, t.len_s1) == (2, 10, 5, 4, 6, 3)
    # default human indices = [origin, task] * 4 (optimizer.py:361-364)
    assert [t.res_human_origin[k] for k in range(10)] == [8, 12, 16, 12, 16, 16, 0, 0, 0, 0]
    assert [t.res_human_task[k] for k in range(10)] == [4, 4, 4, 8, 8, 12, 4, 8, 12, 16]
    assert [t.s2_origin[k] for k in range(3)] == [1, 2, 2] and [t.s2_task[k] for k in range(3)] == [0, 0, 1]
    seq = build_product("offline/shadow_hand_right")
    t = seq.optimizer.build_table()
    assert (t.loss, t.n_res, t.dof, t.n_var, t.n_rounds) == (0, 10, 30, 30, 4)
    assert [t.res_human_task[k] for k in range(10)] == [4, 8, 12, 16, 20, 2, 6, 10, 14, 18]
    assert all(t.res_origin[k] == -1 for k in range(10))


def test_table_compiler_errors():
    from dex_retargeting_b200.table import ObjectiveSpec, compile_table

    seq = build_product("teleop/allegro_hand_right")
    opt = seq.optimizer
    kin = opt.robot.kin
    spec = opt._objective_spec()
    with pytest.raises(ValueError):
        compile_table(kin, ["no_such_joint"], spec, np.zeros((1, 2)))
    with pytest.raises(ValueError):
        compile_table(kin, opt.target_joint_names, spec, np.zeros((3, 2)))
    bad = ObjectiveSpec(spec.loss, spec.link_names, spec.res_task, spec.res_origin, [25] * 4, spec.res_human_origin)
    with pytest.raises(ValueError):
        compile_table(kin, opt.target_joint_names, bad, seq.joint_limits)


def test_maximum_size_robot_32_joints_deep_chain(tmp_path):
    """32 movable joints in ONE chain: the lane budget (32) and the pointer-jumping depth (5 rounds) at their
    limits; one more joint must be refused."""
    from synthetic_robots import write_chain
    from dex_retargeting_b200.retargeting_config import RetargetingConfig

    p, cfg = write_chain(tmp_path, 32, prismatic_every=5)
    seq = RetargetingConfig.from_dict(cfg).build()
    opt = seq.optimizer
    t = opt.build_table()
    assert (t.dof, t.n_var, t.n_rounds, t.n_links, t.n_res) == (32, 32, 5, 4, 4)
    kin = opt.robot.kin
    assert kin.joint_depth.max() == 32
    rng = np.random.RandomState(0)
    q = rng.uniform(kin.joint_limits[:, 0], kin.joint_limits[:, 1])
    R, pp = emulate_table_fk(t, q)
    Rw, pw = kin.forward_kinematics(q)
    np.testing.assert_allclose(R, Rw, atol=5e-6)
    np.testing.assert_allclose(pp, pw, atol=5e-6)
    p33, cfg33 = write_chain(tmp_path, 33)
    with pytest.raises(ValueError, match="at most 32"):
        RetargetingConfig.from_dict(cfg33).build().optimizer.build_table()


def test_block_width_detection():
    """Decoupled fingers (palm-fixed origin, no shared movable ancestor) -> block-diagonal Newton system."""
    expect = {"teleop/allegro_hand_right": 4, "teleop/leap_hand_left": 4,          # 4 fingers x 4 joints, wrist origin
              "teleop/allegro_hand_right_dexpilot": 0,                              # finger pairs couple the fingers
              "teleop/shadow_hand_right": 0,                                        # two wrist joints above every finger
              "offline/allegro_hand_right": 0,                                      # dummy free joints above everything
              "teleop/ability_hand_right": 0, "teleop/schunk_svh_hand_right": 0}    # mimic joints: dense path
    for key, bw in expect.items():
        assert build_product(key).optimizer.build_table().block_width == bw, key


def _solver_bw(t):
    """BW of the Solver<G, BW> instantiation the library runs the table on (dexr.cu solver_kind; arrow counts as dense here:
    it does not read the merged schedule)."""
    return 4 if t.dof <= 16 and t.block_width == 4 else 0


def _pass_schedule(t, bw):
    """Mirror of the greedy pass scheduler in load_shared_table (csrc/dexr_kernels.cuh, merged residual passes), built for
    the instantiation Solver<G, bw> that reads it: slots of pass_slot_width<bw>() lanes."""
    gr, nslot = (bw if bw > 0 else 4), 8
    merge = not (t.block_width == 0 and t.has_mimic)
    passes, touched = [], []
    for k in range(t.n_res):
        m = t.link_anc_mask[t.res_task[k]] | (t.link_anc_mask[t.res_origin[k]] if t.res_origin[k] >= 0 else 0)
        sm = sum(1 << sl for sl in range(nslot) if sl * gr < 32 and (m >> (sl * gr)) & ((1 << gr) - 1)) or 1
        if not merge:
            sm = (1 << nslot) - 1
        touched.append(sm)
        r = 0
        while True:
            if r == len(passes):
                passes.append([-1] * nslot)
            if all(passes[r][sl] < 0 for sl in range(nslot) if (sm >> sl) & 1):
                break
            r += 1
        for sl in range(nslot):
            if (sm >> sl) & 1:
                passes[r][sl] = k
    return passes, touched


def test_merged_residual_passes_are_a_valid_schedule():
    """What the merged residual pass (SharedTable::pass_res) relies on, for every shipped configuration:
    each residual sits in exactly one pass and there owns every lane slot it touches (so all lanes that hold a non-zero
    Jacobian column for it work on it together, and the columns a lane reads belong to its own residual)."""
    counts = {}
    for key in sorted(configs()):
        t = build_product(key).optimizer.build_table()
        passes, touched = _pass_schedule(t, _solver_bw(t))
        assert len(passes) <= t.n_res
        for k in range(t.n_res):
            where = [(r, sl) for r, row in enumerate(passes) for sl, v in enumerate(row) if v == k]
            assert len({r for r, _ in where}) == 1, (key, k)
            assert sum(1 << sl for _, sl in where) == touched[k], (key, k)
        if t.block_width > 0:  # block mode: a residual touches exactly one window
            assert all(bin(sm).count("1") == 1 for sm in touched), key
        counts[key] = len(passes)
    assert counts["teleop/allegro_hand_right"] == 1 and counts["teleop/leap_hand_left"] == 1     # 4 fingertip vectors, 4 fingers
    assert counts["teleop/leap_hand_right_dexpilot"] == 4 and counts["teleop/allegro_hand_right_dexpilot"] == 4  # 3 rounds of pairs + wrist
    assert counts["teleop/ability_hand_right"] == 5       # mimic joints: no merging
    assert counts["offline/shadow_hand_right"] == 10      # every residual touches the free-flying base


def test_merged_residual_passes_on_synthetic_robots(tmp_path):
    """The same schedule properties for the synthetic robots of tests/structure_cases.py, block width 8 among them: a
    width-8 table runs on a dense instantiation, so its schedule has 4-lane slots (a residual of an 8-lane window owns
    both slots of the window)."""
    import structure_cases as SC

    for case in SC.CASES:
        seq, _ = SC.build(case, tmp_path)
        t = seq.optimizer.build_table()
        passes, touched = _pass_schedule(t, _solver_bw(t))
        for k in range(t.n_res):
            where = [(r, sl) for r, row in enumerate(passes) for sl, v in enumerate(row) if v == k]
            assert len({r for r, _ in where}) == 1, (case.id, k)
            assert sum(1 << sl for _, sl in where) == touched[k], (case.id, k)
        if t.block_width == 8:
            assert _solver_bw(t) == 0 and any(bin(sm).count("1") == 2 for sm in touched), case.id
        assert len(passes) <= t.n_res, case.id


def test_library_rejects_inconsistent_block_width():
    import ctypes as C

    lib = N.load()
    h = C.c_void_p()
    t = build_product("teleop/shadow_hand_right").optimizer.build_table()
    t.block_width = 4  # the wrist joints are ancestors of every finger: not block diagonal
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1
    assert b"block_width" in lib.dexr_last_error()
    t = build_product("teleop/allegro_hand_right_dexpilot").optimizer.build_table()
    t.block_width = 4  # pair vectors couple two fingers
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1
    assert b"couples two windows" in lib.dexr_last_error()
    t.block_width = 5
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1


def test_arrow_detection():
    """A trunk (free-flying base and / or wrist) above decoupled fingers -> arrow factorisation (1 + trunk lanes)."""
    expect = {"offline/shadow_hand_right": 9,            # 6 dummy joints + WRJ2 + WRJ1, fingers 4/5/4/4/5
              "teleop/shadow_hand_left": 3,               # WRJ2 + WRJ1
              "offline/allegro_hand_right": 7, "offline/leap_hand_left": 7,   # 6 dummy joints, 4 fingers x 4
              "teleop/shadow_hand_right_dexpilot": 0,     # finger-pair vectors couple the fingers
              "teleop/allegro_hand_right": 0,             # block diagonal already (block_width 4)
              "offline/schunk_svh_hand_right": 0, "offline/inspire_hand_left": 0,  # mimic joints: dense path
              "teleop/leap_hand_right_dexpilot": 0}
    for key, arrow in expect.items():
        t = build_product(key).optimizer.build_table()
        assert t.arrow == arrow, key
        assert not (t.arrow and t.block_width)


def test_library_rejects_inconsistent_arrow():
    import ctypes as C

    lib = N.load()
    h = C.c_void_p()
    t = build_product("teleop/shadow_hand_right_dexpilot").optimizer.build_table()
    t.arrow = 3  # pair vectors couple two fingers
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1
    assert b"couples two fingers" in lib.dexr_last_error()
    t = build_product("teleop/shadow_hand_right").optimizer.build_table()
    t.arrow = 2  # WRJ1 would head a "finger" of 23 joints
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1
    assert b"arrow" in lib.dexr_last_error()
    t = build_product("offline/schunk_svh_hand_right").optimizer.build_table()
    t.arrow = 7  # mimic joints
    assert lib.dexr_robot_create(C.byref(t), 0, C.byref(h)) == -1
    assert b"inconsistent" in lib.dexr_last_error()
