"""Synthetic robots at the edges of the robot-table format (include/dexr.h, dex_retargeting_b200/table.py), shared by the
host emulation (tests/test_structures_emulation.py) and the GPU suite (tests/test_gpu_structures.py).

Every case states the table features it exists for.  `check_features` holds the compiled table to all of them, so a case
that drifts to another solver instantiation or loses the feature it covers fails instead of silently testing something
else; dropping a case drops a visible line here."""
from dataclasses import dataclass, field

import numpy as np

from synthetic_robots import write_tree_hand


@dataclass(frozen=True)
class Case:
    id: str
    trunk: int
    widths: tuple
    kind: str
    expect: dict  # dof, block_width, arrow, n_fixed, has_mimic, group (max group_count), per_lane (max links per lane), n_links, n_res
    opts: dict = field(default_factory=dict)  # write_tree_hand options: prismatic, mimic, extra_links, fixed


def _e(dof, bw, arrow, n_fixed, mimic, group, per_lane, n_links, n_res):
    return dict(dof=dof, block_width=bw, arrow=arrow, n_fixed=n_fixed, has_mimic=mimic, group=group, per_lane=per_lane,
                n_links=n_links, n_res=n_res)


CASES = [
    # ---- block width 8: decoupled fingers that fit 8-lane windows but not 4-lane ones (factorised densely)
    Case("bw8_5344_position", 0, (5, 3, 4, 4), "position", _e(16, 8, 0, 0, 0, 1, 1, 4, 4)),
    Case("bw8_88_vector", 0, (8, 8), "vector", _e(16, 8, 0, 0, 0, 1, 1, 3, 2)),
    Case("bw8_888_vector", 0, (8, 8, 8), "vector", _e(24, 8, 0, 0, 0, 1, 1, 4, 3)),
    Case("bw8_6288_position", 0, (6, 2, 8, 8), "position", _e(24, 8, 0, 0, 0, 1, 1, 4, 4)),
    # ---- several objective links on one joint (2, 3 and 4 = DEXR_MAX_LINKS_PER_LANE)
    Case("links_block4_position", 0, (4, 4, 4, 4), "position", _e(16, 4, 0, 0, 0, 1, 4, 10, 10),
         dict(extra_links={"f0_j3": 3, "f1_j1": 2, "f2_j2": 1})),
    Case("links_block4_vector", 0, (4, 4, 4, 4), "vector", _e(16, 4, 0, 0, 0, 1, 4, 12, 9),
         dict(extra_links={"f0_j3": 3, "f2_j2": 2})),
    Case("links_dense16_max_position", 1, (5, 5, 5), "position", _e(16, 0, 0, 0, 0, 1, 4, 16, 16),  # n_links = n_res = 16
         dict(extra_links={"f0_j4": 3, "f1_j4": 3, "f2_j4": 2, "f1_j1": 2, "f2_j2": 2, "a_trunk0": 1})),
    Case("links_dense16_vector", 1, (5, 5, 5), "vector", _e(16, 0, 0, 0, 0, 1, 4, 11, 8),
         dict(extra_links={"f0_j2": 4, "f2_j3": 1})),
    Case("links_arrow_vector", 2, (4, 5, 4, 4), "vector", _e(19, 0, 3, 0, 0, 1, 4, 14, 10),
         dict(extra_links={"f0_j3": 3, "f1_j2": 2, "f3_j1": 1})),
    Case("links_arrow_position", 2, (4, 5, 4, 4), "position", _e(19, 0, 3, 0, 0, 1, 4, 10, 10),
         dict(extra_links={"f1_j4": 3, "f3_j2": 2, "a_trunk1": 1})),
    Case("links_dense32_position", 9, (3, 3, 3), "position", _e(18, 0, 0, 0, 0, 1, 4, 9, 9),  # 9 trunk joints: no arrow
         dict(extra_links={"f0_j2": 3, "f1_j1": 2, "a_trunk8": 1})),
    # ---- joints held by the caller (fixed_qpos), in a finger and in the trunk
    Case("fixed_dense16", 1, (5, 5, 5), "position", _e(16, 0, 0, 2, 0, 1, 1, 3, 3), dict(fixed=("a_trunk0", "f1_j2"))),
    Case("fixed_dense32", 2, (4, 5, 4, 4), "vector", _e(19, 0, 0, 3, 0, 1, 1, 5, 4), dict(fixed=("a_trunk1", "f2_j0", "f3_j3"))),
    # ---- mimic joints
    Case("mimic_dense16", 1, (5, 5, 5), "position", _e(16, 0, 0, 0, 1, 4, 1, 3, 3), dict(
        prismatic=("f2_j1", "f2_j2"),
        mimic={"f0_j2": ("f0_j1", -0.7, 0.1), "f0_j3": ("f0_j1", 0.5, -0.05), "f0_j4": ("f0_j1", 1.2, 0.0),  # group of 4
               "f1_j0": ("f1_j3", 0.8, 0.0),            # source after its mimic joint
               "f2_j4": ("f1_j2", -0.5, 0.3),           # across fingers
               "f2_j2": ("f2_j1", 0.6, 0.004),          # prismatic mimics prismatic
               "a_trunk0": ("f2_j0", 0.3, 0.0)})),      # a trunk joint that mimics a finger joint
    Case("mimic_dense32", 2, (4, 5, 4, 4), "vector", _e(19, 0, 0, 0, 1, 4, 1, 5, 4), dict(
        prismatic=("f2_j1", "f2_j3"),
        mimic={"f1_j2": ("f1_j0", -1.0, 0.2), "f1_j3": ("f1_j0", 0.4, 0.0), "f1_j4": ("f1_j0", -0.3, -0.1),  # group of 4
               "f0_j3": ("a_trunk0", 0.6, 0.05),        # mimic of a trunk joint
               "a_trunk1": ("f3_j1", 0.5, 0.0),         # trunk joint driven by a later finger joint
               "f2_j1": ("f2_j3", 0.7, -0.002),         # prismatic, source after its mimic joint
               "f3_j3": ("f2_j0", 0.9, 0.1)})),         # across fingers
    Case("mimic_fixed_dense16", 1, (5, 5, 5), "vector", _e(16, 0, 0, 2, 1, 3, 1, 4, 3), dict(
        mimic={"f0_j3": ("f0_j1", -0.8, 0.2), "f0_j4": ("f0_j1", 0.6, 0.0), "f2_j1": ("f1_j1", 1.1, -0.1)},
        fixed=("a_trunk0", "f1_j4"))),
    Case("mimic_fixed_dense32", 2, (4, 5, 4, 4), "position", _e(19, 0, 0, 2, 1, 3, 1, 4, 4), dict(
        mimic={"f1_j3": ("f1_j1", -0.6, 0.15), "f1_j4": ("f1_j1", 0.5, 0.0), "f3_j0": ("a_trunk1", 0.4, 0.0)},
        fixed=("a_trunk0", "f2_j2"))),
    # ---- sizes and joint types
    Case("dof1_vector", 0, (1,), "vector", _e(1, 0, 0, 0, 0, 1, 1, 2, 1)),
    Case("dof3_position", 0, (3,), "position", _e(3, 0, 0, 0, 0, 1, 1, 2, 2), dict(extra_links={"f0_j1": 1})),
    Case("dof17_position", 1, (4, 4, 4, 4), "position", _e(17, 0, 2, 0, 0, 1, 1, 4, 4)),
    Case("dof31_vector", 9, (8, 7, 7), "vector", _e(31, 0, 0, 0, 0, 1, 1, 4, 3)),
    Case("prismatic_block4", 0, (4, 4, 4, 4), "position", _e(16, 4, 0, 0, 0, 1, 1, 4, 4), dict(prismatic=("f1_j2", "f3_j0"))),
    Case("prismatic_arrow", 2, (4, 5, 4, 4), "vector", _e(19, 0, 3, 0, 0, 1, 1, 5, 4), dict(prismatic=("f1_j3", "f3_j0"))),
    # ---- DexPilot on small hands: len_proj 1 / len_s1 1 and len_proj 3 / len_s1 2
    Case("dexpilot_2fingers", 1, (4, 4), "dexpilot", _e(9, 0, 0, 0, 0, 1, 1, 3, 3)),
    Case("dexpilot_3fingers", 0, (4, 4, 4), "dexpilot", _e(12, 0, 0, 0, 0, 1, 1, 4, 6)),
]
BY_ID = {c.id: c for c in CASES}


def table_features(t):
    per_lane = max(sum(1 for k in range(t.n_links) if t.link_parent[k] == c) for c in range(t.dof))
    return dict(dof=t.dof, block_width=t.block_width, arrow=t.arrow, n_fixed=t.n_fixed, has_mimic=t.has_mimic,
                group=max(t.group_count[c] for c in range(t.dof)), per_lane=per_lane, n_links=t.n_links, n_res=t.n_res)


def solver_kind(t, use_arrow=True):
    """The Solver<G, BW> instantiation the library dispatches the table to (dexr.cu solver_kind)."""
    if t.dof <= 16:
        return "<16,4>" if t.block_width == 4 else "<16,0>"
    return "<32,-1>" if t.arrow > 0 and use_arrow else "<32,0>"


def build(case, tmp_path, override=None):
    """(SeqRetargeting of the product, OracleOptimizer) for the case, with the table checked against its features.
    `override`: configuration entries to change (as for helpers.build_product), e.g. {"low_pass_alpha": -1.0}."""
    from dex_retargeting_b200.retargeting_config import RetargetingConfig
    from oracle.objectives import OracleOptimizer

    d = tmp_path / case.id
    d.mkdir(parents=True, exist_ok=True)
    _, cfg = write_tree_hand(d, case.trunk, case.widths, kind=case.kind, name=case.id, **case.opts)
    seq = RetargetingConfig.from_dict(dict(cfg), override).build()
    o = OracleOptimizer(dict(cfg), str(d), override)
    assert o.robot.dof_joint_names == seq.optimizer.robot.dof_joint_names
    check_features(case, seq.optimizer.build_table())
    return seq, o


def check_features(case, t):
    assert table_features(t) == case.expect, (case.id, table_features(t))


def problems(o, n, seed=4):
    """Warm-start problems (0.05 rad noise, 3 mm target noise) with fixed joints drawn per frame inside their limits."""
    from helpers import synth_problems

    refs, fixed, x0, _ = synth_problems(o, n, np.random.RandomState(seed), init_noise=0.05, target_noise=0.003)
    if o.type == "dexpilot":  # pinches: finger-pair targets inside project_dist (every 3rd frame) and inside the hysteresis
        from oracle.solvers import solve_converged  # band between project_dist and escape_dist (the frames after those)

        lp = len(o.projected)
        flags = initial_flags(o, n)
        rng = np.random.RandomState(seed + 1)
        for i in range(n):
            if i % 3 < 2:
                d = np.linalg.norm(refs[i, :lp], axis=1, keepdims=True)
                refs[i, :lp] *= np.float32(0.02 if i % 3 == 0 else 0.04) / d
            if flags[i].any():  # a stream that already pinched in its previous frame starts near the pinch
                o.projected[:] = flags[i].astype(bool)
                xb = solve_converged(o, refs[i], fixed[i], x0[i], update_state=False)[0]
                x0[i] = np.clip(xb + 0.01 * rng.randn(len(xb)), o.joint_limits[:, 0], o.joint_limits[:, 1])
        o.projected[:] = False
    return refs, fixed, x0


def initial_flags(o, n):
    """DexPilot flags the frames start with: set on every other frame (a pinch seen in the stream's previous frame)."""
    return np.array([[i % 2] * len(o.projected) for i in range(n)], np.uint8) if o.type == "dexpilot" else None
