"""Programmatically generated robot descriptions for edge-case tests (maximum sizes, deep chains)."""
import json

import numpy as np


def serial_chain(n_joints=32, seed=0, prismatic_every=0):
    """A single open chain of `n_joints` movable joints with varied axes / offsets and a tip link every 8 joints."""
    rng = np.random.RandomState(seed)
    links = ["base"]
    joints = []
    axes = [[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [0, -1.0, 0], [0.6, 0.8, 0.0]]
    for i in range(n_joints):
        links.append(f"l{i}")
        jt = "prismatic" if prismatic_every and (i % prismatic_every == prismatic_every - 1) else "revolute"
        joints.append(dict(name=f"j{i:02d}", type=jt, parent="base" if i == 0 else f"l{i - 1}", child=f"l{i}",
                           xyz=[0.0, 0.0, 0.03] if i else [0.0, 0.0, 0.0], rpy=[float(rng.uniform(-0.3, 0.3)), 0.0, float(rng.uniform(-0.3, 0.3))],
                           axis=axes[i % len(axes)], limit=[-0.1, 0.1] if jt == "prismatic" else [-0.6, 0.6]))
        if i % 8 == 7:
            links.append(f"tip{i}")
            joints.append(dict(name=f"fix{i:02d}", type="fixed", parent=f"l{i}", child=f"tip{i}", xyz=[0.01, 0.0, 0.02],
                               rpy=[0.0, 0.0, 0.0], axis=[1.0, 0, 0]))
    return dict(name=f"chain{n_joints}", links=links, joints=joints)


def write_chain(tmp_path, n_joints=32, seed=0, prismatic_every=0):
    desc = serial_chain(n_joints, seed, prismatic_every)
    p = tmp_path / f"chain{n_joints}.json"
    p.write_text(json.dumps(desc))
    tips = [f"tip{i}" for i in range(7, n_joints, 8)]
    cfg = dict(type="position", urdf_path=str(p), target_link_names=tips, target_link_human_indices=[4 * (k + 1) for k in range(len(tips))],
               low_pass_alpha=1.0)
    return p, cfg


def _joint_names(trunk, widths):
    """Movable joint names in pinocchio's depth-first order (= lane order): trunk, then finger 0, finger 1, ..."""
    return [f"a_trunk{i}" for i in range(trunk)] + [f"f{f}_j{i}" for f, w in enumerate(widths) for i in range(w)]


def _child_link(joint):
    return f"trunk{joint[7:]}" if joint.startswith("a_trunk") else joint.replace("_j", "_l")


def tree_hand(trunk=2, widths=(4, 5, 4, 4, 5), seed=0, prismatic=(), mimic=None, extra_links=None):
    """A hand-shaped tree: a chain of `trunk` joints from the base, then one chain of widths[f] joints per finger, all
    attached to the last trunk link, each ending in a tip link.  Joint names sort so that pinocchio's depth-first order is
    trunk first, then finger 0, finger 1, ... (contiguous lanes).

    prismatic:   names of joints made prismatic (limits in metres);
    mimic:       {joint: (source joint, multiplier, offset)}, written as the JSON reader's `mimic` entry;
    extra_links: {joint: count} fixed child links riding on that joint at distinct offsets, named `<joint>_x<k>` (objective
                 links beyond the tips: write_tree_hand puts them into the objective)."""
    rng = np.random.RandomState(seed)
    axes = [[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [0, -1.0, 0], [0.6, 0.8, 0.0]]
    prismatic, mimic, extra_links = set(prismatic), dict(mimic or {}), dict(extra_links or {})
    unknown = (prismatic | set(mimic) | set(extra_links)) - set(_joint_names(trunk, widths))
    assert not unknown, unknown
    links, joints = ["base"], []

    def add(name, parent, child, xyz, rpy, axis, limit):
        links.append(child)
        jt = "prismatic" if name in prismatic else "revolute"
        j = dict(name=name, type=jt, parent=parent, child=child, xyz=xyz, rpy=rpy, axis=axis,
                 limit=[-0.02, 0.03] if jt == "prismatic" else limit)
        if name in mimic:
            j["mimic"] = [mimic[name][0], float(mimic[name][1]), float(mimic[name][2])]
        joints.append(j)
        for k in range(extra_links.get(name, 0)):  # fixed riders, one offset per rider
            links.append(f"{name}_x{k}")
            joints.append(dict(name=f"{name}_x{k}fix", type="fixed", parent=child, child=f"{name}_x{k}",
                               xyz=[0.012 * (k + 1), -0.006 * k, 0.01 + 0.004 * k], rpy=[0.0, 0.0, 0.0], axis=[1.0, 0, 0]))

    parent = "base"
    for i in range(trunk):
        add(f"a_trunk{i}", parent, f"trunk{i}", [0.0, 0.0, 0.02 if i else 0.0], [float(rng.uniform(-0.2, 0.2)), 0.0, 0.0],
            axes[i % 5], [-0.5, 0.5])
        parent = f"trunk{i}"
    palm = parent
    tips = []
    for f, w in enumerate(widths):
        ang = (f - (len(widths) - 1) / 2) * 0.35
        par = palm
        for i in range(w):
            xyz = [0.03 * float(np.sin(ang)), 0.01 * f, 0.05 * float(np.cos(ang))] if i == 0 else [0.0, 0.0, 0.028]
            add(f"f{f}_j{i}", par, f"f{f}_l{i}", xyz, [0.0, float(rng.uniform(-0.2, 0.2)), ang if i == 0 else 0.0],
                axes[(f + i) % 5], [-0.2, 1.2])
            par = f"f{f}_l{i}"
        links.append(f"f{f}_tip")
        joints.append(dict(name=f"f{f}_tipfix", type="fixed", parent=par, child=f"f{f}_tip", xyz=[0.0, 0.0, 0.025], rpy=[0.0, 0.0, 0.0],
                           axis=[1.0, 0, 0]))
        tips.append(f"f{f}_tip")
    return dict(name=f"tree{trunk}_" + "".join(str(w) for w in widths), links=links, joints=joints), tips


def write_tree_hand(tmp_path, trunk, widths, seed=0, kind="position", prismatic=(), mimic=None, extra_links=None, fixed=(),
                    name=None):
    """Robot description + retargeting config of a tree_hand.

    kind "position": tips and extra links are points.  "vector": tips from the base, every extra link of finger f from that
    finger's first link f<f>_l0 (extra links on a trunk joint: from the base).  "dexpilot": the tips are the fingers, the
    palm (last trunk link, or the base) is the wrist.
    fixed: joints left out of target_joint_names -- the caller supplies them per frame (fixed_qpos).  Mimic joints are
    never targets."""
    mimic = dict(mimic or {})
    desc, tips = tree_hand(trunk, widths, seed, prismatic, mimic, extra_links)
    if name:
        desc["name"] = name
    p = tmp_path / f"{desc['name']}.json"
    p.write_text(json.dumps(desc))
    extras = [(j, f"{j}_x{k}") for j in _joint_names(trunk, widths) for k in range((extra_links or {}).get(j, 0))]
    cfg = dict(urdf_path=str(p), low_pass_alpha=1.0)
    held = set(fixed) | set(mimic)
    if held:
        cfg["target_joint_names"] = [j for j in _joint_names(trunk, widths) if j not in held]
    hi = [min(20, 4 * (k + 1)) for k in range(len(tips))] + [1 + k % 20 for k in range(len(extras))]
    if kind == "position":
        cfg.update(type="position", target_link_names=tips + [x for _, x in extras], target_link_human_indices=hi)
    elif kind == "vector":
        origins = ["base"] * len(tips) + [(j.split("_")[0] + "_l0") if j.startswith("f") else "base" for j, _ in extras]
        hi_origin = [0 if o == "base" else 1 + (k + 7) % 20 for k, o in enumerate(origins)]
        cfg.update(type="vector", target_origin_link_names=origins, target_task_link_names=tips + [x for _, x in extras],
                   target_link_human_indices=[hi_origin, hi], scaling_factor=1.0)
    else:
        assert kind == "dexpilot" and not extras
        cfg.update(type="dexpilot", finger_tip_link_names=tips, wrist_link_name=f"trunk{trunk - 1}" if trunk else "base",
                   scaling_factor=1.0)
    return p, cfg
