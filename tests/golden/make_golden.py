"""Generates the committed golden vectors under tests/golden/*_pop*.npz from the IEEE-strict CPU oracle
(oracle/liboracle_strict.so): they pin the oracle restatement.  The stored answers of the reference's own code,
reference_calls.npz, are recorded differently (tests/golden/README.md).
Run:  python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle_lib  # noqa: E402
from bio_ik_b200 import workloads  # noqa: E402

# name -> (config, batch, population, mode, generations, steps)
CASES = {
    "cfg1_pop64_25steps": ("cfg1", 1, 64, "q", 8, 25),
    "cfg2_pop18_12steps": ("cfg2", 6, 18, "q", 8, 12),
    "cfg2_pop128_25steps": ("cfg2", 4, 128, "q", 8, 25),
    "cfg2_bio2_pop18": ("cfg2", 4, 18, 0, 16, 6),
    "cfg2_memetic_l_pop18": ("cfg2", 4, 18, "l", 8, 6),
    "cfg3_pop128_6steps": ("cfg3", 3, 128, "q", 8, 6),
    "cfg4_pop128_5steps": ("cfg4", 3, 128, "q", 8, 5),
    "cfg5_pop128_5steps": ("cfg5", 3, 128, "q", 8, 5),
    "mimic_virtual_joints_pop40": ("mimic_virtual_joints", 4, 40, "q", 8, 6),
    "tied_preselection_pop128": ("tied_preselection", 3, 128, "q", 8, 4),
}


def custom_workload(oracle, cfgname, B):
    """problems that are not a BASELINE configuration: (workload, problem) built here, goals from the oracle's FK of sampled targets"""
    from bio_ik_b200 import goals as G, robots
    from bio_ik_b200.problem import Problem
    rng = np.random.default_rng(31)
    if cfgname == "mimic_virtual_joints":
        # a PLANAR joint mimicking a prismatic joint, a FLOATING joint mimicking a revolute one (forward_kinematics.h:230-246,698-699)
        rm, groups = robots.mimic_virtual_joint_arm()
        w = workloads.Workload(cfgname, rm, groups["all"], Problem().initialize(rm, groups["all"], [G.PoseGoal("ee"), G.PositionGoal("probe")]), 0, 0, B)
        base = robots.mimic_virtual_joint_base(rm)
    else:
        # cfg2's arm with AvoidJointLimitsGoal as the only secondary goal: most children tie at exactly 0.0 in the pre-selection (:366-378)
        w = workloads.cfg2(B)
        w.problem = Problem().initialize(w.robot, w.group, [G.PoseGoal("r_wrist_roll_link"), G.AvoidJointLimitsGoal(1.0)])
        base = None
    rm, pr = w.robot, w.problem
    w.targets = workloads.sample_configurations(rm, pr.active_variables, B, rng, base=base)
    w.seeds = workloads.sample_configurations(rm, pr.active_variables, B, rng, base=base)
    tips = oracle.fk(rm, pr, w.targets)
    gp = np.repeat(pr.default_goal_params()[None], B, 0)
    gp[:, 0, 0:7] = tips[:, 0, :]
    if cfgname == "mimic_virtual_joints":
        gp[:, 1, 0:3] = tips[:, 1, 0:3]
    w.goal_params = np.ascontiguousarray(gp)
    w.rng_seeds = (1 + np.arange(B)).astype(np.uint32)
    return w


def make_workload(oracle, cfgname, B):
    if cfgname in workloads.CONFIGS:
        return workloads.make(cfgname, lambda rm, pr, v: oracle.fk(rm, pr, v), batch=B)
    return custom_workload(oracle, cfgname, B)


def run_case(oracle, name):
    cfgname, B, pop, mode, gens, steps = CASES[name]
    w = make_workload(oracle, cfgname, B)
    cfg = oracle_lib.make_cfg(population=pop, memetic=mode, generations=gens)
    res = oracle.solve(w.robot, w.problem, cfg, w.goal_params, w.seeds, w.rng_seeds, steps)
    return w, cfg, res


if __name__ == "__main__":
    o = oracle_lib.Oracle()
    for name in CASES:
        w, cfg, res = run_case(o, name)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), goal_params=w.goal_params, seeds=w.seeds, rng_seeds=w.rng_seeds, targets=w.targets, **res)
        print(name, "success", res["success"].tolist(), "fitness", res["fitness"].max())
