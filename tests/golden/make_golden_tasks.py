"""Golden vectors for the Walk / ObjHold / Reach task logic, produced by RUNNING THE REFERENCE'S OWN CLASSES
(WalkEnvV0 / ObjHoldFixedEnvV0 / ReachEnvV0 get_obs_dict, get_reward_dict and helpers, unmodified, created with __new__ so that no
simulator is constructed) on mj_data-like records filled from this repo's CPU oracle.  Output: tests/golden/tasks.npz
Run with a MyoSuite checkout (MYOSUITE_CHECKOUT=<its root>) and oracle/libmyo_oracle.so built:  python tests/golden/make_golden_tasks.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE); sys.path.insert(0, ROOT)
import _ref_stubs  # noqa: E402

_ref_stubs.install()
from myosuite.envs.myo.myobase.obj_hold_v0 import ObjHoldFixedEnvV0  # noqa: E402
from myosuite.envs.myo.myobase.reach_v0 import ReachEnvV0  # noqa: E402
from myosuite.envs.myo.myobase.walk_v0 import WalkEnvV0  # noqa: E402
from myosuite.envs.obs_vec_dict import ObsVecDict  # noqa: E402

from myosuite_b200 import assets, blob  # noqa: E402
from oracle.oracle_py import Oracle  # noqa: E402

out = {}
rng = np.random.default_rng(77)


def fake_model(m):
    fm = types.SimpleNamespace(na=m.na, nu=m.nu, body_mass=m.body_mass, jnt_qposadr=m.jnt_qposadr, key_qpos=m.key_qpos,
                               opt=types.SimpleNamespace(timestep=m.opt_timestep))
    fm.body = lambda name: types.SimpleNamespace(id=m.name2id("body", name))
    fm.joint = lambda name: types.SimpleNamespace(id=m.name2id("joint", name))
    fm.site = lambda name: types.SimpleNamespace(id=m.name2id("site", name))
    return fm


def fake_data(o, nb):
    return types.SimpleNamespace(time=0.0, qpos=o.f("qpos").copy(), qvel=o.f("qvel").copy(), act=o.f("act").copy(), xpos=o.f("xpos").reshape(nb, 3).copy(),
                                 xquat=o.f("xquat").reshape(nb, 4).copy(), xipos=o.f("xipos").reshape(nb, 3).copy(), cvel=o.f("cvel").reshape(nb, 6).copy(),
                                 actuator_length=o.f("actuator_length").copy(), actuator_velocity=o.f("actuator_velocity").copy(),
                                 actuator_force=o.f("actuator_force").copy(), site_xpos=o.f("site_xpos").reshape(-1, 3).copy())


# ---- Walk: states = keyframes + noise, a few oracle steps in between to get velocities / muscle states
m = assets.load("myolegs")
o = Oracle(*blob.pack(m))
N = 24
S = dict(qpos=[], qvel=[], act=[], steps=[], obs=[], dense=[], done=[], vel_reward=[], cyclic_hip=[], ref_rot=[], joint_angle_rew=[])
for i in range(N):
    o.reset()
    q = m.key_qpos[i % 4].copy(); q[7:] += rng.normal(0, 0.05, m.nq - 7)
    if i >= 16:                                      # tilted / low states so that the done branches fire
        q[2] = 0.7 if i % 2 else 0.95
        ang = rng.uniform(0.5, 1.4); q[3:7] = [np.cos(ang / 2), 0, np.sin(ang / 2) * (i % 2), np.sin(ang / 2) * (1 - i % 2)]
    o.set(qpos=q, qvel=rng.normal(0, 0.5, m.nv), act=rng.uniform(0, 1, m.na), ctrl=np.zeros(m.nu))
    o.forward()                                      # the reference's observed data: forward on the state with ctrl = 0 (robot.py:595-607)
    steps = int(rng.integers(0, 300))
    env = WalkEnvV0.__new__(WalkEnvV0)
    env.mj_model, env.mj_data = fake_model(m), fake_data(o, m.nbody)
    env.frame_skip, env.steps, env.hip_period, env.min_height, env.max_rot = 10, steps, 100, 0.8, 0.8      # dt = timestep * frame_skip = 0.01
    env.target_x_vel, env.target_y_vel, env.target_rot, env.init_qpos = 0.0, 1.2, None, m.key_qpos[0].copy()
    env.rwd_keys_wt = WalkEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS
    od = env.get_obs_dict(env.mj_model, env.mj_data)
    env.obs_dict = od
    ovd = ObsVecDict()
    t, vec = ovd.obsdict2obsvec(od, WalkEnvV0.DEFAULT_OBS_KEYS + ["act"])      # base_v0.py:33-37 appends "act"
    rd = env.get_reward_dict(od)
    S["qpos"].append(o.f("qpos").copy()); S["qvel"].append(o.f("qvel").copy()); S["act"].append(o.f("act").copy()); S["steps"].append(steps); S["obs"].append(vec)
    for k in ("dense", "done", "vel_reward", "cyclic_hip", "ref_rot", "joint_angle_rew"):
        S[k].append(float(np.asarray(rd[k]).ravel()[0]))
for k, v in S.items():
    out["walk_" + k] = np.array(v)
assert out["walk_obs"].shape == (N, 403) and out["walk_obs"].dtype == np.float32 and out["walk_done"].sum() >= 2

# ---- ObjHold
m = assets.load("myohand_hold")
o = Oracle(*blob.pack(m))
N = 16
H = dict(qpos=[], qvel=[], act=[], goal=[], obs=[], dense=[], done=[])
for i in range(N):
    o.reset()
    q = m.qpos0.copy(); q[:-7] = rng.uniform(m.jnt_range[:23, 0], m.jnt_range[:23, 1]); q[-7:-4] += rng.normal(0, 0.01 if i < 12 else 0.4, 3)
    o.set(qpos=q, qvel=rng.normal(0, 0.5, m.nv), act=rng.uniform(0, 1, m.na)); o.forward()
    goal = np.array([-.240, -.520, 1.470]) + rng.uniform(-0.03, 0.03, 3)
    env = ObjHoldFixedEnvV0.__new__(ObjHoldFixedEnvV0)
    env.mj_model, env.mj_data, env.frame_skip = fake_model(m), fake_data(o, m.nbody), 10                 # dt = 0.02
    env.object_sid, env.goal_sid = m.name2id("site", "object"), m.name2id("site", "goal")
    env.mj_data.site_xpos[env.goal_sid] = goal
    env.rwd_keys_wt = ObjHoldFixedEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS
    od = env.get_obs_dict(env.mj_model, env.mj_data)
    env.obs_dict = od
    t, vec = ObsVecDict().obsdict2obsvec(od, ObjHoldFixedEnvV0.DEFAULT_OBS_KEYS + ["act"])
    rd = env.get_reward_dict(od)
    H["qpos"].append(o.f("qpos").copy()); H["qvel"].append(o.f("qvel").copy()); H["act"].append(o.f("act").copy()); H["goal"].append(goal); H["obs"].append(vec)
    H["dense"].append(float(np.asarray(rd["dense"]).ravel()[0])); H["done"].append(float(np.asarray(rd["done"]).ravel()[0]))
for k, v in H.items():
    out["hold_" + k] = np.array(v)
assert out["hold_obs"].shape == (N, 91) and out["hold_done"].sum() >= 1

# ---- Reach (myoHandReachRandom-v0: hand model, five finger tips; registry kwargs from the reference's own registration)
import json  # noqa: E402
reg = json.load(open(os.path.join(ROOT, "myosuite_b200", "assets", "registry.json")))["envs"]["myoHandReachRandom-v0"]["kwargs"]
m = assets.load("myohand_pose")
o = Oracle(*blob.pack(m))
tips = list(reg["target_reach_range"].keys())
N = 20
R = dict(qpos=[], qvel=[], act=[], targets=[], time=[], obs=[], dense=[], done=[], solved=[])
for i in range(N):
    o.reset()
    o.set(qpos=rng.uniform(m.jnt_range[:, 0], m.jnt_range[:, 1]) * (0.15 if i < 8 else 1.0), qvel=rng.normal(0, 0.5, m.nv), act=rng.uniform(0, 1, m.na)); o.forward()
    env = ReachEnvV0.__new__(ReachEnvV0)
    env.mj_model, env.mj_data, env.frame_skip, env.far_th = fake_model(m), fake_data(o, m.nbody), 10, reg["far_th"]       # dt = 0.02
    env.tip_sids = [m.name2id("site", t) for t in tips]; env.target_sids = [m.name2id("site", t + "_target") for t in tips]
    sx = env.mj_data.site_xpos
    if i < 4:            # targets on / next to the tips: the bonus and solved branches
        tg = np.array([sx[sid] for sid in env.tip_sids]) + rng.normal(0, 0.004 if i < 2 else 0.012, (len(tips), 3))
    else:
        tg = np.array([rng.uniform(reg["target_reach_range"][t][0], reg["target_reach_range"][t][1]) for t in tips])
    for k, sid in enumerate(env.target_sids):
        sx[sid] = tg[k]
    # mjData.time as MuJoCo accumulates it (one addition per substep): steps 1, 2, 3 sit around the `time > 2 dt` switch of far_th
    nstep = [1, 2, 3, 7][i % 4]; tm = 0.0
    for _ in range(10 * nstep):
        tm += m.opt_timestep
    env.mj_data.time = tm
    env.rwd_keys_wt = ReachEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS
    od = env.get_obs_dict(env.mj_model, env.mj_data)
    env.obs_dict = od
    t, vec = ObsVecDict().obsdict2obsvec(od, ReachEnvV0.DEFAULT_OBS_KEYS + ["act"])                      # base_v0.py:33-37 appends "act"
    rd = env.get_reward_dict(od)
    R["qpos"].append(o.f("qpos").copy()); R["qvel"].append(o.f("qvel").copy()); R["act"].append(o.f("act").copy()); R["targets"].append(tg); R["time"].append(tm); R["obs"].append(vec)
    for k in ("dense", "done", "solved"):
        R[k].append(float(np.asarray(rd[k]).ravel()[0]))
for k, v in R.items():
    out["reach_" + k] = np.array(v)
assert out["reach_obs"].shape == (N, 115) and out["reach_done"].sum() >= 2 and out["reach_solved"].sum() >= 1 and (out["reach_done"] == 0).sum() >= 4
np.savez_compressed(os.path.join(HERE, "tasks.npz"), **out)
print("wrote tasks.npz", {k: v.shape for k, v in out.items()})
