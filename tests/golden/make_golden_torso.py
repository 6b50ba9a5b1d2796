"""Golden vectors for the Torso task, produced by RUNNING THE REFERENCE'S OWN TorsoEnvV0 (get_obs_dict / get_reward_dict and the target
rule of _setup, unmodified, instance created with __new__ so that no simulator is constructed) on random states of the torso model.
Output: tests/golden/torso.npz.   Run with MYOSUITE_CHECKOUT set:  python tests/golden/make_golden_torso.py"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE); sys.path.insert(0, ROOT)
import _ref_stubs  # noqa: E402

_ref_stubs.install()
from myosuite.envs.myo.myobase.torso_v0 import TorsoEnvV0  # noqa: E402
from myosuite.envs.obs_vec_dict import ObsVecDict  # noqa: E402

from myosuite_b200 import assets  # noqa: E402

reg = json.load(open(os.path.join(ROOT, "myosuite_b200", "assets", "registry.json")))["envs"]["myoTorsoPoseFixed-v0"]
kw = reg["kwargs"]
m = assets.load("myotorso")
rng = np.random.default_rng(5)
N = 48
env = TorsoEnvV0.__new__(TorsoEnvV0)
fm = types.SimpleNamespace(na=m.na, nu=m.nu, opt=types.SimpleNamespace(timestep=m.opt_timestep))
fm.joint = lambda name: types.SimpleNamespace(id=m.name2id("joint", name))
env.mj_model = fm
env.frame_skip = kw["frame_skip"]
# the target rule of TorsoEnvV0._setup (torso_v0.py:58-68), executed verbatim on the registry kwargs
env.target_jnt_ids, env.target_jnt_range = [], []
for jnt_name, jnt_range in kw["target_jnt_range"].items():
    env.target_jnt_ids.append(env.mj_model.joint(jnt_name).id); env.target_jnt_range.append(jnt_range)
env.target_jnt_range = np.array(env.target_jnt_range)
env.target_jnt_value = np.mean(env.target_jnt_range, axis=1)
env.pose_thd = 0.25                                  # _setup default (torso_v0.py:52)
env.rwd_keys_wt = TorsoEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS
out = dict(qpos=[], qvel=[], act=[], obs=[], dense=[], done=[], solved=[], sparse=[])
for i in range(N):
    scale = [0.05, 0.3, 1.0, 3.0][i % 4]             # near the target ... far beyond the joint ranges (the done / penalty branch at pi)
    q = rng.uniform(m.jnt_range[:, 0], m.jnt_range[:, 1]) * scale
    data = types.SimpleNamespace(time=0.0, qpos=q, qvel=rng.normal(0, 0.5, m.nv), act=rng.uniform(0, 1, m.na))
    od = env.get_obs_dict(env.mj_model, data)
    env.obs_dict = od
    _, vec = ObsVecDict().obsdict2obsvec(od, TorsoEnvV0.DEFAULT_OBS_KEYS + ["act"])
    rd = env.get_reward_dict(od)
    out["qpos"].append(q); out["qvel"].append(data.qvel); out["act"].append(data.act); out["obs"].append(vec)
    for k in ("dense", "done", "solved", "sparse"):
        out[k].append(float(np.asarray(rd[k]).ravel()[0]))
out = {k: np.array(v) for k, v in out.items()}
out["target"] = env.target_jnt_value
out["dt"] = np.array(m.opt_timestep * kw["frame_skip"])
assert out["obs"].shape == (N, 18 + 18 + 18 + 210) and out["done"].sum() >= 1 and out["solved"].sum() >= 1
np.savez_compressed(os.path.join(HERE, "torso.npz"), **out)
print("wrote torso.npz", {k: v.shape for k, v in out.items()}, "target", out["target"])
