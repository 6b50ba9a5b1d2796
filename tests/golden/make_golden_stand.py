"""Golden vectors for the leg stand task (myoLegStandRandom-v0), produced by RUNNING THE REFERENCE'S OWN ReachEnvV0 of
myosuite/envs/myo/myobase/walk_v0.py (get_obs_dict, get_reward_dict, generate_qpos, generate_targets, unmodified, created with __new__ so
that no simulator is constructed) on mj_data-like records filled from this repo's CPU oracle, and on a fake np_random that returns
recorded uniforms.  Output: tests/golden/stand.npz
Run with a MyoSuite checkout (MYOSUITE_CHECKOUT=<its root>) and oracle/libmyo_oracle.so built:  python tests/golden/make_golden_stand.py
"""
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
from myosuite.envs.myo.myobase.walk_v0 import ReachEnvV0  # noqa: E402
from myosuite.envs.obs_vec_dict import ObsVecDict  # noqa: E402

from myosuite_b200 import assets, blob  # noqa: E402
from oracle.oracle_py import Oracle  # noqa: E402

reg = json.load(open(os.path.join(ROOT, "myosuite_b200", "assets", "registry.json")))["envs"]["myoLegStandRandom-v0"]["kwargs"]
m = assets.load("myolegs")
o = Oracle(*blob.pack(m))
rng = np.random.default_rng(2024)
tips = list(reg["target_reach_range"].keys())


class RecordedUniform:
    """np_random stand-in: uniform(low, high, size) = low + (high - low) u (numpy's own formula) with u taken from `us` in order."""

    def __init__(self, us):
        self.us = list(us)

    def uniform(self, low=0.0, high=1.0, size=None):
        u = self.us.pop(0)
        low, high = np.asarray(low, dtype=np.float64), np.asarray(high, dtype=np.float64)
        return low + (high - low) * u


def fake_model():
    fm = types.SimpleNamespace(na=m.na, nu=m.nu, jnt_qposadr=m.jnt_qposadr, jnt_range=m.jnt_range, key_qpos=m.key_qpos, site_pos=m.site_pos.copy(),
                               opt=types.SimpleNamespace(timestep=m.opt_timestep))
    fm.site = lambda name: types.SimpleNamespace(id=m.name2id("site", name))
    return fm


def fake_data():
    return types.SimpleNamespace(time=0.0, qpos=o.f("qpos").copy(), qvel=o.f("qvel").copy(), act=o.f("act").copy(), site_xpos=o.f("site_xpos").reshape(-1, 3).copy())


def make_env(us=()):
    env = ReachEnvV0.__new__(ReachEnvV0)
    env.mj_model, env.frame_skip, env.far_th = fake_model(), 10, reg["far_th"]            # dt = 0.01
    env.joint_random_range, env.target_reach_range = tuple(reg["joint_random_range"]), reg["target_reach_range"]
    env.init_qpos, env.init_qvel = m.key_qpos[0].copy(), m.key_qvel[0].copy()            # walk_v0.py:65-66
    env.tip_sids = [m.name2id("site", t) for t in tips]; env.target_sids = [m.name2id("site", t + "_target") for t in tips]
    env.rwd_keys_wt = ReachEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS
    env.np_random = RecordedUniform(us)
    return env


def forward(q, v=None, a=None):
    o.reset()
    o.set(qpos=q, qvel=np.zeros(m.nv) if v is None else v, act=np.zeros(m.na) if a is None else a, ctrl=np.zeros(m.nu))
    o.forward()


out = {}
# ---- the reset rule: generate_qpos on recorded uniforms (one nq-vector per draw, as the reference draws them)
ND = 64
U = rng.random((ND, m.nq))
env = make_env(list(U))
out["reset_u"], out["reset_qpos"] = U, np.array([env.generate_qpos() for _ in range(ND)])

# ---- the target: generate_targets after a first draw, on mj_data filled from the oracle at that draw
NT = 8
TU, TQ, TC, TT = rng.random((NT, 3)), [], [], []
for i in range(NT):
    u1 = rng.random(m.nq)
    env = make_env([u1, TU[i]])
    q1 = env.generate_qpos(); forward(q1)
    env.mj_data = fake_data()
    centre = env.mj_data.site_xpos[env.tip_sids[0]].copy()
    env.generate_targets()
    TQ.append(q1); TC.append(centre); TT.append(env.mj_model.site_pos[env.target_sids[0]].copy())
out["target_u"], out["target_draw_qpos"], out["target_centre"], out["target"] = TU, np.array(TQ), np.array(TC), np.array(TT)

# ---- obs / reward: distances on both sides of 0.05, 0.1 and 0.44, times on both sides of 2 dt
DIST = [0.02, 0.045, 0.055, 0.08, 0.095, 0.105, 0.2, 0.43, 0.45, 0.7]
NSTEP = [1, 2, 3, 7]
S = {k: [] for k in ("qpos", "qvel", "act", "targets", "time", "obs", "dense", "reach", "bonus", "act_reg", "penalty", "sparse", "solved", "done")}
for i in range(len(DIST) * len(NSTEP)):
    dist, nstep = DIST[i % len(DIST)], NSTEP[i // len(DIST)]
    if i % 2:        # a state the randomised reset starts from (couplings of the slide / coupled joints broken)
        q = out["reset_qpos"][i % ND].copy()
    else:            # keyframe 0 with small joint noise
        q = m.key_qpos[0].copy(); q[7:] += rng.normal(0, 0.05, m.nq - 7)
    forward(q, rng.normal(0, 0.5 if i % 3 else 3.0, m.nv), rng.uniform(0, 1, m.na))
    env = make_env()
    env.mj_data = fake_data()
    tip = env.mj_data.site_xpos[env.tip_sids[0]]
    dvec = rng.normal(0, 1, 3); tg = tip + dist * dvec / np.linalg.norm(dvec)
    env.mj_data.site_xpos[env.target_sids[0]] = tg
    tm = 0.0
    for _ in range(10 * nstep):       # mjData.time as MuJoCo accumulates it, one addition per substep
        tm += m.opt_timestep
    env.mj_data.time = tm
    od = env.get_obs_dict(env.mj_model, env.mj_data)
    env.obs_dict = od
    t, vec = ObsVecDict().obsdict2obsvec(od, ReachEnvV0.DEFAULT_OBS_KEYS + ["act"])                      # base_v0.py:33-37 appends "act"
    rd = env.get_reward_dict(od)
    S["qpos"].append(o.f("qpos").copy()); S["qvel"].append(o.f("qvel").copy()); S["act"].append(o.f("act").copy())
    S["targets"].append(tg); S["time"].append(tm); S["obs"].append(vec)
    for k in ("dense", "reach", "bonus", "act_reg", "penalty", "sparse", "solved", "done"):
        S[k].append(float(np.asarray(rd[k]).ravel()[0]))
for k, v in S.items():
    out["obs_" + k if k != "obs" else "obs"] = np.array(v)
n = len(S["obs"])
assert out["obs"].shape == (n, 155) and out["obs"].dtype == np.float32
assert out["obs_done"].sum() >= 4 and (out["obs_done"] == 0).sum() >= 4 and out["obs_solved"].sum() >= 4
np.savez_compressed(os.path.join(HERE, "stand.npz"), **out)
print("wrote stand.npz", {k: v.shape for k, v in out.items()})
