"""Golden vectors for the muscle-condition variants (myoSarc* / myoFati* / myoReaf*), produced by RUNNING THE REFERENCE'S OWN
BaseV0.initializeConditions and BaseV0.step (base_v0.py:60-118, unmodified) with robot.step stubbed to record ctrl_desired.  The model
is a stub that carries the shipped model's actuator_dyntype, gainprm, biasprm, dynprm, timestep and actuator names.
Output: tests/golden/variants.npz.   Run with MYOSUITE_CHECKOUT set:  python tests/golden/make_golden_variants.py

  reaf_<norm>_<dtype>_action / _ctrl   reafferentation on the hand pose model, normalize_act True / False, float64 and float32 actions
                                        (rows 0..8: EIP and EPL at every pair of -1, 0.5, 1; then uniform random actions)
  reaf_ids                              (EPL, EIP) actuator ids the reference looks up
  sarc_<model>_gainprm / _biasprm       actuator_gainprm / biasprm after initializeConditions of the sarcopenia condition
  fati_torso_action / _ctrl             a 60-step fatigue chain on the torso's 210 muscles (normalize_act True, float64 actions)
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
from myosuite.envs.myo.base_v0 import BaseV0  # noqa: E402

from myosuite_b200 import assets  # noqa: E402

MODELS = ("myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso")
out = {}
rng = np.random.default_rng(20261017)


def stub_model(m):
    """The fields of mjModel that initializeConditions, BaseV0.step and CumulativeFatigue read, copied from the shipped model."""
    fm = types.SimpleNamespace(na=m.na, nu=m.nu, opt=types.SimpleNamespace(timestep=m.opt_timestep),
                               actuator_dyntype=np.array(m.actuator_dyntype).copy(), actuator_dynprm=np.array(m.actuator_dynprm, dtype=np.float64).copy(),
                               actuator_gainprm=np.array(m.actuator_gainprm, dtype=np.float64).copy(),
                               actuator_biasprm=np.array(m.actuator_biasprm, dtype=np.float64).copy())
    fm.actuator = lambda name: types.SimpleNamespace(id=m.name2id("actuator", name))
    return fm


def stub_env(m, cond, normalize_act, frame_skip=10):
    rec = []
    env = types.SimpleNamespace(mj_model=stub_model(m), normalize_act=normalize_act, muscle_condition=cond, frame_skip=frame_skip,
                                dt=m.opt_timestep * frame_skip, mujoco_render_frames=False, mj_render=None, forward=lambda **kw: None,
                                get_input_seed=lambda: 0)
    env.robot = types.SimpleNamespace(step=lambda ctrl_desired, **kw: rec.append(np.array(ctrl_desired, dtype=np.float64)) or ctrl_desired)
    BaseV0.initializeConditions(env)
    return env, rec


def run(env, rec, A):
    rec.clear()
    for a in A:
        BaseV0.step(env, a.copy())
    return np.stack(rec)


# ---- 1. reafferentation on the hand (EIP -> EPL, EIP = 0), with and without the sigmoid, float64 and float32 actions
hand = assets.load("myohand_pose")
epl, eip = hand.name2id("actuator", "EPL"), hand.name2id("actuator", "EIP")
out["reaf_ids"] = np.array([epl, eip])
A = rng.uniform(-1, 1, (40, hand.nu))
k = 0
for x in (-1.0, 0.5, 1.0):
    for y in (-1.0, 0.5, 1.0):
        A[k, eip], A[k, epl] = x, y; k += 1
for norm in (True, False):
    env, rec = stub_env(hand, "reafferentation", norm)
    assert (env.EPLpos, env.EIPpos) == (epl, eip)
    for dt in (np.float64, np.float32):
        tag = "reaf_%s_%s" % ("norm" if norm else "raw", np.dtype(dt).name)
        out[tag + "_action"] = A.astype(dt)
        out[tag + "_ctrl"] = run(env, rec, A.astype(dt))

# ---- 2. sarcopenia: gainprm[:, 2] halved, biasprm untouched, on every shipped model
for name in MODELS:
    env, _ = stub_env(assets.load(name), "sarcopenia", True)
    out["sarc_%s_gainprm" % name] = env.mj_model.actuator_gainprm
    out["sarc_%s_biasprm" % name] = env.mj_model.actuator_biasprm

# ---- 3. fatigue chain on the torso's 210 muscles (CumulativeFatigue with the model's own tauact / taudeact, frame_skip 10)
torso = assets.load("myotorso")
env, rec = stub_env(torso, "fatigue", True)
A = rng.uniform(-1, 1, (60, torso.nu))
A[20:30] = 1.0
A[40:45] = -1.0
out["fati_torso_action"] = A
out["fati_torso_ctrl"] = run(env, rec, A)

np.savez_compressed(os.path.join(HERE, "variants.npz"), **out)
print("wrote variants.npz:", {k: v.shape for k, v in out.items()})
