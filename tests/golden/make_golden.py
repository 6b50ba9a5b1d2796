"""Generate golden vectors by RUNNING THE REFERENCE'S OWN PYTHON CODE (unmodified, imported from
a MyoSuite checkout, MYOSUITE_CHECKOUT=<its root>, with third-party imports stubbed, see _ref_stubs.py).  Output: tests/golden/pylogic.npz

Covers the Python-side part of the hot path that is independent of MuJoCo:
  * CumulativeFatigue.compute_act / reset      (envs/myo/fatigue.py:38-99)
  * BaseV0.step action->ctrl remap (+fatigue)   (envs/myo/base_v0.py:82-118)  -- robot.step stubbed to record ctrl
  * PoseEnvV0.get_obs_dict / get_reward_dict     (envs/myo/myobase/pose_v0.py:100-140)
  * ObsVecDict.obsdict2obsvec                    (envs/obs_vec_dict.py:76-88)
Run with MYOSUITE_CHECKOUT set:  python tests/golden/make_golden.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_stubs  # noqa: E402

_ref_stubs.install()
from myosuite.envs.myo.base_v0 import BaseV0  # noqa: E402
from myosuite.envs.myo.fatigue import CumulativeFatigue  # noqa: E402
from myosuite.envs.myo.myobase.pose_v0 import PoseEnvV0  # noqa: E402
from myosuite.envs.obs_vec_dict import ObsVecDict  # noqa: E402

out = {}
rng = np.random.default_rng(20260922)


def fake_model(nmus, timestep, tauact=0.01, taudeact=0.04):
    return types.SimpleNamespace(opt=types.SimpleNamespace(timestep=timestep), actuator_dyntype=np.full(nmus, 4), na=nmus, nu=nmus,
                                 actuator_dynprm=np.tile([tauact, taudeact, 0, 0, 0, 0, 0, 0, 0, 0], (nmus, 1)))


# ---- 1. fatigue: the reference's own 4-step known-answer sequence (tests/mjx/test_fatigue.py:179-184) + a long random run
f = CumulativeFatigue(fake_model(5, 0.002), frame_skip=5, seed=0)
seq = [np.zeros(5), np.ones(5), np.array([.3, .5, .7, .2, .8]), np.full(5, 0.5)]
kat = []
for a in seq:
    MA, MR, MF = f.compute_act(a.copy())
    kat.append(np.stack([MA.copy(), MR.copy(), MF.copy()]))
out["fatigue_kat_in"] = np.stack(seq)
out["fatigue_kat_out"] = np.stack(kat)            # [4, 3, 5]
f = CumulativeFatigue(fake_model(80, 0.001), frame_skip=10, seed=0)
acts = np.random.default_rng(7).uniform(0, 1, (2000, 80))    # tests regenerate this input from the same seed
acts[500:700] = 1.0
acts[1200:1300] = 0.0
traj = []
for a in acts:
    MA, MR, MF = f.compute_act(a.copy())
    traj.append(np.stack([MA.copy(), MR.copy(), MF.copy()]))
out["fatigue_long_out"] = np.stack(traj)[::50]    # every 50th step, [40, 3, 80]
out["fatigue_long_final"] = np.stack(traj)[-1]

# ---- 2. BaseV0.step: action -> ctrl (sigmoid remap, optional fatigue), robot.step stubbed to record what reaches the simulator
for cond in ("", "fatigue"):
    rec = []
    fake = types.SimpleNamespace()
    fake.mj_model = fake_model(39, 0.002)
    fake.normalize_act = True
    fake.muscle_condition = cond
    fake.dt = 0.02
    fake.mujoco_render_frames = False
    fake.mj_render = None
    fake.robot = types.SimpleNamespace(step=lambda ctrl_desired, **kw: rec.append((np.array(ctrl_desired, dtype=np.float64), kw["ctrl_normalized"], kw["step_duration"])) or ctrl_desired)
    fake.forward = lambda **kw: None
    if cond == "fatigue":
        fake.muscle_fatigue = CumulativeFatigue(fake.mj_model, 10, seed=0)
    A = rng.uniform(-1, 1, (50, 39))
    for a in A:
        BaseV0.step(fake, a.copy())
    out["step_action_%s" % (cond or "none")] = A
    out["step_ctrl_%s" % (cond or "none")] = np.stack([r[0] for r in rec])
    assert all(r[1] is False for r in rec)
    # float32 actions (what action_space.sample() produces): the reference then computes the sigmoid in float32
    rec.clear()
    if cond == "":
        A32 = A.astype(np.float32)
        for a in A32:
            BaseV0.step(fake, a.copy())
        out["step_ctrl_f32in"] = np.stack([r[0] for r in rec])

# ---- 3. pose obs / reward
for tag, nq, na, thd in (("elbow", 1, 6, 0.175), ("hand", 23, 39, 0.7)):
    N = 64
    qpos = rng.uniform(-1, 2, (N, nq)); qvel = rng.normal(0, 3, (N, nq)); act = rng.uniform(0, 1, (N, na)); target = rng.uniform(-1, 2, (N, nq))
    qpos[:4] = target[:4] + rng.normal(0, 0.02, (4, nq))      # near-target cases (bonus branches)
    qpos[4:6] = target[4:6] + 7.0                              # beyond far_th (penalty/done)
    obs, rwd = [], {k: [] for k in ("pose", "bonus", "penalty", "act_reg", "sparse", "solved", "done", "dense")}
    for i in range(N):
        fake = types.SimpleNamespace(dt=0.02, target_jnt_value=target[i], pose_thd=thd, mj_model=types.SimpleNamespace(na=na),
                                     rwd_keys_wt=PoseEnvV0.DEFAULT_RWD_KEYS_AND_WEIGHTS, obs_keys=["qpos", "qvel", "pose_err", "act"])
        data = types.SimpleNamespace(time=0.0, qpos=qpos[i], qvel=qvel[i], act=act[i])
        od = PoseEnvV0.get_obs_dict(fake, fake.mj_model, data)
        fake.obs_dict = od
        ovd = ObsVecDict()
        t, vec = ovd.obsdict2obsvec(od, fake.obs_keys)
        obs.append(vec)
        ovd.expand_dims(od)                       # env_base.py:423 mutates self.obs_dict in place
        rd = PoseEnvV0.get_reward_dict(fake, fake.obs_dict)
        for k in rwd:
            rwd[k].append(np.asarray(rd[k], dtype=np.float64).ravel()[0])
    out["pose_%s_qpos" % tag], out["pose_%s_qvel" % tag], out["pose_%s_act" % tag], out["pose_%s_target" % tag] = qpos, qvel, act, target
    out["pose_%s_obs" % tag] = np.stack(obs)
    assert out["pose_%s_obs" % tag].dtype == np.float32
    for k, v in rwd.items():
        out["pose_%s_rwd_%s" % (tag, k)] = np.array(v)

np.savez_compressed(os.path.join(HERE, "pylogic.npz"), **out)
print("wrote pylogic.npz:", {k: v.shape for k, v in out.items()})
print("fatigue KAT MA:", out["fatigue_kat_out"][:, 0])
