"""Gym-level drop-in surface (SURVEY.md section 8b).  CPU part: the host-side obs_dict / rwd_dict logic against the goldens produced by
the reference's own env classes (tests/golden/make_golden*.py).  GPU part: the contract of the reference's tests/test_envs.py:54-123
(seeded determinism, dict APIs, pickle round trip, spaces) on MyoEnv for the four BASELINE config ids."""
import copy
import os
import pickle

import numpy as np
import pytest

from myosuite_b200 import gym_api

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_spaces_match_reference_definition():
    a, o = gym_api.make_spaces(39, 108)                       # env_base.py:145-155, 210-218
    assert a.shape == (39,) and a.dtype == np.float32 and np.all(a.low == -1) and np.all(a.high == 1)
    assert o.shape == (108,) and np.all(o.low == -10) and np.all(o.high == 10)
    assert a == gym_api.make_spaces(39, 108)[0] and a.contains(a.sample())
    b = gym_api.Box(-np.ones(3), np.ones(3)); b.seed(1); x = b.sample(); b.seed(1)
    assert np.array_equal(x, b.sample())


@pytest.mark.parametrize("tag,nq,na,thd", [("elbow", 1, 6, 0.175), ("hand", 23, 39, 0.7)])
def test_pose_dicts_vs_reference_golden(tag, nq, na, thd):
    z = np.load(os.path.join(G, "pylogic.npz"))
    obs = z["pose_%s_obs" % tag]
    d = gym_api.obs_dict_from_vec("pose", obs, np.zeros(len(obs)), nq, nq, na)
    assert list(d.keys()) == ["time", "qpos", "qvel", "pose_err", "act"]
    np.testing.assert_array_equal(d["qpos"], z["pose_%s_qpos" % tag].astype(np.float32))
    r = gym_api.reward_dict("pose", d, gym_api.DEFAULT_WEIGHTS["pose"], {"pose_thd": thd})
    for k in ("pose", "bonus", "penalty", "act_reg", "sparse", "dense"):
        np.testing.assert_allclose(r[k], z["pose_%s_rwd_%s" % (tag, k)], rtol=2e-6, atol=2e-6)      # the host side sees the f32 observation
    for k in ("solved", "done"):
        assert np.array_equal(np.asarray(r[k], dtype=bool), z["pose_%s_rwd_%s" % (tag, k)].astype(bool))


def test_reach_hold_walk_dicts_vs_reference_golden(models):
    z = np.load(os.path.join(G, "tasks.npz"))
    # reach
    obs = z["reach_obs"]; d = gym_api.obs_dict_from_vec("reach", obs, z["reach_time"], 23, 23, 39, ntip=5)
    import json
    from myosuite_b200 import blob
    reg = json.load(open(os.path.join(os.path.dirname(blob.__file__), "assets", "registry.json")))["envs"]["myoHandReachRandom-v0"]["kwargs"]
    r = gym_api.reward_dict("reach", d, gym_api.DEFAULT_WEIGHTS["reach"], {"ntip": 5, "far_th": reg["far_th"], "dt": 0.02})
    np.testing.assert_allclose(r["dense"], z["reach_dense"], rtol=5e-6, atol=5e-6)
    assert np.array_equal(np.asarray(r["done"], bool), z["reach_done"].astype(bool)) and np.array_equal(np.asarray(r["solved"], bool), z["reach_solved"].astype(bool))
    # hold
    obs = z["hold_obs"]; d = gym_api.obs_dict_from_vec("hold", obs, np.zeros(len(obs)), 30, 29, 39)
    r = gym_api.reward_dict("hold", d, gym_api.DEFAULT_WEIGHTS["hold"], {})
    np.testing.assert_allclose(r["dense"], z["hold_dense"], rtol=2e-5, atol=2e-5)
    assert np.array_equal(np.asarray(r["done"], bool), z["hold_done"].astype(bool))
    # walk
    m = models["myolegs"]
    obs = z["walk_obs"]; d = gym_api.obs_dict_from_vec("walk", obs, np.zeros(len(obs)), 35, 34, 80)
    cfg = dict(target_x_vel=0.0, target_y_vel=1.2, min_height=0.8, max_rot=0.8, target_rot=m.key_qpos[0][3:7])
    for j in ("hip_flexion_l", "hip_flexion_r", "hip_adduction_l", "hip_adduction_r", "hip_rotation_l", "hip_rotation_r"):
        cfg["q_" + j] = int(m.jnt_qposadr[m.name2id("joint", j)])
    r = gym_api.reward_dict("walk", d, gym_api.DEFAULT_WEIGHTS["walk"], cfg)
    for k in ("vel_reward", "cyclic_hip", "ref_rot", "joint_angle_rew"):
        np.testing.assert_allclose(r[k], z["walk_" + k], rtol=2e-5, atol=2e-5)
    assert np.array_equal(np.asarray(r["done"], bool), z["walk_done"].astype(bool))
    np.testing.assert_allclose(r["dense"], z["walk_dense"], rtol=5e-5, atol=5e-4)


def _assert_close(a, b, atol=1e-5, rtol=1e-8):
    if a is None and b is None:
        return
    if isinstance(a, dict):
        for k in a:
            _assert_close(a[k], b[k], atol, rtol)
    else:
        np.testing.assert_allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), atol=atol, rtol=rtol)


@pytest.mark.gpu
@pytest.mark.parametrize("env_id", ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0", "myoFatiLegWalk-v0", "myoHandObjHoldRandom-v0"])
def test_env_contract_like_reference_test_envs(env_id):
    """Mirror of myosuite/tests/test_envs.py:54-123 (check_env)."""
    import myosuite_b200 as myo
    input_seed = 1234
    env1 = myo.make(env_id, seed=input_seed).unwrapped
    assert env1.get_input_seed() == input_seed
    env1.seed(input_seed)
    reset_obs1, *_ = env1.reset()
    assert isinstance(reset_obs1, np.ndarray) and reset_obs1.dtype == np.float32 and env1.observation_space.shape == reset_obs1.shape
    u = 0.01 * np.random.default_rng(0).uniform(0, 1, env1.mj_model.nu)
    assert env1.action_space.shape == u.shape
    obs1, rwd1, done1, *_, infos1 = env1.step(u.copy())
    infos1 = copy.deepcopy(infos1)
    assert len(obs1) > 0 and isinstance(rwd1, float) and isinstance(done1, bool)
    for k in ("time", "rwd_dense", "rwd_sparse", "solved", "done", "obs_dict", "rwd_dict", "state"):
        assert k in infos1
    od = env1.get_obs_dict(env1.mj_model, env1.mj_data); assert len(od) > 0 and "act" in od and "time" in od
    rd = env1.get_reward_dict(od); assert {"dense", "sparse", "solved", "done"} <= set(rd)
    np.testing.assert_allclose(np.concatenate([np.ravel(od[k]) for k in env1.obs_keys]), obs1)       # obs vector == concatenated obs_dict (obs_vec_dict.py:76-88)
    assert abs(float(np.squeeze(rd["dense"])) - rwd1) < 1e-9          # the device's own reward is reported for the current observation
    st = env1.get_env_state(); assert {"time", "qpos", "qvel", "act"} <= set(st) and len(st["qpos"]) == env1.mj_model.nq
    np.testing.assert_allclose(env1.mj_data.qpos, st["qpos"])
    env1.reset()
    # serialize / deserialize
    env2 = pickle.loads(pickle.dumps(env1)).unwrapped
    assert env2.get_input_seed() == input_seed
    assert env1.action_space == env2.action_space and env1.observation_space == env2.observation_space
    env2.seed(input_seed)
    reset_obs2, *_ = env2.reset()
    _assert_close(reset_obs1, reset_obs2)
    obs2, rwd2, done2, *_, infos2 = env2.step(u)
    _assert_close(obs1, obs2); _assert_close(rwd1, rwd2); assert done1 == done2 and len(infos1) == len(infos2)
    _assert_close({k: infos1[k] for k in ("time", "rwd_dense", "rwd_sparse", "obs_dict", "rwd_dict")}, infos2)
    _assert_close(infos1["state"]["qpos"], infos2["state"]["qpos"])
    # set_env_state restores a state exactly (env_base.py:720-759)
    env2.step(u); env2.set_env_state(infos1["state"])
    _assert_close(env2.get_env_state()["qpos"], infos1["state"]["qpos"], atol=0)
    obs3, *_ = env2.forward()
    # path-level helpers (env_base.py:434-459, 664-686, 763-826)
    assert env2.id == env_id and env2.time == pytest.approx(float(infos1["time"])) and np.array_equal(env2.get_obs(), obs3)
    od3 = env2.obsvec2obsdict(np.stack([obs3, obs3])[None]); assert list(od3) == list(env2.obs_keys) and od3["act"].shape == (1, 2, env2.mj_model.na)
    if "Reach" not in env_id:
        pr = env2.compute_path_rewards({"observations": np.stack([obs3, obs3, obs3])[None]})
        assert pr["rewards"].shape == (3,) and pr["done"].shape == (3,)
    assert env2.evaluate_success([{"env_infos": {"solved": np.ones(7, bool), "rwd_sparse": np.zeros(7), "rwd_dense": np.zeros(7)}}]) == 100.0
    if "Walk" in env_id:       # phase_var = steps / hip_period: the reference builds a step's observation BEFORE it increments `steps` (walk_v0.py:339-342), forward() sees the count after
        k = list(env1.obs_keys).index("phase_var"); off = sum(np.size(env1.obs_dict[q]) for q in env1.obs_keys[:k])
        obs3 = obs3.copy(); obs3[off] = obs1[off]
    _assert_close(obs3, obs1, atol=1e-6)


def test_torso_dicts_vs_reference_golden():
    """TorsoEnvV0 (torso_v0.py:84-125): the pose rule with far_th = pi, pose_thd 0.25, target = mean of the registered ranges."""
    z = np.load(os.path.join(G, "torso.npz"))
    d = gym_api.obs_dict_from_vec("pose", z["obs"], np.zeros(len(z["obs"])), 18, 18, 210)
    np.testing.assert_array_equal(d["pose_err"], (z["target"] - z["qpos"]).astype(np.float32))
    r = gym_api.reward_dict("pose", d, {"pose": 1.0, "bonus": 4.0, "act_reg": 1.0, "penalty": 50, "done": 0}, {"pose_thd": 0.25, "pose_far_th": np.pi})
    np.testing.assert_allclose(r["dense"], z["dense"], rtol=3e-6, atol=3e-6)
    assert np.array_equal(np.asarray(r["done"], bool), z["done"].astype(bool)) and np.array_equal(np.asarray(r["solved"], bool), z["solved"].astype(bool))


def test_path_methods_like_env_base():
    """compute_path_rewards / truncate_paths / evaluate_success / obsvec2obsdict (env_base.py:763-826, obs_vec_dict.py:90-97) on the elbow pose layout."""
    z = np.load(os.path.join(G, "pylogic.npz"))
    obs = z["pose_elbow_obs"]; N = (len(obs) // 4) * 4
    lay = gym_api.obs_layout("pose", 1, 1, 6)
    vec = obs[:N].reshape(4, N // 4, -1)
    od = gym_api.obsvec2obsdict(vec, lay)
    assert list(od) == ["qpos", "qvel", "pose_err", "act"] and od["act"].shape == (4, N // 4, 6)
    with pytest.raises(AssertionError):
        gym_api.obsvec2obsdict(vec[0], lay)
    paths = gym_api.compute_path_rewards("pose", {"observations": vec.copy()}, lay, gym_api.DEFAULT_WEIGHTS["pose"], {"pose_thd": 0.175})
    dense = z["pose_elbow_rwd_dense"][:N].reshape(4, N // 4); done = z["pose_elbow_rwd_done"][:N].reshape(4, N // 4).astype(bool)
    np.testing.assert_allclose(paths["rewards"][:, :-1], dense[:, 1:], rtol=2e-6, atol=2e-6)          # time-aligned: entry t is the reward of observation t+1
    np.testing.assert_allclose(paths["rewards"][:, -1], dense[:, -1], rtol=2e-6, atol=2e-6)           # (last entry redundant, as in the reference)
    assert np.array_equal(paths["done"][:, :-1], done[:, 1:])
    # truncate_paths: first done at step 3 -> entries 0..4 kept (the reference's sum(~done) + 1 rule) and terminated = True
    p1 = {"rewards": np.arange(8.0), "done": np.array([0, 0, 0, 1, 1, 1, 1, 1], bool), "observations": np.zeros((8, 2))}
    p2 = {"rewards": np.arange(8.0), "done": np.zeros(8, bool), "observations": np.zeros((8, 2))}
    out = gym_api.truncate_paths([p1, p2])
    assert out[0]["terminated"] is True and len(out[0]["rewards"]) == 5 and out[0]["observations"].shape == (5, 2) and out[1]["terminated"] is False and len(out[1]["rewards"]) == 8
    logged = {}
    lg = type("L", (), {"log_kv": lambda self, k, v: logged.__setitem__(k, v)})()
    mk = lambda n_solved: {"env_infos": {"solved": np.array([True] * n_solved + [False] * (10 - n_solved)), "rwd_sparse": np.ones(10), "rwd_dense": np.full(10, 2.0)}}
    assert gym_api.evaluate_success([mk(6), mk(5), mk(0), mk(10)], horizon=10, logger=lg) == 50.0          # "solved for MORE than 5 steps"
    assert logged == {"rwd_sparse": 1.0, "rwd_dense": 2.0, "success_percentage": 50.0}
