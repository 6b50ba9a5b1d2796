"""myosuite_b200/tasks.py: the kernel configuration of every registered id, built on the host alone (no torch, no device, no library),
and the info quantities derived from the observation against the reference's own reward dicts."""
import os

import numpy as np
import pytest

from myosuite_b200 import abi, assets, program, tasks, vec_env

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _configure(env_id, **overrides):
    steps, kw, entry = vec_env.env_spec(env_id)
    kw.update(overrides)
    m = assets.load(vec_env._MODEL_OF_XML[kw["model_path"]])
    return m, kw, tasks.configure(entry, m, program.build_program(m)[1], kw, steps)


@pytest.mark.parametrize("env_id", vec_env.registered_ids())
def test_configure_every_registered_id_without_a_device(env_id):
    steps, kw, entry = vec_env.env_spec(env_id)
    m, kw, c = _configure(env_id)
    cfg, task = c.cfg, c.task
    assert tasks.task_of(entry) == (task, c.torso, c.hold_random)
    assert cfg.task == tasks.TASK_CODE[task] and cfg.max_episode_steps == steps and cfg.auto_reset == 1 and cfg.frame_skip == c.n_frames == kw.get("frame_skip", 10)
    assert cfg.muscle_condition == (abi.COND_FATIGUE if kw.get("muscle_condition") == "fatigue" else abi.COND_NONE)
    assert (cfg.reaf_dst >= 0) == (kw.get("muscle_condition") == "reafferentation")
    # the weights the kernel reads, in its order
    w = tasks.DEFAULT_WEIGHTS[task]
    assert [cfg.weights[i] for i in range(len(tasks.WEIGHT_ORDER[task]))] == [w.get(k, 0.0) for k in tasks.WEIGHT_ORDER[task]]
    # reset rows, target ranges and the obs layout the host slices
    assert np.shape(c.init_qpos)[-1] == m.nq and np.shape(c.init_qvel)[-1] == m.nv and np.shape(c.init_qpos)[:-1] == np.shape(c.init_qvel)[:-1]
    assert c.target_range.shape == (m.nq, 2) and np.all(c.target_range[:, 0] <= c.target_range[:, 1])
    assert [k for k, _ in c.layout] == [k for k, _ in tasks.obs_layout(task, m.nq, m.nv, m.na, len(c.tip_names))] and c.layout[-1] == ("act", m.na)
    assert c.reward_cfg["ntip"] == len(c.tip_names) and c.reward_cfg["pose_thd"] == cfg.pose_thd and c.reward_cfg["dt"] == c.dt
    if c.torso:
        assert cfg.task_d[0] == np.pi and cfg.pose_thd == tasks.TORSO_POSE_THD and c.reward_cfg["pose_far_th"] == np.pi
        assert np.all(c.target_range[:, 0] == c.target_range[:, 1])
    if task in ("reach", "stand"):
        assert c.tip_names == list(kw["target_reach_range"]) and cfg.task_i[0] == len(c.tip_names)
        assert cfg.task_d[3 * len(c.tip_names)] == kw.get("far_th", tasks.REACH_FAR_TH)
    else:
        assert c.tip_names == [] and c.target_center is None
    if task == "stand":
        assert tuple(cfg.reach_shape) == tasks.STAND_SHAPE and tuple(cfg.joint_random) == (-0.2, 0.2)
        np.testing.assert_array_equal(c.init_qpos, m.key_qpos[0])
        np.testing.assert_allclose(c.target_center, [[0.0, 0.0, 0.92]], atol=1e-12)
        np.testing.assert_allclose(c.target_range[:3], c.target_center[0][:, None] + np.array([[-0.05, 0.05], [-0.05, 0.05], [0.0, 0.0]]), atol=1e-15)
    else:
        assert tuple(cfg.reach_shape) == (0.0,) * 4 and tuple(cfg.joint_random) == (0.0, 0.0)
    if task == "hold":
        assert cfg.reset_random == int(c.hold_random) and np.array_equal(c.env_prm, [cfg.task_d[6 + i] for i in range(6)])
    else:
        assert c.env_prm is None
    if task == "walk":
        assert [c.reward_cfg["q_" + j] for j in tasks.HIP_JOINTS] == [cfg.task_i[4 + i] for i in range(6)]
        assert cfg.task_d[4:9] == [0.8, 0.8, 100, 0.0, 1.2] and np.array_equal(c.reward_cfg["target_rot"], m.key_qpos[0][3:7])


def test_configure_rejects_and_defaults():
    with pytest.raises(NotImplementedError):
        tasks.configure("myosuite.envs.myo.myobase.walk_v0:TerrainEnvV0", None, None, {})
    with pytest.raises(NotImplementedError):
        _configure("myoHandPoseRandom-v0", joint_random_range=(-0.1, 0.1))
    with pytest.raises(NotImplementedError):
        _configure("myoLegStandRandom-v0", joint_random_range=(0.0, 0.0))
    with pytest.raises(KeyError):                              # pose, walk and hold need every weight the kernel reads
        _configure("myoHandPoseRandom-v0", weighted_reward_keys={"pose": 1.0})
    _, _, c = _configure("myoHandReachRandom-v0", weighted_reward_keys={"reach": 2.0})          # reach counts a missing weight as 0
    assert list(c.cfg.weights)[:4] == [2.0, 0.0, 0.0, 0.0]
    _, _, c = _configure("myoLegWalk-v0", reset_type="random")
    assert c.init_qpos.shape[0] == c.init_qvel.shape[0] == 2 and c.cfg.reset_random == 1
    m = assets.load("myoelbow_1dof6muscles")
    c = tasks.configure(None, m, program.build_program(m)[1], {"normalize_act": True}, auto_reset=False)
    assert c.task == "none" and c.cfg.task == abi.TASK_NONE and c.layout == [] and c.cfg.auto_reset == 0


def test_info_from_obs_matches_reference_goldens():
    """rwd_sparse / solved derived from the observation vector (tasks.info_from_obs) vs the reference's own reward dicts."""
    G = np.load(os.path.join(GOLDEN, "pylogic.npz")); T = np.load(os.path.join(GOLDEN, "tasks.npz"))
    for tag, thd, nq, na in (("elbow", 0.175, 1, 6), ("hand", 0.7, 23, 39)):
        obs = G["pose_%s_obs" % tag]
        inf = tasks.info_from_obs("pose", obs, nq, nq, na, pose_thd=thd)
        np.testing.assert_allclose(inf["rwd_sparse"], G["pose_%s_rwd_sparse" % tag], rtol=2e-6, atol=2e-6)
        ok = np.abs(-inf["rwd_sparse"] - thd) > 1e-5                                     # (f32 obs: skip cases on the threshold)
        np.testing.assert_array_equal(inf["solved"][ok], G["pose_%s_rwd_solved" % tag].astype(bool)[ok])
    inf = tasks.info_from_obs("reach", T["reach_obs"], 23, 23, 39, ntip=5)
    np.testing.assert_array_equal(inf["solved"], T["reach_solved"].astype(bool))
    import torch
    inf_t = tasks.info_from_obs("reach", torch.as_tensor(T["reach_obs"]), 23, 23, 39, ntip=5)
    np.testing.assert_allclose(inf_t["rwd_sparse"].numpy(), inf["rwd_sparse"], rtol=1e-12)
    d = np.linalg.norm(T["hold_obs"][:, 49:52].astype(np.float64), axis=1)
    inf = tasks.info_from_obs("hold", T["hold_obs"], 30, 29, 39)
    np.testing.assert_allclose(inf["rwd_sparse"], -d) and np.array_equal(inf["solved"], d < 0.010)
    assert tasks.info_from_obs("walk", T["walk_obs"], 35, 34, 80) is None
