"""Gym-level drop-in surface of the reference's env classes (SURVEY.md section 8b "must be preserved"), host side only.

What the reference exposes on `env.unwrapped` and its tests exercise (myosuite/tests/test_envs.py:54-123):
  action_space / observation_space      envs/env_base.py:145-155, 210-218      (Box(-1, 1, nu) f32 ; Box(-10, 10, obs_dim) f32)
  obs_dict / rwd_dict                   envs/env_base.py:409-432               (per-key views of the observation; reward terms)
  get_obs_dict / get_reward_dict        myobase/pose_v0.py:100-140, reach_v0.py:98-160, obj_hold_v0.py:79-121, walk_v0.py:80-140,268-319
  get_env_infos                         envs/env_base.py:585-616
  get_env_state / set_env_state         envs/env_base.py:688-759
  seed / get_input_seed / pickling      envs/env_base.py:119-123, gym.utils.EzPickle (pose_v0.py:32)
The per-key quantities are all contained in the observation vector the kernel writes (obs_vec_dict.py:76-88 concatenates
them in `obs_keys` order + "act"), so the dicts are sliced / recomputed from that vector and a few state scalars on the host;
nothing here touches the device.  Values therefore carry float32 precision where the reference's dicts hold float64.
"""
import collections

import numpy as np


# --------------------------------------------------------------------------------------------- spaces
class Box:
    """Minimal stand-in for gym.spaces.Box, used only when neither gymnasium nor gym is importable."""

    def __init__(self, low, high, shape=None, dtype=np.float32, seed=None):
        self.dtype = np.dtype(dtype)
        self.low = np.broadcast_to(np.asarray(low, dtype=self.dtype), shape if shape is not None else np.shape(low)).copy()
        self.high = np.broadcast_to(np.asarray(high, dtype=self.dtype), self.low.shape).copy()
        self.shape = self.low.shape
        self._rng = np.random.default_rng(seed)

    def seed(self, seed=None):
        self._rng = np.random.default_rng(seed)
        return [seed]

    def sample(self):
        return self._rng.uniform(self.low, self.high).astype(self.dtype)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

    __contains__ = contains

    def __eq__(self, other):
        return isinstance(other, Box) and self.shape == other.shape and self.dtype == other.dtype and np.array_equal(self.low, other.low) and np.array_equal(self.high, other.high)

    def __repr__(self):
        return "Box(%s, %s, %s, %s)" % (self.low.min(), self.high.max(), self.shape, self.dtype)


def box_class():
    """gymnasium.spaces.Box, else gym.spaces.Box, else the shim above."""
    for mod in ("gymnasium", "gym"):
        try:
            return __import__(mod + ".spaces", fromlist=["Box"]).Box
        except Exception:
            pass
    return Box


def make_spaces(nu, obs_dim, normalize_act=True, ctrlrange=None):
    """env_base.py:145-155 (action) and :210-218 (observation)."""
    B = box_class()
    if normalize_act or ctrlrange is None:
        lo, hi = -np.ones(nu, dtype=np.float32), np.ones(nu, dtype=np.float32)
    else:
        lo, hi = np.asarray(ctrlrange[:, 0], dtype=np.float32), np.asarray(ctrlrange[:, 1], dtype=np.float32)
    return B(lo, hi, dtype=np.float32), B(-10 * np.ones(obs_dim, dtype=np.float32), 10 * np.ones(obs_dim, dtype=np.float32), dtype=np.float32)


# --------------------------------------------------------------------------------------------- obs_dict
def obs_layout(task, nq, nv, na, ntip=0):
    """[(key, width)] in the order of the reference's DEFAULT_OBS_KEYS + "act" (base_v0.py:33-37)."""
    if task == "pose":
        return [("qpos", nq), ("qvel", nv), ("pose_err", nq), ("act", na)]
    if task in ("reach", "stand"):
        return [("qpos", nq), ("qvel", nv), ("tip_pos", 3 * ntip), ("reach_err", 3 * ntip), ("act", na)]
    if task == "hold":
        return [("hand_qpos", nq - 7), ("hand_qvel", nv - 6), ("obj_pos", 3), ("obj_err", 3), ("act", na)]
    if task == "walk":
        return [("qpos_without_xy", nq - 2), ("qvel", nv), ("com_vel", 2), ("torso_angle", 4), ("feet_heights", 2), ("height", 1), ("feet_rel_positions", 6),
                ("phase_var", 1), ("muscle_length", na), ("muscle_velocity", na), ("muscle_force", na), ("act", na)]
    raise KeyError(task)


def obs_dict_from_vec(task, obs, time, nq, nv, na, ntip=0):
    """obs: [..., obs_dim] (numpy) -> OrderedDict(time, key -> slice).  `qvel` entries are already scaled by dt, as in the reference."""
    d = collections.OrderedDict(time=np.asarray(time, dtype=np.float64))
    o = 0
    for k, wdt in obs_layout(task, nq, nv, na, ntip):
        d[k] = np.asarray(obs[..., o:o + wdt])
        o += wdt
    return d


# --------------------------------------------------------------------------------------------- rwd_dict
def reward_dict(task, obs_dict, weights, cfg):
    """The reference's get_reward_dict for the device tasks, on an obs_dict (batched over leading dims).
    cfg: task constants (pose_thd ; far_th, ntip, dt ; walk targets, hip_period ...).  Returns OrderedDict incl. sparse / solved / done / dense."""
    na = obs_dict["act"].shape[-1]
    act_mag = np.linalg.norm(obs_dict["act"], axis=-1) / na if na else 0.0
    if task == "pose":                                                     # pose_v0.py:113-140
        d = np.linalg.norm(obs_dict["pose_err"], axis=-1); far_th = cfg.get("pose_far_th", 4 * np.pi / 2); thd = cfg["pose_thd"]      # TorsoEnvV0: far_th = pi (torso_v0.py:104)
        r = collections.OrderedDict((("pose", -1.0 * d), ("bonus", 1.0 * (d < thd) + 1.0 * (d < 1.5 * thd)), ("penalty", -1.0 * (d > far_th)), ("act_reg", -1.0 * act_mag),
                                     ("sparse", -1.0 * d), ("solved", d < thd), ("done", d > far_th)))
    elif task == "reach":                                                  # reach_v0.py:120-160
        d = np.linalg.norm(obs_dict["reach_err"], axis=-1); ntip = cfg["ntip"]
        far_th = np.where(np.asarray(obs_dict["time"]) > 2 * cfg["dt"], cfg["far_th"] * ntip, np.inf); near = ntip * 0.0125
        r = collections.OrderedDict((("reach", -1.0 * d), ("bonus", 1.0 * (d < 2 * near) + 1.0 * (d < near)), ("act_reg", -1.0 * act_mag), ("penalty", -1.0 * (d > far_th)),
                                     ("sparse", -1.0 * d), ("solved", d < near), ("done", d > far_th)))
    elif task == "stand":                                                  # walk_v0.py:104-140 (ReachEnvV0 of the legs)
        d = np.linalg.norm(obs_dict["reach_err"], axis=-1); v = np.linalg.norm(obs_dict["qvel"], axis=-1); ntip = cfg["ntip"]
        far_th = np.where(np.squeeze(obs_dict["time"]) > 2 * cfg["dt"], cfg["far_th"] * ntip, np.inf); near = ntip * 0.050       # (squeezed as the reference does)
        r = collections.OrderedDict((("reach", 10.0 - 1.0 * d - 10.0 * v), ("bonus", 1.0 * (d < 2 * near) + 1.0 * (d < near)), ("act_reg", -100.0 * act_mag),
                                     ("penalty", -1.0 * (d > far_th)), ("sparse", -1.0 * d), ("solved", d < near), ("done", d > far_th)))
    elif task == "hold":                                                   # obj_hold_v0.py:92-121
        d = np.abs(np.linalg.norm(obs_dict["obj_err"], axis=-1)); th = 0.010; drop = d > 0.300
        r = collections.OrderedDict((("goal_dist", -1.0 * d), ("bonus", 1.0 * (d < 2 * th) + 1.0 * (d < th)), ("act_reg", -1.0 * act_mag), ("penalty", -1.0 * drop),
                                     ("sparse", -d), ("solved", d < th), ("done", drop)))
    elif task == "walk":                                                   # walk_v0.py:289-319, 358-494
        q = obs_dict["qpos_without_xy"]; cv = obs_dict["com_vel"]; phase = obs_dict["phase_var"][..., 0]
        vel = np.exp(-np.square(cfg["target_y_vel"] - cv[..., 1])) + np.exp(-np.square(cfg["target_x_vel"] - cv[..., 0]))
        des = np.stack([0.8 * np.cos(phase * 2 * np.pi + np.pi), 0.8 * np.cos(phase * 2 * np.pi)], -1).astype(np.float32)
        ang = np.stack([q[..., cfg["q_hip_flexion_l"] - 2], q[..., cfg["q_hip_flexion_r"] - 2]], -1)
        cyc = np.linalg.norm(des - ang, axis=-1)
        quat = q[..., 1:5]                                                 # qpos[3:7]
        ref_rot = np.exp(-np.linalg.norm(5.0 * (quat - np.asarray(cfg["target_rot"])), axis=-1))
        jr = np.exp(-5 * np.mean(np.abs(np.stack([q[..., cfg[k] - 2] for k in ("q_hip_adduction_l", "q_hip_adduction_r", "q_hip_rotation_l", "q_hip_rotation_r")], -1)), axis=-1))
        w_, x_, y_, z_ = (quat[..., i].astype(np.float64) for i in range(4)); nrm = w_ * w_ + x_ * x_ + y_ * y_ + z_ * z_
        r00 = 1.0 - 2.0 / nrm * (y_ * y_ + z_ * z_)
        done = (obs_dict["height"][..., 0] < cfg["min_height"]) | (np.abs(r00) > cfg["max_rot"])
        r = collections.OrderedDict((("vel_reward", vel), ("cyclic_hip", cyc), ("ref_rot", ref_rot), ("joint_angle_rew", jr), ("act_mag", act_mag),
                                     ("sparse", vel), ("solved", vel >= 1.0), ("done", done)))
    else:
        raise KeyError(task)
    r["dense"] = np.sum([wt * r[k] for k, wt in weights.items()], axis=0)
    return r


DEFAULT_WEIGHTS = {
    "pose": {"pose": 1.0, "bonus": 4.0, "act_reg": 1.0, "penalty": 50},                                               # pose_v0.py:18-23
    "reach": {"reach": 1.0, "bonus": 4.0, "penalty": 50},                                                              # reach_v0.py:18-22
    "stand": {"reach": 1.0, "bonus": 4.0, "penalty": 50, "act_reg": 1},                                              # walk_v0.py:18-24
    "hold": {"goal_dist": 100.0, "bonus": 4.0, "penalty": 10},                                                         # obj_hold_v0.py:17-21
    "walk": {"vel_reward": 5.0, "done": -100, "cyclic_hip": -10, "ref_rot": 10.0, "joint_angle_rew": 5.0},          # walk_v0.py:205-211
}


# --------------------------------------------------------------------------------------------- methods on paths (env_base.py:763-826)
def obsvec2obsdict(obsvec, key_widths):
    """ObsVecDict.obsvec2obsdict (obs_vec_dict.py:90-97): obsvec [num_traj, horizon, obs_dim] -> {key: [num_traj, horizon, width]} for the keys
    (and widths) that form the observation vector, in order."""
    obsvec = np.asarray(obsvec)
    assert obsvec.ndim == 3, "obsvec should be of shape (num_traj, horizon, obs_dim)"
    d, o = {}, 0
    for k, w in key_widths:
        d[k] = obsvec[:, :, o:o + w]; o += w
    assert o == obsvec.shape[-1], "observation width %d does not match the obs_keys (%d)" % (obsvec.shape[-1], o)
    return d


def compute_path_rewards(task, paths, key_widths, weights, cfg, rwd_mode="dense"):
    """MujocoEnv.compute_path_rewards (env_base.py:763-780): vectorised rewards / done flags of paths["observations"] [num_traj, horizon, obs_dim],
    time-aligned the way the reference does it (entry t takes the value computed from observation t+1; the last entry is redundant)."""
    od = obsvec2obsdict(paths["observations"], key_widths)
    if task in ("reach", "stand") and "time" not in od:
        raise KeyError("the reach reward needs obs_dict['time'] (reach_v0.py:127-131), which an observation vector does not carry")
    rd = reward_dict(task, od, weights, cfg)
    rewards, done = np.array(rd[rwd_mode], dtype=np.float64), np.array(rd["done"])
    done[..., :-1] = done[..., 1:]; rewards[..., :-1] = rewards[..., 1:]
    paths["done"] = done if done.shape[0] > 1 else done.ravel()
    paths["rewards"] = rewards if rewards.shape[0] > 1 else rewards.ravel()
    return paths


def truncate_paths(paths):
    """MujocoEnv.truncate_paths (env_base.py:782-796): cut every path at its first done flag and mark it terminated."""
    hor = paths[0]["rewards"].shape[0]
    for path in paths:
        if path["done"][-1] == False:          # noqa: E712  (the reference's own comparisons: done may be an object / float array)
            path["terminated"] = False
            terminated_idx = hor               # noqa: F841
        elif path["done"][0] == False:         # noqa: E712
            terminated_idx = sum(~np.asarray(path["done"], dtype=bool)) + 1
            for key in list(path.keys()):
                path[key] = path[key][: terminated_idx + 1, ...]
            path["terminated"] = True
    return paths


def evaluate_success(paths, horizon, logger=None, successful_steps=5):
    """MujocoEnv.evaluate_success (env_base.py:798-826): percentage of paths solved for more than `successful_steps` steps; optional mjrl-style logger."""
    num_success = sum(1 for p in paths if np.sum(np.asarray(p["env_infos"]["solved"]) * 1.0) > successful_steps)
    success_percentage = num_success * 100.0 / len(paths)
    if logger:
        logger.log_kv("rwd_sparse", np.mean([np.mean(p["env_infos"]["rwd_sparse"]) for p in paths]))
        logger.log_kv("rwd_dense", np.mean([np.sum(p["env_infos"]["rwd_dense"]) / horizon for p in paths]))
        logger.log_kv("success_percentage", success_percentage)
    return success_percentage
