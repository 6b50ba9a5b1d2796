"""Gym-level drop-in surface of the reference's env classes (SURVEY.md section 8b "must be preserved"), host side only.

What the reference exposes on `env.unwrapped` and its tests exercise (myosuite/tests/test_envs.py:54-123):
  action_space / observation_space      envs/env_base.py:145-155, 210-218      (Box(-1, 1, nu) f32 ; Box(-10, 10, obs_dim) f32)
  obs_dict / rwd_dict                   envs/env_base.py:409-432               (per-key views of the observation; reward terms)
  get_obs_dict / get_reward_dict        myobase/pose_v0.py:100-140, reach_v0.py:98-160, obj_hold_v0.py:79-121, walk_v0.py:80-140,268-319
  get_env_infos                         envs/env_base.py:585-616
  get_env_state / set_env_state         envs/env_base.py:688-759
  seed / get_input_seed / pickling      envs/env_base.py:119-123, gym.utils.EzPickle (pose_v0.py:32)
The per-key quantities are all contained in the observation vector the kernel writes (obs_vec_dict.py:76-88 concatenates
them in `obs_keys` order + "act"), so the dicts are sliced / recomputed from that vector and a few state scalars on the host
(per task: myosuite_b200/tasks.py); nothing here touches the device.  Values therefore carry float32 precision where the reference's
dicts hold float64.  This module holds the task-independent part: the spaces and the methods on paths.
"""
import numpy as np

# the per-task obs / reward logic lives in tasks.py; its names stay importable from here, where callers of the gym surface found them
from .tasks import DEFAULT_WEIGHTS, obs_dict_from_vec, obs_layout, reward_dict  # noqa: F401


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
