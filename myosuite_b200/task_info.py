"""Host-side `info` quantities the reference returns next to (obs, reward, done): `rwd_sparse` and `solved`
(env_base.py:585-616 get_env_infos).  They are functions of the observation the kernel already wrote, so they are derived
lazily from it (numpy arrays or torch tensors, any device) instead of costing the kernel extra outputs.

  pose  (pose_v0.py:113-140):     dist = |pose_err|,   sparse = -dist, solved = dist < pose_thd
  reach (reach_v0.py:120-160):    dist = |reach_err|,  sparse = -dist, solved = dist < 0.0125 * ntip
  stand (walk_v0.py:104-140):     dist = |reach_err|,  sparse = -dist, solved = dist < 0.050 * ntip
  hold  (obj_hold_v0.py:92-121):  dist = |obj_err|,    sparse = -dist, solved = dist < 0.010
"""


def _norm_rows(x):
    if hasattr(x, "norm"):                 # torch
        return x.double().norm(dim=-1)
    import numpy as np
    return np.linalg.norm(np.asarray(x, dtype=np.float64), axis=-1)


def info_from_obs(task, obs, nq, nv, na, pose_thd=None, ntip=None):
    """obs: [n, obs_dim] in the task's reference layout -> dict(rwd_sparse [n], solved [n] bool); None for tasks without a
    distance-type success signal (walk)."""
    if task == "pose":
        err, thd = obs[..., nq + nv:nq + nv + nq], pose_thd
    elif task in ("reach", "stand"):
        base = nq + nv + 3 * ntip
        err, thd = obs[..., base:base + 3 * ntip], (0.0125 if task == "reach" else 0.050) * ntip
    elif task == "hold":
        base = (nq - 7) + (nv - 6) + 3
        err, thd = obs[..., base:base + 3], 0.010
    else:
        return None
    d = _norm_rows(err)
    return {"rwd_sparse": -d, "solved": d < thd}
