"""Host-side facts of every device task, in one place: which reference entry point a task stands for, its kernel configuration, its
default reward weights and the order the kernel reads them in, its observation layout, its host reward dict and the `info` quantities
derived from the observation.  Nothing here touches a device: `configure` builds the `MyoTaskCfg` and the per-env initial buffers on the
CPU, and `MyoVecEnv` then allocates and binds them.

Tasks: pose (pose_v0.py PoseEnvV0, and torso_v0.py TorsoEnvV0 with its own flag), walk (walk_v0.py WalkEnvV0), hold (obj_hold_v0.py
ObjHold{Fixed,Random}EnvV0), reach (reach_v0.py ReachEnvV0) and stand (walk_v0.py ReachEnvV0 of the legs: the device's reach task with
its own reward shape and a randomised joint reset); "none" is a physics-only batch of a model (no obs, no reward, no reset sampling).
"""
import collections
import types

import numpy as np

from . import abi

# reference entry point (module:class) -> (task, torso, hold_random)
ENTRY_POINTS = {
    "pose_v0:PoseEnvV0": ("pose", False, False),
    "torso_v0:TorsoEnvV0": ("pose", True, False),       # the pose task with a fixed mean-of-range target, far_th = pi, pose_thd 0.25
    "walk_v0:WalkEnvV0": ("walk", False, False),
    "obj_hold_v0:ObjHoldFixedEnvV0": ("hold", False, False),
    "obj_hold_v0:ObjHoldRandomEnvV0": ("hold", False, True),
    "reach_v0:ReachEnvV0": ("reach", False, False),
    "walk_v0:ReachEnvV0": ("stand", False, False),
}
TASK_CODE = {"none": abi.TASK_NONE, "pose": abi.TASK_POSE, "walk": abi.TASK_WALK, "hold": abi.TASK_HOLD, "reach": abi.TASK_REACH, "stand": abi.TASK_REACH}

DEFAULT_WEIGHTS = {
    "pose": {"pose": 1.0, "bonus": 4.0, "act_reg": 1.0, "penalty": 50},                                               # pose_v0.py:18-23
    "reach": {"reach": 1.0, "bonus": 4.0, "penalty": 50},                                                              # reach_v0.py:18-22
    "stand": {"reach": 1.0, "bonus": 4.0, "penalty": 50, "act_reg": 1},                                              # walk_v0.py:18-24
    "hold": {"goal_dist": 100.0, "bonus": 4.0, "penalty": 10},                                                         # obj_hold_v0.py:17-21
    "walk": {"vel_reward": 5.0, "done": -100, "cyclic_hip": -10, "ref_rot": 10.0, "joint_angle_rew": 5.0},          # walk_v0.py:205-211
}
# cfg.weights[i] is the weight of WEIGHT_ORDER[task][i]; reach and stand count a missing weight as 0, the others require every key
WEIGHT_ORDER = {
    "pose": ("pose", "bonus", "act_reg", "penalty"),
    "walk": ("vel_reward", "done", "cyclic_hip", "ref_rot", "joint_angle_rew"),
    "hold": ("goal_dist", "bonus", "penalty"),
    "reach": ("reach", "bonus", "act_reg", "penalty"),
    "stand": ("reach", "bonus", "act_reg", "penalty"),
}

POSE_THD, TORSO_POSE_THD = 0.35, 0.25              # pose_v0.py:43 / torso_v0.py:52
POSE_FAR_TH, TORSO_FAR_TH = 4 * np.pi / 2, np.pi   # pose_v0.py:125 / torso_v0.py:104
REACH_FAR_TH, REACH_NEAR = 0.35, 0.0125            # reach_v0.py: far_th default, near_th per tip
STAND_SHAPE = (10.0, 10.0, 100.0, 0.05)            # cfg.reach_shape, walk_v0.py:104-140: reach = 10 - d - 10 |qvel dt|, act_reg = -100 |act|/na, near_th = 0.05 ntip
HOLD_TH, HOLD_DROP = 0.010, 0.300                  # obj_hold_v0.py:92-121
WALK_DEFAULTS = {"min_height": 0.8, "max_rot": 0.8, "hip_period": 100, "target_x_vel": 0.0, "target_y_vel": 1.2}     # myobase/__init__.py:443-458
HIP_JOINTS = ("hip_flexion_l", "hip_flexion_r", "hip_adduction_l", "hip_adduction_r", "hip_rotation_l", "hip_rotation_r")


def task_of(entry):
    """(task, torso, hold_random) of a reference entry point, None when no device task implements it."""
    return ENTRY_POINTS.get(entry.rsplit(".", 1)[-1])


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


# --------------------------------------------------------------------------------------------- rwd_dict and info
def _near(task, ntip):
    return ntip * (REACH_NEAR if task == "reach" else STAND_SHAPE[3])


def reward_dict(task, obs_dict, weights, cfg):
    """The reference's get_reward_dict for the device tasks, on an obs_dict (batched over leading dims).
    cfg: the host reward constants of `configure` (pose_thd ; far_th, ntip, dt ; walk targets ...).  Returns OrderedDict incl. sparse /
    solved / done / dense."""
    na = obs_dict["act"].shape[-1]
    act_mag = np.linalg.norm(obs_dict["act"], axis=-1) / na if na else 0.0
    if task in ("reach", "stand") and "time" not in obs_dict:
        raise KeyError("the reach reward needs obs_dict['time'] (reach_v0.py:127-131), which an observation vector does not carry")
    if task == "pose":                                                     # pose_v0.py:113-140
        d = np.linalg.norm(obs_dict["pose_err"], axis=-1); far_th = cfg.get("pose_far_th", POSE_FAR_TH); thd = cfg["pose_thd"]
        r = collections.OrderedDict((("pose", -1.0 * d), ("bonus", 1.0 * (d < thd) + 1.0 * (d < 1.5 * thd)), ("penalty", -1.0 * (d > far_th)), ("act_reg", -1.0 * act_mag),
                                     ("sparse", -1.0 * d), ("solved", d < thd), ("done", d > far_th)))
    elif task == "reach":                                                  # reach_v0.py:120-160
        d = np.linalg.norm(obs_dict["reach_err"], axis=-1); ntip = cfg["ntip"]
        far_th = np.where(np.squeeze(obs_dict["time"]) > 2 * cfg["dt"], cfg["far_th"] * ntip, np.inf); near = _near(task, ntip)      # (the single env's time is [1])
        r = collections.OrderedDict((("reach", -1.0 * d), ("bonus", 1.0 * (d < 2 * near) + 1.0 * (d < near)), ("act_reg", -1.0 * act_mag), ("penalty", -1.0 * (d > far_th)),
                                     ("sparse", -1.0 * d), ("solved", d < near), ("done", d > far_th)))
    elif task == "stand":                                                  # walk_v0.py:104-140 (ReachEnvV0 of the legs)
        c_off, c_vel, c_act, _ = STAND_SHAPE
        d = np.linalg.norm(obs_dict["reach_err"], axis=-1); v = np.linalg.norm(obs_dict["qvel"], axis=-1); ntip = cfg["ntip"]
        far_th = np.where(np.squeeze(obs_dict["time"]) > 2 * cfg["dt"], cfg["far_th"] * ntip, np.inf); near = _near(task, ntip)       # (squeezed as the reference does)
        r = collections.OrderedDict((("reach", c_off - 1.0 * d - c_vel * v), ("bonus", 1.0 * (d < 2 * near) + 1.0 * (d < near)), ("act_reg", -c_act * act_mag),
                                     ("penalty", -1.0 * (d > far_th)), ("sparse", -1.0 * d), ("solved", d < near), ("done", d > far_th)))
    elif task == "hold":                                                   # obj_hold_v0.py:92-121
        d = np.abs(np.linalg.norm(obs_dict["obj_err"], axis=-1)); th = HOLD_TH; drop = d > HOLD_DROP
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
        jr = np.exp(-5 * np.mean(np.abs(np.stack([q[..., cfg["q_" + j] - 2] for j in HIP_JOINTS[2:]], -1)), axis=-1))
        w_, x_, y_, z_ = (quat[..., i].astype(np.float64) for i in range(4)); nrm = w_ * w_ + x_ * x_ + y_ * y_ + z_ * z_
        r00 = 1.0 - 2.0 / nrm * (y_ * y_ + z_ * z_)
        done = (obs_dict["height"][..., 0] < cfg["min_height"]) | (np.abs(r00) > cfg["max_rot"])
        r = collections.OrderedDict((("vel_reward", vel), ("cyclic_hip", cyc), ("ref_rot", ref_rot), ("joint_angle_rew", jr), ("act_mag", act_mag),
                                     ("sparse", vel), ("solved", vel >= 1.0), ("done", done)))
    else:
        raise KeyError(task)
    r["dense"] = np.sum([wt * r[k] for k, wt in weights.items()], axis=0)
    return r


_DIST_KEY = {"pose": "pose_err", "reach": "reach_err", "stand": "reach_err", "hold": "obj_err"}


def _norm_rows(x):
    if hasattr(x, "norm"):                 # torch
        return x.double().norm(dim=-1)
    return np.linalg.norm(np.asarray(x, dtype=np.float64), axis=-1)


def info_from_obs(task, obs, nq, nv, na, pose_thd=None, ntip=None):
    """`rwd_sparse` / `solved` of the reference's info dict (env_base.py:585-616 get_env_infos), derived lazily from the observation the
    kernel already wrote (numpy arrays or torch tensors, any device) instead of costing the kernel extra outputs.
    obs: [n, obs_dim] in the task's layout -> dict(rwd_sparse [n], solved [n] bool); None for tasks without a distance-type success
    signal (walk).  sparse = -|err| and solved = |err| < the threshold reward_dict uses."""
    key = _DIST_KEY.get(task)
    if key is None:
        return None
    o = 0
    for k, w in obs_layout(task, nq, nv, na, ntip or 0):
        if k == key:
            break
        o += w
    thd = pose_thd if task == "pose" else HOLD_TH if task == "hold" else _near(task, ntip)
    d = _norm_rows(obs[..., o:o + w])
    return {"rwd_sparse": -d, "solved": d < thd}


# --------------------------------------------------------------------------------------------- kernel configuration
def _dyn(m, prog_info, body_name):
    return prog_info["dyn_body_ids"].index(m.name2id("body", body_name))


def stand_target_centre(m, tips, init_qpos):
    """[ntip, 3] world positions the leg stand task samples its targets around.  The reference samples them around the tip sites of
    a first generate_qpos() draw (walk_v0.py:142-174), then starts the episode from an independent second draw.  That centre is a
    constant only when no draw moves a tip site: every joint between a tip's body and the world has a range of zero width (the draw
    clips the one coordinate it touches to that range; the other coordinates of a free or ball joint keep init_qpos).  On the legs
    the pelvis hangs from the free root, whose range [0, 0] pins x.  Any other structure raises instead of sampling a different
    distribution."""
    from . import mjcf
    q = np.array(init_qpos, dtype=np.float64)
    for j in range(m.njnt):                         # the first draw, on the coordinates it pins
        if m.jnt_range[j][0] == m.jnt_range[j][1]:
            q[m.jnt_qposadr[j]] = m.jnt_range[j][0]
    kin, centre = mjcf.kinematics(m, q), []
    for name in tips:
        sid = m.name2id("site", name)
        b = int(m.site_bodyid[sid])
        while b != 0:
            for j in range(int(m.body_jntadr[b]), int(m.body_jntadr[b]) + int(m.body_jntnum[b])):
                if m.jnt_range[j][0] != m.jnt_range[j][1]:
                    raise NotImplementedError("stand task: joint %d moves tip site %r under the randomised reset, so its target centre is not constant" % (j, name))
            b = int(m.body_parentid[b])
        b = int(m.site_bodyid[sid])
        centre.append(kin["xpos"][b] + np.reshape(kin["xmat"][b], (3, 3)) @ m.site_pos[sid])
    return np.array(centre)


def _setup_walk(c, m, prog_info, kw):
    """WalkEnvV0 constants (walk_v0.py:235-266,358-494, registry myobase/__init__.py:443-458) and its reset keyframes."""
    from . import mjmath as mm
    cfg = c.cfg
    root, torso = m.name2id("body", "root"), m.name2id("body", "torso")
    q, b = np.array([1.0, 0, 0, 0]), torso
    while b != root:                                   # torso xquat = root quat (x) constant chain offset (no joints in between)
        if m.body_jntnum[b] != 0:
            raise NotImplementedError("torso must be rigidly attached to the free root body")
        q = mm.quat_mul(m.body_quat[b], q); b = int(m.body_parentid[b])
    hips = [int(m.jnt_qposadr[m.name2id("joint", j)]) for j in HIP_JOINTS]
    for i, v in enumerate([_dyn(m, prog_info, b_) for b_ in ("root", "talus_l", "talus_r", "pelvis")] + hips):
        cfg.task_i[i] = v
    wk = {k: kw.get(k, d) for k, d in WALK_DEFAULTS.items()}
    target_rot = kw.get("target_rot") if kw.get("target_rot") is not None else m.key_qpos[0][3:7]      # init_qpos = key_qpos[0] (walk_v0.py:258)
    td = list(q) + [wk[k] for k in ("min_height", "max_rot", "hip_period", "target_x_vel", "target_y_vel")] + list(target_rot) + [float(np.sum(m.body_mass))]
    for i, v in enumerate(td):
        cfg.task_d[i] = float(v)
    c.reward_cfg.update(target_x_vel=wk["target_x_vel"], target_y_vel=wk["target_y_vel"], min_height=wk["min_height"], max_rot=wk["max_rot"],
                        target_rot=np.asarray(target_rot, dtype=np.float64))
    c.reward_cfg.update(("q_" + j, a) for j, a in zip(HIP_JOINTS, hips))
    rt = kw.get("reset_type", "init")                                                      # walk_v0.py:344-352
    if rt == "random":       # keyframe 2 or 3 + N(0, 0.02) noise, drawn in the kernel (walk_v0.py:321-337): two rows
        c.init_qpos, c.init_qvel = np.stack([m.key_qpos[2], m.key_qpos[3]]), np.stack([m.key_qvel[2], m.key_qvel[3]])
    else:
        key = 2 if rt == "init" else 0
        c.init_qpos, c.init_qvel = m.key_qpos[key].copy(), m.key_qvel[key].copy()


def _setup_hold(c, m, prog_info, kw):
    """ObjHold constants (obj_hold_v0.py:46-62,126-145): object and goal sites, and the per-env goal / object size defaults."""
    from . import mjcf
    cfg = c.cfg
    c.init_qpos[:-7] = 0.0; c.init_qpos[0] = -1.5                                                  # obj_hold_v0.py:61-62
    cfg.reset_random = int(c.hold_random)
    obj_body, sid, gid = m.name2id("body", "object"), m.name2id("site", "object"), m.name2id("geom", "object")
    pg = {v: k for k, v in prog_info["geom_model_ids"].items()}[gid]
    cfg.task_i[0], cfg.task_i[1] = _dyn(m, prog_info, "object"), pg
    kin = mjcf.kinematics(m, m.qpos0)
    obj_init = kin["xpos"][obj_body] + kin["xmat"][obj_body] @ m.site_pos[sid]                    # object_init_pos (obj_hold_v0.py:52)
    goal = m.site_pos[m.name2id("site", "goal")]
    for i in range(3):
        cfg.task_d[i] = m.site_pos[sid][i]; cfg.task_d[3 + i] = obj_init[i]; cfg.task_d[6 + i] = goal[i]; cfg.task_d[9 + i] = m.geom_size[gid][i]
    c.env_prm = np.array([cfg.task_d[6 + i] for i in range(6)])                                   # env_prm[0:6]: goal, object size


def _setup_reach(c, m, prog_info, kw):
    """ReachEnvV0 constants (reach_v0.py:52-67): tip sites (body + offset), world-fixed target sites, far_th."""
    cfg = c.cfg
    tips = list(kw["target_reach_range"].keys())
    if 3 * len(tips) > m.nq or len(tips) > 7:
        raise NotImplementedError("reach task: at most 7 tips and 3*ntip <= nq")
    cfg.task_i[0] = len(tips)
    dyn = prog_info["dyn_body_ids"]
    for k, name in enumerate(tips):
        sid, tid = m.name2id("site", name), m.name2id("site", name + "_target")
        if int(m.site_bodyid[tid]) != 0:
            raise NotImplementedError("reach targets must be world-fixed sites")
        b = int(m.site_bodyid[sid])
        cfg.task_i[1 + k] = dyn.index(b) if b in dyn else -1
        for i in range(3):
            cfg.task_d[3 * k + i] = float(m.site_pos[sid][i])
    cfg.task_d[3 * len(tips)] = float(kw.get("far_th", REACH_FAR_TH))
    c.tip_names = tips


def _setup_stand(c, m, prog_info, kw):
    """walk_v0.py ReachEnvV0 (walk_v0.py:49-79,104-186): the reach constants, keyframe 0, reward shape, randomised joint reset and the
    target centre (stand_target_centre)."""
    c.init_qpos, c.init_qvel = m.key_qpos[0].copy(), m.key_qvel[0].copy()                  # walk_v0.py:65-66
    _setup_reach(c, m, prog_info, kw)
    lo, hi = (float(x) for x in kw.get("joint_random_range", (0.0, 0.0)))
    if not hi > lo:
        raise NotImplementedError("stand task without joint randomisation: the reference then samples the target around the previous episode's last state")
    for i, v in enumerate(STAND_SHAPE):
        c.cfg.reach_shape[i] = v
    c.cfg.joint_random[0], c.cfg.joint_random[1] = lo, hi
    c.target_center = stand_target_centre(m, c.tip_names, c.init_qpos)


_SETUP = {"walk": _setup_walk, "hold": _setup_hold, "reach": _setup_reach, "stand": _setup_stand}


def _target_range(c, m, kw):
    """[nq, 2] sampling range of `target` per row: pose targets per qpos (pose_v0.py:60-70, "fixed" targets collapse the range); reach rows
    3k..3k+2 span target site k (reach_v0.py:163-170), the stand task's around its constant tip position (walk_v0.py:142-150)."""
    tr = np.zeros((m.nq, 2))
    if kw.get("target_jnt_range"):
        for jn, (lo, hi) in kw["target_jnt_range"].items():
            qa = m.jnt_qposadr[m.name2id("joint", jn)]
            tr[qa] = (0.5 * (lo + hi),) * 2 if c.torso else (lo, hi)     # TorsoEnvV0 never resamples: target = mean of the range (torso_v0.py:66-68)
    elif kw.get("target_jnt_value") is not None:
        v = np.asarray(kw["target_jnt_value"], dtype=np.float64)
        tr[:, 0] = tr[:, 1] = v
    elif c.tip_names:
        for k, span in enumerate(kw["target_reach_range"].values()):
            centre = c.target_center[k] if c.target_center is not None else 0.0
            tr[3 * k:3 * k + 3, 0], tr[3 * k:3 * k + 3, 1] = centre + np.asarray(span[0], dtype=np.float64), centre + np.asarray(span[1], dtype=np.float64)
    return tr


def site_sources(task, m, kw, tip_names):
    """int32 [nsite, 2] (kind, index) of the sites whose model site_pos the reference moves per episode (abi.SITE_* kinds, the
    myo_data_buffers.site_source of the mjData readout), or None when the task moves none:
      reach / stand  <tip>_target = the target row's 3 values of that tip (reach_v0.py:163-170, walk_v0.py:142-150)
      hold           goal = env_prm[0:3] (obj_hold_v0.py:126-145)
      pose           <tip>_target of every viz_site_targets tip = the tip site at the kinematics of the target pose (pose_v0.py:154-170)"""
    src = np.zeros((m.nsite, 2), dtype=np.int32)
    if task in ("reach", "stand"):
        for k, name in enumerate(tip_names):
            src[m.name2id("site", name + "_target")] = (abi.SITE_TARGET, 3 * k)
    elif task == "hold":
        src[m.name2id("site", "goal")] = (abi.SITE_ENV_PRM, 0)
    elif task == "pose":
        for name in kw.get("viz_site_targets") or ():
            src[m.name2id("site", name + "_target")] = (abi.SITE_AT_TARGET_POSE, m.name2id("site", name))
    return src if np.any(src[:, 0]) else None


def configure(entry, m, prog_info, kw, max_episode_steps=0, auto_reset=True):
    """Everything a batch of `entry` (a reference entry point, None for physics only) needs besides the device, from the model `m`, its
    program info (program.build_program) and the env kwargs.  Returns a namespace with
      task, torso, hold_random      the task and its variant flags
      cfg                           the abi.MyoTaskCfg passed to myo_batch_create
      frame_skip, dt, n_frames      control step
      init_qpos, init_qvel          reset rows ([2, nq] / [2, nv] for walk's random reset)
      target_range                  [nq, 2]
      tip_names, target_center      reach sites (empty otherwise) and the stand task's target centre (None otherwise)
      env_prm                       hold: the per-env goal / object size defaults [6] (None otherwise)
      fatigue_reset_vec             the validated fatigue reset vector, or None
      layout                        obs_layout of the task ([] for physics only)
      reward_cfg                    host reward constants for reward_dict"""
    kind = ("none", False, False) if entry is None else task_of(entry)
    if kind is None:
        raise NotImplementedError("device task for %s is not built yet (pose, torso, walk, hold, reach, stand are; MyoVecEnv.from_model gives physics only)" % entry)
    task, torso, hold_random = kind
    if kw.get("joint_random_range") is not None and task != "stand":
        raise NotImplementedError("joint_random_range is implemented for the leg stand task (walk_v0.py ReachEnvV0) only")
    c = types.SimpleNamespace(task=task, torso=torso, hold_random=hold_random, cfg=abi.MyoTaskCfg(), tip_names=[], target_center=None, env_prm=None)
    cfg = c.cfg
    c.frame_skip = int(kw.get("frame_skip", 10))
    c.dt = m.opt_timestep * c.frame_skip
    c.n_frames = int(c.dt / m.opt_timestep)      # robot.py:901
    cfg.task = TASK_CODE[task]
    cfg.frame_skip = c.n_frames
    cfg.max_episode_steps = int(max_episode_steps or 0)
    cfg.normalize_act = int(bool(kw.get("normalize_act", True)))
    muscle_condition = kw.get("muscle_condition", "")
    cfg.muscle_condition = abi.COND_FATIGUE if muscle_condition == "fatigue" else abi.COND_NONE
    # fatigue state at reset (base_v0.py:120-128 -> fatigue.py:82-99)
    c.fatigue_reset_vec = None if kw.get("fatigue_reset_vec") is None else np.asarray(kw["fatigue_reset_vec"], dtype=np.float64).ravel()
    if c.fatigue_reset_vec is not None and len(c.fatigue_reset_vec) != m.na:
        raise AssertionError("Invalid length of initial/reset fatigue vector (expected %d, but obtained %d)" % (m.na, len(c.fatigue_reset_vec)))      # fatigue.py:91
    cfg.fatigue_reset = 1 if kw.get("fatigue_reset_random") else (2 if c.fatigue_reset_vec is not None else 0)
    cfg.auto_reset = int(bool(auto_reset))
    cfg.reset_random = int(kw.get("reset_type", "init") == "random")
    cfg.pose_thd = float(kw.get("pose_thd", TORSO_POSE_THD if torso else POSE_THD))
    if torso:
        cfg.task_d[0] = float(TORSO_FAR_TH)
    cfg.solver_tolerance = float(kw.get("solver_tolerance", 0.0))
    cfg.maxcon = int(kw.get("maxcon", 0))
    cfg.barrier_mode = int(kw.get("barrier_mode", 0))
    cfg.reserved_i = int(kw.get("lockstep_groups", 0))
    cfg.reserved[0] = float(bool(kw.get("profile_waits", False)))
    cfg.reaf_dst = cfg.reaf_src = -1
    if muscle_condition == "reafferentation":   # base_v0.py:78-79,104-108
        cfg.reaf_dst, cfg.reaf_src = m.name2id("actuator", "EPL"), m.name2id("actuator", "EIP")
    # reward weights in kernel order (a physics-only batch carries the pose weights, which it never reads)
    wt = "pose" if task == "none" else task
    w = kw.get("weighted_reward_keys", DEFAULT_WEIGHTS[wt])
    for i, k in enumerate(WEIGHT_ORDER[wt]):
        cfg.weights[i] = w.get(k, 0.0) if wt in ("reach", "stand") else w[k]
    c.init_qpos, c.init_qvel = np.asarray(m.qpos0, dtype=np.float64).copy(), np.zeros(m.nv)
    c.reward_cfg = {"pose_thd": float(cfg.pose_thd), "dt": c.dt, "ntip": 0, "far_th": float(kw.get("far_th", REACH_FAR_TH))}
    if torso:
        c.reward_cfg["pose_far_th"] = float(TORSO_FAR_TH)
    if task in _SETUP:
        _SETUP[task](c, m, prog_info, kw)
    c.reward_cfg["ntip"] = len(c.tip_names)
    c.target_range = _target_range(c, m, kw)
    c.layout = [] if task == "none" else obs_layout(task, m.nq, m.nv, m.na, len(c.tip_names))
    return c
