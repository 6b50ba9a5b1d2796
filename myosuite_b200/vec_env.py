"""Batched env mirror of the reference's BaseV0 / PoseEnvV0 stack on top of the C-ABI library.

Reference interface mirrored (same names, argument meaning, return layout):
  * ``gym.make(id)`` registry ids + kwargs      myosuite/envs/myo/myobase/__init__.py:124-138,402-415
  * ``env.reset() -> (obs, info)``               myosuite/envs/env_base.py:647-654
  * ``env.step(a) -> (obs, reward, terminated, truncated, info)``   envs/env_base.py:403-407, envs/myo/base_v0.py:82-118
  * muscle-condition variants myoFati*/myoSarc*/myoReaf*           myobase/__init__.py:17-49, base_v0.py:60-79
All per-env state lives in torch CUDA tensors owned here and bound to the library by pointer.
"""
import json
import os

import numpy as np

from . import abi, assets, blob, program

_HERE = os.path.dirname(os.path.abspath(__file__))
_REG = None


def registry():
    global _REG
    if _REG is None:
        _REG = json.load(open(os.path.join(_HERE, "assets", "registry.json")))
    return _REG


def env_spec(env_id):
    """id -> (max_episode_steps, merged kwargs) including the Sarc/Fati/Reaf variants."""
    reg = registry()
    if env_id in reg["envs"]:
        e = reg["envs"][env_id]
        return e["max_episode_steps"], dict(e["kwargs"]), e["entry_point"]
    if env_id in reg["variants"]:
        v = reg["variants"][env_id]
        steps, kw, ep = env_spec(v["base"])
        kw.update(v["variants"])
        return steps, kw, ep
    raise KeyError("unknown env id %r (known: %s)" % (env_id, sorted(reg["envs"]) + sorted(reg["variants"])))


def registered_ids():
    reg = registry()
    return sorted(reg["envs"]) + sorted(reg["variants"])


_MODEL_OF_XML = {v[0]: k for k, v in assets.MODEL_XML.items()}


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


class MyoVecEnv:
    """n independent envs of one registry id, resident on one GPU.  Tensors in, tensors out."""

    @classmethod
    def from_model(cls, model_name, num_envs, **kw):
        """Physics-only batch of a named model asset (no task logic: obs_dim 0, no reset sampling)."""
        return cls(None, num_envs, model=assets.load(model_name), **kw)

    def __init__(self, env_id, num_envs, device=0, seed=0, env_offset=0, auto_reset=True, taps=False, model=None, **overrides):
        import torch
        self.torch = torch
        if not torch.cuda.is_available():
            raise RuntimeError("MyoVecEnv needs a CUDA device: the physics has no CPU fallback (the CPU oracle under oracle/ is test-only)")
        self.env_id, self.num_envs, self.seed_value, self.env_offset = env_id, int(num_envs), int(seed), int(env_offset)
        if env_id is None:
            self.max_episode_steps, kw, entry = 0, {"normalize_act": True}, None
            auto_reset = False
        else:
            self.max_episode_steps, kw, entry = env_spec(env_id)
        kw.update(overrides)
        self.kwargs = kw
        self._check_kwargs(kw)
        self.torso = entry is not None and entry.endswith("torso_v0:TorsoEnvV0")        # TorsoEnvV0 = the pose task with a fixed mean-of-range target, far_th = pi, pose_thd 0.25
        # "stand": walk_v0.py's ReachEnvV0 (myoLegStandRandom), the device's reach task with its own reward shape and randomised joint reset
        self.task = ("none" if entry is None else "pose" if (entry.endswith("pose_v0:PoseEnvV0") or self.torso) else "walk" if entry.endswith("walk_v0:WalkEnvV0")
                     else "hold" if "obj_hold_v0:ObjHold" in entry else "reach" if entry.endswith("reach_v0:ReachEnvV0")
                     else "stand" if entry.endswith("walk_v0:ReachEnvV0") else None)
        if self.task is None:
            raise NotImplementedError("device task for %s (%s) is not built yet (pose, torso, walk, hold, reach, stand are; MyoVecEnv.from_model gives physics only)" % (env_id, entry))
        if kw.get("joint_random_range") is not None and self.task != "stand":
            raise NotImplementedError("joint_random_range is implemented for the leg stand task (walk_v0.py ReachEnvV0) only")
        self.hold_random = entry is not None and entry.endswith("ObjHoldRandomEnvV0")
        self.mj_model = m = model if model is not None else assets.load(_MODEL_OF_XML[kw["model_path"]])
        self.muscle_condition = kw.get("muscle_condition", "")
        if self.muscle_condition == "sarcopenia":       # base_v0.py:62-67: gainprm[:,2] *= 0.5 (biasprm untouched)
            import copy
            self.mj_model = m = copy.deepcopy(m)
            m.actuator_gainprm[:, 2] *= 0.5
        self.frame_skip = int(kw.get("frame_skip", 10))
        self.dt = m.opt_timestep * self.frame_skip
        self.n_frames = int(self.dt / m.opt_timestep)      # robot.py:901
        prog, self.prog_info = program.build_program(m)
        self.prog = prog
        self.I, self.D = blob.pack(m, prog)
        # row_storage: "p48" (product: contact Jacobian rows held as the upper 48 bits of the f64 value -- 36 mantissa bits -- in shared memory,
        # 14 env-warps per SM on the hand) or "f64" (verification build of the same source, abi.lib("f64rows"): plain doubles, fewer warps)
        self.row_storage = kw.get("row_storage", "p48")
        if self.row_storage not in ("p48", "f64"):
            raise ValueError("row_storage must be 'p48' or 'f64'")
        self.dev_model = abi.DeviceModel(self.I, self.D, variant="f64rows" if self.row_storage == "f64" else None)
        cfg = abi.MyoTaskCfg()
        cfg.task = {"none": abi.TASK_NONE, "pose": abi.TASK_POSE, "walk": abi.TASK_WALK, "hold": abi.TASK_HOLD, "reach": abi.TASK_REACH, "stand": abi.TASK_REACH}[self.task]
        cfg.frame_skip = self.n_frames
        cfg.max_episode_steps = int(self.max_episode_steps or 0)
        cfg.normalize_act = int(bool(kw.get("normalize_act", True)))
        cfg.muscle_condition = abi.COND_FATIGUE if self.muscle_condition == "fatigue" else abi.COND_NONE
        # fatigue state at reset (base_v0.py:120-128 -> fatigue.py:82-99)
        self.fatigue_reset_vec = None if kw.get("fatigue_reset_vec") is None else np.asarray(kw["fatigue_reset_vec"], dtype=np.float64).ravel()
        if self.fatigue_reset_vec is not None and len(self.fatigue_reset_vec) != m.na:
            raise AssertionError("Invalid length of initial/reset fatigue vector (expected %d, but obtained %d)" % (m.na, len(self.fatigue_reset_vec)))      # fatigue.py:91
        cfg.fatigue_reset = 1 if kw.get("fatigue_reset_random") else (2 if self.fatigue_reset_vec is not None else 0)
        cfg.auto_reset = int(bool(auto_reset))
        cfg.reset_random = int(kw.get("reset_type", "init") == "random")
        cfg.pose_thd = float(kw.get("pose_thd", 0.25 if self.torso else 0.35))         # pose_v0.py:43 / torso_v0.py:52
        if self.torso:
            cfg.task_d[0] = float(np.pi)                                                # far_th (torso_v0.py:104)
        init_qpos, init_qvel = np.asarray(m.qpos0, dtype=np.float64).copy(), np.zeros(m.nv)
        if self.task in ("pose", "none"):
            w = kw.get("weighted_reward_keys", {"pose": 1.0, "bonus": 4.0, "act_reg": 1.0, "penalty": 50})     # pose_v0.py:18-23
            for i, k in enumerate(("pose", "bonus", "act_reg", "penalty")):
                cfg.weights[i] = w[k]
        elif self.task == "walk":
            w = kw.get("weighted_reward_keys", {"vel_reward": 5.0, "done": -100, "cyclic_hip": -10, "ref_rot": 10.0, "joint_angle_rew": 5.0})   # walk_v0.py:205-211
            for i, k in enumerate(("vel_reward", "done", "cyclic_hip", "ref_rot", "joint_angle_rew")):
                cfg.weights[i] = w[k]
            self._setup_walk(m, kw, cfg, prog_info=None)
            rt = kw.get("reset_type", "init")                                                      # walk_v0.py:344-352
            if rt == "random":       # keyframe 2 or 3 + N(0, 0.02) noise, drawn in the kernel (walk_v0.py:321-337): two rows
                init_qpos, init_qvel = np.stack([m.key_qpos[2], m.key_qpos[3]]), np.stack([m.key_qvel[2], m.key_qvel[3]])
            else:
                key = 2 if rt == "init" else 0
                init_qpos, init_qvel = m.key_qpos[key].copy(), m.key_qvel[key].copy()
        elif self.task == "hold":
            w = kw.get("weighted_reward_keys", {"goal_dist": 100.0, "bonus": 4.0, "penalty": 10})     # obj_hold_v0.py:17-21
            for i, k in enumerate(("goal_dist", "bonus", "penalty")):
                cfg.weights[i] = w[k]
            init_qpos[:-7] = 0.0; init_qpos[0] = -1.5                                                  # obj_hold_v0.py:61-62
            cfg.reset_random = int(self.hold_random)
        elif self.task in ("reach", "stand"):
            w = kw.get("weighted_reward_keys", {"reach": 1.0, "bonus": 4.0, "penalty": 50} if self.task == "reach"      # reach_v0.py:18-22
                       else {"reach": 1.0, "bonus": 4.0, "penalty": 50, "act_reg": 1})                                     # walk_v0.py:18-24
            for i, k in enumerate(("reach", "bonus", "act_reg", "penalty")):
                cfg.weights[i] = w.get(k, 0.0)
            if self.task == "stand":     # walk_v0.py:65-66: init_qpos / init_qvel = keyframe 0
                init_qpos, init_qvel = m.key_qpos[0].copy(), m.key_qvel[0].copy()
        cfg.solver_tolerance = float(kw.get("solver_tolerance", 0.0))
        cfg.maxcon = int(kw.get("maxcon", 0))
        cfg.barrier_mode = int(kw.get("barrier_mode", 0))
        cfg.reserved_i = int(kw.get("lockstep_groups", 0))
        cfg.reserved[0] = float(bool(kw.get("profile_waits", False)))
        cfg.reaf_dst = cfg.reaf_src = -1
        if self.muscle_condition == "reafferentation":   # base_v0.py:78-79,104-108
            cfg.reaf_dst, cfg.reaf_src = m.name2id("actuator", "EPL"), m.name2id("actuator", "EIP")
        if self.task == "hold":
            self._setup_hold(m, cfg)
        if self.task in ("reach", "stand"):
            self._setup_reach(m, kw, cfg)
        if self.task == "stand":
            self._setup_stand(m, kw, cfg, init_qpos)
        self.cfg = cfg
        self.device_index = int(device)
        self.device = torch.device("cuda", self.device_index)
        self.batch = abi.Batch(self.dev_model, self.device_index, self.num_envs, cfg)
        self.dims = self.dev_model.dims(cfg)
        n, dv = self.num_envs, self.device
        f64, f32 = torch.float64, torch.float32
        z = lambda *s, dtype=f64: torch.zeros(*s, dtype=dtype, device=dv)
        self.full_obs_dim = self.obs_dim = max(self.batch.obs_dim, 1); self.act_dim = m.nu
        # custom obs_keys (env_base.py:110,190,458 obsdict2obsvec over `obs_keys`; base_v0.py:33-37 appends "act"): the kernel always writes the
        # task's full default layout into t["obs_full"]; t["obs"] is the gather of the requested keys' columns, refreshed after every launch
        self._obs_cols = None
        if kw.get("obs_keys") is not None and self.task != "none":
            from . import gym_api
            keys = list(kw["obs_keys"])
            if m.na > 0 and "act" not in keys:
                keys.append("act")
            lay, off, o = gym_api.obs_layout(self.task, m.nq, m.nv, m.na, len(getattr(self, "tip_names", ()))), {}, 0
            for k_, w_ in lay:
                off[k_] = (o, w_); o += w_
            missing = [k_ for k_ in keys if k_ not in off]
            if missing:
                raise KeyError("obs_keys not available from this task's obs_dict: %s (available: %s)" % (missing, [k_ for k_, _ in lay]))
            self.obs_keys = keys
            if keys != [k_ for k_, _ in lay]:
                cols = np.concatenate([np.arange(off[k_][0], off[k_][0] + off[k_][1]) for k_ in keys])
                self._obs_cols, self._obs_cols_np = torch.as_tensor(cols, dtype=torch.int64, device=self.device), cols
                self.obs_dim = int(len(cols))
        t = dict(action=z(n, m.nu, dtype=f32), qpos=z(n, m.nq), qvel=z(n, m.nv), act=z(n, max(m.na, 1)), qacc_warmstart=z(n, m.nv),
                 time=z(n), target=z(n, m.nq), step_count=z(n, dtype=torch.int32), episode_count=z(n, dtype=torch.int64),
                 obs=z(n, self.full_obs_dim, dtype=f32), reward=z(n, dtype=f32), done=z(n, dtype=torch.uint8), truncated=z(n, dtype=torch.uint8),
                 ep_return=z(n, dtype=f32), last_return=z(n, dtype=f32), overflow=z(n, dtype=torch.int32))
        t["qpos"][:] = torch.as_tensor(m.qpos0, device=dv)
        # target ranges per qpos (pose_v0.py:60-70); "fixed" targets collapse the range
        tr = np.zeros((m.nq, 2))
        if kw.get("target_jnt_range"):
            for jn, (lo, hi) in kw["target_jnt_range"].items():
                qa = m.jnt_qposadr[m.name2id("joint", jn)]
                tr[qa] = (0.5 * (lo + hi),) * 2 if self.torso else (lo, hi)     # TorsoEnvV0 never resamples: target = mean of the range (torso_v0.py:66-68)
        elif kw.get("target_jnt_value") is not None:
            v = np.asarray(kw["target_jnt_value"], dtype=np.float64)
            tr[:, 0] = tr[:, 1] = v
        elif self.task in ("reach", "stand"):       # rows 3k..3k+2: span of target site k (reach_v0.py:163-170); `target` rows hold the sampled site positions
            for k, span in enumerate(kw["target_reach_range"].values()):         # stand: around the constant tip position of the first draw (walk_v0.py:142-150)
                c = self.target_center[k] if self.task == "stand" else 0.0
                tr[3 * k:3 * k + 3, 0], tr[3 * k:3 * k + 3, 1] = c + np.asarray(span[0], dtype=np.float64), c + np.asarray(span[1], dtype=np.float64)
        t["target_range"] = torch.as_tensor(tr, device=dv).contiguous()
        t["init_qpos"] = torch.as_tensor(init_qpos, device=dv).contiguous()
        t["init_qvel"] = torch.as_tensor(init_qvel, device=dv).contiguous()
        self.init_qpos, self.init_qvel = init_qpos, init_qvel
        if self.task == "hold":
            t["env_prm"] = z(n, 8)
            t["env_prm"][:, :6] = torch.as_tensor(np.array([cfg.task_d[6 + i] for i in range(6)]), device=dv)
        if cfg.muscle_condition == abi.COND_FATIGUE:
            t["fatigue"] = z(n, 3, m.nu)
            t["fatigue"][:, 1, :] = 1.0
            if self.fatigue_reset_vec is not None:
                t["fatigue_reset_vec"] = torch.as_tensor(self.fatigue_reset_vec, device=dv).contiguous()
        if taps:
            t.update(tap_qacc=z(n, m.nv), tap_actuator_force=z(n, m.nu), tap_ten_length=z(n, m.nu), tap_qfrc_smooth=z(n, m.nv),
                     tap_ncon=z(n, 4, dtype=torch.int32), tap_contact_pair=z(n, max(self.dims.maxcon, 1), dtype=torch.int32),
                     tap_contact_dist=z(n, max(self.dims.maxcon, 1)), tap_moment=z(n, max(self.dims.reserved[0], 1)), tap_qM=z(n, m.nM),
                     tap_phase_cycles=z(n, 20, dtype=torch.int64))
        self.t = t
        self.batch.bind(**t)
        t["obs_full"] = t["obs"]                                  # what the kernel writes (bound above); t["obs"] is what callers see
        if self._obs_cols is not None:
            t["obs"] = z(n, self.obs_dim, dtype=f32)
        self._h_action = None

    def _sync_obs(self):
        if self._obs_cols is not None:
            self.torch.index_select(self.t["obs_full"], 1, self._obs_cols, out=self.t["obs"])

    # kwargs of the reference's env classes this backend implements; anything else with a non-default value is an error, not a silent no-op
    _KNOWN = {"model_path", "normalize_act", "frame_skip", "muscle_condition", "reset_type", "target_type", "pose_thd", "weighted_reward_keys", "target_jnt_range",
              "target_jnt_value", "viz_site_targets", "target_reach_range", "far_th", "min_height", "max_rot", "hip_period", "target_x_vel", "target_y_vel", "target_rot",
              "obs_keys", "fatigue_reset_vec", "fatigue_reset_random", "weight_bodyname", "weight_range", "joint_random_range",
              # backend knobs
              "solver_tolerance", "maxcon", "barrier_mode", "lockstep_groups", "profile_waits", "row_storage"}

    @staticmethod
    def _check_kwargs(kw):
        unknown = sorted(set(kw) - MyoVecEnv._KNOWN)
        if unknown:
            raise NotImplementedError("env kwargs not implemented by this backend: %s" % unknown)
        bad = []
        if kw.get("fatigue_reset_vec") is not None and kw.get("fatigue_reset_random"):
            raise AssertionError("Cannot use 'fatigue_reset_vec' if fatigue_reset_random=False.")          # (the reference's own assertion and wording, fatigue.py:84)
        if kw.get("reset_type", "init") not in ("init", "random"):
            bad.append("reset_type=%r (init and random are implemented)" % kw.get("reset_type"))
        if kw.get("target_type", "generate") == "switch":
            bad.append("target_type='switch'")
        if kw.get("weight_bodyname") is not None or kw.get("weight_range") is not None:
            bad.append("weight_bodyname / weight_range")
        if bad:
            raise NotImplementedError("reference kwargs accepted by the reference but not by this backend: " + "; ".join(bad))

    # ---------------------------------------------------------------- task parameter blocks (indices into the kernel's dynamic-body list)
    def _dyn(self, body_name):
        return self.prog_info["dyn_body_ids"].index(self.mj_model.name2id("body", body_name))

    def _setup_walk(self, m, kw, cfg, prog_info=None):
        """WalkEnvV0 constants (walk_v0.py:235-266,358-494, registry myobase/__init__.py:443-458)."""
        from . import mjmath as mm
        root, torso = m.name2id("body", "root"), m.name2id("body", "torso")
        q, b = np.array([1.0, 0, 0, 0]), torso
        while b != root:                                   # torso xquat = root quat (x) constant chain offset (no joints in between)
            if m.body_jntnum[b] != 0:
                raise NotImplementedError("torso must be rigidly attached to the free root body")
            q = mm.quat_mul(m.body_quat[b], q); b = int(m.body_parentid[b])
        ti = [self._dyn("root"), self._dyn("talus_l"), self._dyn("talus_r"), self._dyn("pelvis")]
        ti += [int(m.jnt_qposadr[m.name2id("joint", j)]) for j in ("hip_flexion_l", "hip_flexion_r", "hip_adduction_l", "hip_adduction_r", "hip_rotation_l", "hip_rotation_r")]
        for i, v in enumerate(ti):
            cfg.task_i[i] = v
        target_rot = kw.get("target_rot") if kw.get("target_rot") is not None else m.key_qpos[0][3:7]      # init_qpos = key_qpos[0] (walk_v0.py:258)
        td = list(q) + [kw.get("min_height", 0.8), kw.get("max_rot", 0.8), kw.get("hip_period", 100), kw.get("target_x_vel", 0.0), kw.get("target_y_vel", 1.2)] + \
            list(target_rot) + [float(np.sum(m.body_mass))]
        for i, v in enumerate(td):
            cfg.task_d[i] = float(v)

    def _setup_reach(self, m, kw, cfg):
        """ReachEnvV0 constants (reach_v0.py:52-67): tip sites (body + offset), world-fixed target sites, far_th."""
        tips = list(kw["target_reach_range"].keys())
        if 3 * len(tips) > m.nq or len(tips) > 7:
            raise NotImplementedError("reach task: at most 7 tips and 3*ntip <= nq")
        cfg.task_i[0] = len(tips)
        dyn = self.prog_info["dyn_body_ids"]
        for k, name in enumerate(tips):
            sid, tid = m.name2id("site", name), m.name2id("site", name + "_target")
            if int(m.site_bodyid[tid]) != 0:
                raise NotImplementedError("reach targets must be world-fixed sites")
            b = int(m.site_bodyid[sid])
            cfg.task_i[1 + k] = dyn.index(b) if b in dyn else -1
            for c in range(3):
                cfg.task_d[3 * k + c] = float(m.site_pos[sid][c])
        cfg.task_d[3 * len(tips)] = float(kw.get("far_th", 0.35))
        self.tip_names = tips

    STAND_SHAPE = (10.0, 10.0, 100.0, 0.05)      # walk_v0.py:104-140: reach = 10 - d - 10 |qvel dt|, act_reg = -100 |act|/na, near_th = 0.05 ntip

    def _setup_stand(self, m, kw, cfg, init_qpos):
        """walk_v0.py ReachEnvV0 (walk_v0.py:49-79,104-186): reward shape, randomised joint reset, target centre (stand_target_centre)."""
        lo, hi = (float(x) for x in kw.get("joint_random_range", (0.0, 0.0)))
        if not hi > lo:
            raise NotImplementedError("stand task without joint randomisation: the reference then samples the target around the previous episode's last state")
        for i, v in enumerate(self.STAND_SHAPE):
            cfg.reach_shape[i] = v
        cfg.joint_random[0], cfg.joint_random[1] = lo, hi
        self.target_center = stand_target_centre(m, self.tip_names, init_qpos)

    def _setup_hold(self, m, cfg):
        """ObjHold constants (obj_hold_v0.py:46-62,126-145)."""
        from . import mjcf
        obj_body, sid, gid = m.name2id("body", "object"), m.name2id("site", "object"), m.name2id("geom", "object")
        pg = {v: k for k, v in self.prog_info["geom_model_ids"].items()}[gid]
        cfg.task_i[0], cfg.task_i[1] = self._dyn("object"), pg
        kin = mjcf.kinematics(m, m.qpos0)
        obj_init = kin["xpos"][obj_body] + kin["xmat"][obj_body] @ m.site_pos[sid]                    # object_init_pos (obj_hold_v0.py:52)
        goal = m.site_pos[m.name2id("site", "goal")]
        for i in range(3):
            cfg.task_d[i] = m.site_pos[sid][i]; cfg.task_d[3 + i] = obj_init[i]; cfg.task_d[6 + i] = goal[i]; cfg.task_d[9 + i] = m.geom_size[gid][i]

    # ---------------------------------------------------------------- gym-style API (batched)
    @property
    def horizon(self):
        return self.max_episode_steps

    def reset(self, seed=None, mask=None):
        """Reset all envs (mask None) or those whose mask entry is non-zero.  Passing `seed` also rewinds the per-env episode counters of
        the envs being reset (they key the Philox streams), so reset(seed=s) is reproducible like the reference's seeded np_random."""
        torch = self.torch
        if mask is not None:
            mask = torch.as_tensor(mask, device=self.device)
            if mask.numel() != self.num_envs:
                raise ValueError("reset mask must have %d entries, got %d" % (self.num_envs, mask.numel()))
            mask = (mask.reshape(-1) != 0).to(torch.uint8).contiguous()
        if seed is not None:
            self.seed_value = int(seed)
            if mask is None:
                self.t["episode_count"].zero_()
            else:
                self.t["episode_count"][mask.bool()] = 0
        self._reset_mask = mask          # keep alive until the launch has consumed it
        self.batch.reset(mask=mask, seed=self.seed_value, env_offset=self.env_offset, stream=self._stream())
        self._sync_obs()
        return self.t["obs"], {}

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def step(self, action):
        """action: float32 CUDA tensor [num_envs, nu] (values as the reference's action_space: [-1, 1])."""
        a = self.t["action"]
        if action.data_ptr() != a.data_ptr():
            if tuple(action.shape) != tuple(a.shape):
                raise ValueError("action must have shape %s, got %s" % (tuple(a.shape), tuple(action.shape)))
            a.copy_(action, non_blocking=True)
        self.batch.step(stream=self._stream())
        self._sync_obs()
        t = self.t
        return t["obs"], t["reward"], t["done"], t["truncated"], {"last_return": t["last_return"], "time": t["time"], "overflow": t["overflow"]}

    def step_host(self, action_cpu_pinned):
        """End-to-end call with HOST buffers: H2D action copy, step, D2H of reward/done (the e2e bench path)."""
        torch = self.torch
        self.t["action"].copy_(action_cpu_pinned, non_blocking=True)
        self.batch.step(stream=self._stream())
        self._sync_obs()
        if self._h_action is None:
            self._h_reward = torch.empty(self.num_envs, dtype=torch.float32, pin_memory=True)
            self._h_done = torch.empty(self.num_envs, dtype=torch.uint8, pin_memory=True)
            self._h_obs = torch.empty(self.num_envs, self.obs_dim, dtype=torch.float32, pin_memory=True)
            self._h_action = True
        self._h_obs.copy_(self.t["obs"], non_blocking=True)
        self._h_reward.copy_(self.t["reward"], non_blocking=True)
        self._h_done.copy_(self.t["done"], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self._h_obs, self._h_reward, self._h_done

    # ---------------------------------------------------------------- state access (get_env_state-like) and parity taps
    def set_state(self, qpos=None, qvel=None, act=None, target=None):
        torch = self.torch
        for name, v in (("qpos", qpos), ("qvel", qvel), ("act", act), ("target", target)):
            if v is not None:
                self.t[name][:, : np.shape(v)[-1]] = torch.as_tensor(np.asarray(v), dtype=torch.float64, device=self.device)
        self.t["qacc_warmstart"].zero_()

    STATE_KEYS = ("time", "qpos", "qvel", "act", "qacc_warmstart", "target", "step_count", "episode_count", "ep_return", "fatigue", "env_prm")

    def get_env_state(self, index=None):
        """Full state of the batch (or of env `index`) as numpy arrays: the reference's get_env_state (env_base.py:688-718: time, qpos, qvel, act)
        plus what this backend keeps per env besides mjData: the solver warm start, the task target (the reference stores it in site_pos /
        target_jnt_value), TimeLimit and episode counters, fatigue compartments (fatigue.py MA/MR/MF) and per-env model overrides."""
        self.torch.cuda.current_stream(self.device).synchronize()
        out = {}
        for k in self.STATE_KEYS:
            if k in self.t:
                v = self.t[k] if index is None else self.t[k][index]
                out[k] = v.detach().cpu().numpy().copy()
        return out

    def set_env_state(self, state, index=None):
        """Inverse of get_env_state (env_base.py:720-759); obs / reward / done are refreshed from the new state like the reference's forward()."""
        torch = self.torch
        for k, v in state.items():
            if k in self.t and k in self.STATE_KEYS and v is not None:
                dst = self.t[k] if index is None else self.t[k][index]
                dst.copy_(torch.as_tensor(np.asarray(v), device=self.device).to(dst.dtype).reshape(dst.shape))
        self.refresh_obs()

    def task_info(self):
        """`rwd_sparse` / `solved` of the current observations (the reference's info dict, env_base.py:585-616), derived lazily from obs."""
        from . import task_info
        m = self.mj_model
        return task_info.info_from_obs(self.task, self.t["obs_full"], m.nq, m.nv, m.na, pose_thd=float(self.cfg.pose_thd),
                                       ntip=len(getattr(self, "tip_names", ())) or None)

    def refresh_obs(self):
        """obs / reward / done of the current state (the reference's env.forward(), env_base.py:393-432)."""
        self.batch.observe(stream=self._stream())
        self._sync_obs()
        return self.t["obs"], self.t["reward"], self.t["done"]

    def examine_policy(self, policy, horizon=None, mode="exploration", seed=None, generator=None, keep_obs=True):
        """Batched MujocoEnv.examine_policy_new (env_base.py:853-969): one episode per env, observations / actions stay on the device;
        returns (Trace with one "Trial<k>" group per env, summary dict).  See myosuite_b200/rollout.py."""
        from . import rollout
        return rollout.examine_policy(self, policy, horizon=horizon, mode=mode, seed=seed, generator=generator, keep_obs=keep_obs)

    def forward_debug(self, ctrl, n_substeps=0):
        c = self.torch.as_tensor(np.asarray(ctrl), dtype=self.torch.float64, device=self.device).contiguous()
        self._dbg_ctrl = c
        self.batch.forward_debug(c, n_substeps, stream=self._stream())


class _DataView:
    """`env.mj_data`-like read access to the single env's state (numpy copies of the device rows)."""

    def __init__(self, vec):
        self._vec = vec

    def _row(self, k):
        self._vec.torch.cuda.current_stream(self._vec.device).synchronize()
        return self._vec.t[k][0].detach().cpu().numpy().copy()

    qpos = property(lambda self: self._row("qpos"))
    qvel = property(lambda self: self._row("qvel"))
    act = property(lambda self: self._row("act")[: self._vec.mj_model.na])
    time = property(lambda self: float(self._row("time")))


class MyoEnv:
    """Single-env facade with the reference's gym call shapes (numpy in / numpy out), n_env = 1 on the GPU.

    Mirrors what agents and the reference's own tests use on `env.unwrapped` (tests/test_envs.py:54-123): action_space, observation_space,
    obs_dict, rwd_dict, get_obs_dict, get_reward_dict, get_env_infos, get_env_state / set_env_state, seed / get_input_seed, dt, horizon,
    mj_model, mj_data, pickling (EzPickle semantics: the constructor arguments are pickled, plus the env state).  One device->host
    transfer per step: obs, reward, done, truncated and time travel in one packed float64 row."""

    metadata = {"render_modes": []}

    def __init__(self, env_id, seed=None, device=0, **kwargs):
        from . import gym_api
        self._ctor = (env_id, seed, device, dict(kwargs))
        self.vec = MyoVecEnv(env_id, 1, device=device, seed=0 if seed is None else seed, auto_reset=False, **kwargs)
        v = self.vec
        self.unwrapped = self
        self.env_id, self.mj_model, self.mj_data = env_id, v.mj_model, _DataView(v)
        self.dt, self.horizon, self.frame_skip = v.dt, v.max_episode_steps, v.frame_skip
        self.input_seed = seed
        m = v.mj_model
        self.action_space, self.observation_space = gym_api.make_spaces(m.nu, v.obs_dim, bool(v.kwargs.get("normalize_act", True)), m.actuator_ctrlrange)
        self._ntip = len(getattr(v, "tip_names", ()))
        self.obs_keys = list(getattr(v, "obs_keys", None) or [k for k, _ in gym_api.obs_layout(v.task, m.nq, m.nv, m.na, self._ntip)])
        self.rwd_keys_wt = dict(v.kwargs.get("weighted_reward_keys") or gym_api.DEFAULT_WEIGHTS[v.task])
        self.rwd_mode = "dense"
        self.obs_dict, self.rwd_dict, self.proprio_dict, self.visual_dict = {}, {}, {}, {}
        self._reseed = True
        self._task_cfg = self._make_task_cfg()
        self.reset()

    # ---- task constants for the host-side reward dict
    def _make_task_cfg(self):
        v, m, kw = self.vec, self.vec.mj_model, self.vec.kwargs
        cfg = {"pose_thd": float(v.cfg.pose_thd), "dt": v.dt, "ntip": self._ntip, "far_th": float(kw.get("far_th", 0.35))}
        if v.torso:
            cfg["pose_far_th"] = float(np.pi)
        if v.task == "walk":
            cfg.update(target_x_vel=kw.get("target_x_vel", 0.0), target_y_vel=kw.get("target_y_vel", 1.2), min_height=kw.get("min_height", 0.8), max_rot=kw.get("max_rot", 0.8),
                       target_rot=np.asarray(kw.get("target_rot") if kw.get("target_rot") is not None else m.key_qpos[0][3:7], dtype=np.float64))
            for j in ("hip_flexion_l", "hip_flexion_r", "hip_adduction_l", "hip_adduction_r", "hip_rotation_l", "hip_rotation_r"):
                cfg["q_" + j] = int(m.jnt_qposadr[m.name2id("joint", j)])
        return cfg

    # ---- seeding (env_base.py:119-123)
    def seed(self, seed=None):
        self.input_seed = seed
        self.vec.seed_value = 0 if seed is None else int(seed)
        self.action_space.seed(seed)
        self._reseed = True
        return [seed]

    def get_input_seed(self):
        return self.input_seed

    # ---- one packed device->host transfer
    def _fetch(self):
        torch, t = self.vec.torch, self.vec.t
        row = torch.cat([t["obs_full"][0].double(), t["reward"].double(), t["done"].double(), t["truncated"].double(), t["time"]]).cpu().numpy()
        n = self.vec.full_obs_dim
        full = row[:n].astype(np.float32)
        obs = full if self.vec._obs_cols is None else full[self.vec._obs_cols_np]          # obs vector = concatenation of obs_keys (obs_vec_dict.py:76-88)
        self._last = dict(obs=obs, obs_full=full, reward=float(row[n]), done=bool(row[n + 1]), truncated=bool(row[n + 2]), time=float(row[n + 3]))
        self.obs_dict = self.get_obs_dict()
        self.rwd_dict = self.get_reward_dict(self.obs_dict)
        return self._last

    def reset(self, seed=None, **kwargs):
        if seed is not None:
            self.seed(seed)
        self.vec.reset(seed=self.vec.seed_value if self._reseed else None)      # a (re)seed rewinds the Philox episode counter: reproducible resets
        self._reseed = False
        return self._fetch()["obs"], {}

    def step(self, a, **kwargs):
        torch = self.vec.torch
        act = torch.as_tensor(np.asarray(a, dtype=np.float32).reshape(1, -1), device=self.vec.device)
        self.vec.step(act)
        r = self._fetch()
        return r["obs"], r["reward"], r["done"], r["truncated"], self.get_env_infos()

    def forward(self, **kwargs):
        """env.forward() (env_base.py:393-432): recompute obs / reward / done of the current state."""
        self.vec.refresh_obs()
        r = self._fetch()
        return r["obs"], r["reward"], r["done"], self.get_env_infos()

    # ---- dicts (env_base.py:409-432, task get_obs_dict / get_reward_dict)
    def get_obs_dict(self, *sim_args):
        """obs_dict of the current observation.  (The reference signature takes (mj_model, mj_data); the state lives on the device here, so
        any arguments are ignored.)"""
        from . import gym_api
        m = self.mj_model
        return gym_api.obs_dict_from_vec(self.vec.task, self._last["obs_full"], np.array([self._last["time"]]), m.nq, m.nv, m.na, self._ntip)

    def get_reward_dict(self, obs_dict):
        from . import gym_api
        r = gym_api.reward_dict(self.vec.task, obs_dict, self.rwd_keys_wt, self._task_cfg)
        if float(np.squeeze(obs_dict["time"])) == self._last["time"]:
            r["dense"] = np.float64(self._last["reward"])        # the device's f64 reward (the host recomputation only sees the f32 observation)
        return r

    # ---- methods on paths and small accessors (env_base.py:434-459, 664-686, 763-826)
    @property
    def time(self):
        return self._last["time"]

    @property
    def id(self):
        return self.env_id

    def get_obs(self, **kwargs):
        return self.forward()[0]

    def _key_widths(self):
        from . import gym_api
        m = self.mj_model
        w = dict(gym_api.obs_layout(self.vec.task, m.nq, m.nv, m.na, self._ntip))
        return [(k, w[k]) for k in self.obs_keys]

    def obsvec2obsdict(self, obsvec):
        from . import gym_api
        return gym_api.obsvec2obsdict(obsvec, self._key_widths())

    def compute_path_rewards(self, paths):
        from . import gym_api
        return gym_api.compute_path_rewards(self.vec.task, paths, self._key_widths(), self.rwd_keys_wt, self._task_cfg, self.rwd_mode)

    def truncate_paths(self, paths):
        from . import gym_api
        return gym_api.truncate_paths(paths)

    def evaluate_success(self, paths, logger=None, successful_steps=5):
        from . import gym_api
        return gym_api.evaluate_success(paths, self.horizon, logger, successful_steps)

    def get_proprioception(self, obs_dict=None):
        """env_base.py get_proprioception: (None, None, None) when no proprio_keys are configured (the default of the hot-path envs)."""
        return None, None, None

    def get_exteroception(self, **kwargs):
        return {}

    def get_env_infos(self):
        """env_base.py:585-616."""
        return {"time": self._last["time"], "rwd_dense": self._last["reward"], "rwd_sparse": float(np.squeeze(self.rwd_dict["sparse"])),
                "solved": bool(np.squeeze(self.rwd_dict["solved"])), "done": self._last["done"], "obs_dict": self.obs_dict, "visual_dict": {},
                "proprio_dict": self.proprio_dict, "rwd_dict": self.rwd_dict, "state": self.get_env_state()}

    # ---- state (env_base.py:688-759)
    def get_env_state(self):
        return self.vec.get_env_state(index=0)

    def set_env_state(self, state_dict):
        self.vec.set_env_state(state_dict, index=0)
        self._fetch()

    # ---- pickling: constructor arguments (EzPickle) + the current state
    def __getstate__(self):
        return {"ctor": self._ctor, "input_seed": self.input_seed, "state": self.get_env_state()}

    def __setstate__(self, d):
        env_id, seed, device, kwargs = d["ctor"]
        self.__init__(env_id, seed=seed, device=device, **kwargs)
        self.input_seed = d["input_seed"]
        self.set_env_state(d["state"])

    def examine_policy_new(self, policy, horizon=1000, num_episodes=1, mode="exploration", render=None, **kwargs):
        """MujocoEnv.examine_policy_new (env_base.py:853-969) for the single env: `policy.get_action(obs)` as in mjrl, a Trace with one
        "Trial<k>" group per episode (time, observations, actions, rewards, env_infos, done; NaN action in the last row).  No rendering."""
        from .rollout import Trace
        trace = Trace(str(self.env_id) + "_rollouts")
        for ep in range(num_episodes):
            g = "Trial" + str(ep); trace.create_group(g)
            self.reset()
            obs, rwd, done, env_info = self.forward()
            t = 0
            while t < horizon and done is False:
                act = policy.get_action(obs)[0] if mode == "exploration" else policy.get_action(obs)[1]["evaluation"]
                trace.append_datums(g, dict(time=self._last["time"], observations=obs, actions=np.asarray(act).copy(), rewards=rwd, env_infos=env_info, done=done))
                obs, rwd, done, trunc, env_info = self.step(act)
                t += 1
            trace.append_datums(g, dict(time=self._last["time"], observations=obs, actions=np.nan * np.ones(self.action_space.shape), rewards=rwd, env_infos=env_info, done=done))
        trace.stack()
        return trace

    def close(self):
        pass


def register_gym():
    """Register every implemented id with gymnasium (or gym) when one of them is installed: gymnasium.make("myoHandPoseRandom-v0") then
    returns a MyoEnv (wrapped in the library's TimeLimit / checker wrappers).  Returns the list of registered ids ([] without a gym)."""
    for mod in ("gymnasium", "gym"):
        try:
            g = __import__(mod)
            break
        except Exception:
            g = None
    if g is None:
        return []
    done = []
    for eid in registered_ids():
        try:
            steps, _, entry = env_spec(eid)
            if not any(entry.endswith(x) for x in ("pose_v0:PoseEnvV0", "walk_v0:WalkEnvV0", "reach_v0:ReachEnvV0", "torso_v0:TorsoEnvV0", "walk_v0:ReachEnvV0")) and "obj_hold_v0:ObjHold" not in entry:
                continue
            g.register(id=eid, entry_point="myosuite_b200.vec_env:MyoEnv", max_episode_steps=steps, kwargs={"env_id": eid})
            done.append(eid)
        except Exception:
            pass
    return done


def make(env_id, num_envs=None, **kwargs):
    """``make(id)`` -> single env (reference call shape); ``make(id, num_envs=N)`` -> batched MyoVecEnv."""
    if num_envs is None:
        return MyoEnv(env_id, **kwargs)
    return MyoVecEnv(env_id, num_envs, **kwargs)
