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

from . import abi, assets, blob, program, tasks

_HERE = os.path.dirname(os.path.abspath(__file__))
_REG = None


def _check_f64(name, x, shape, device):
    """Raise ValueError unless x is a contiguous float64 tensor of `shape` on `device` (the analysis calls' input tensors)."""
    import torch
    if (not isinstance(x, torch.Tensor) or x.dtype != torch.float64 or x.device != device or tuple(x.shape) != tuple(shape)
            or not x.is_contiguous()):
        raise ValueError("%s must be a contiguous float64 tensor of shape %s on %s, got %s" % (name, tuple(shape), device, (
            type(x).__name__, getattr(x, "dtype", None), getattr(x, "device", None), tuple(getattr(x, "shape", ())),
            x.is_contiguous() if isinstance(x, torch.Tensor) else None)))


def _check_fields(kind, fields, available):
    """The requested output fields as a tuple; KeyError names those not in `available`."""
    fields = tuple(fields)
    bad = [f for f in fields if f not in available]
    if bad:
        raise KeyError("unknown %s fields %s (available: %s)" % (kind, bad, list(available)))
    return fields


def _output(device, lead, trailing, size, int32=False):
    """An output tensor of shape lead + trailing, with the model-size names in `trailing` looked up in `size`, filled with NaN (float64)
    or -1 (int32) so that an entry the launch does not write stands out."""
    import torch
    shape = tuple(lead) + tuple(size[x] if isinstance(x, str) else x for x in trailing)
    return torch.full(shape, -1, dtype=torch.int32, device=device) if int32 else torch.full(shape, float("nan"), dtype=torch.float64, device=device)


def _outputs(device, fields, lead, shapes, size):
    """Fresh output tensors {field: tensor} of the analysis calls: overflow the [n] int32 zero tensor (lead = (n, ...)), every other field
    _output(device, lead, shapes[field], size), int32 for niter and converged."""
    import torch
    return {f: torch.zeros(lead[0], dtype=torch.int32, device=device) if f == "overflow"
            else _output(device, lead, shapes[f], size, f in ("niter", "converged")) for f in fields}


def _flags(constraints, discrete):
    """The MYO_INV_* flags of the constraints / discrete arguments (mjDSBL_CONSTRAINT, mjENBL_INVDISCRETE)."""
    return (0 if constraints else abi.INV_NOCONSTRAINT) | (abi.INV_DISCRETE if discrete else 0)


def _check_substeps(substeps):
    """substeps as an int, ValueError unless >= 1."""
    substeps = int(substeps)
    if substeps < 1:
        raise ValueError("substeps must be >= 1, got %d" % substeps)
    return substeps


def _check_solver(call, params, max_iter, tol):
    """params (a ctypes struct with max_iter and tol), ValueError unless it holds max_iter >= 0 and a finite tol >= 0; the message quotes
    the caller's max_iter and tol."""
    if not (params.max_iter >= 0 and params.tol >= 0 and np.isfinite(params.tol)):
        raise ValueError("%s needs max_iter >= 0 and a finite tol >= 0, got max_iter %r, tol %r" % (call, max_iter, tol))
    return params


def _vector(name, x, width, device, positive=True):
    """A per-dof or per-muscle parameter: a number, array or tensor of any numeric dtype, device and layout, of shape () or (width,), as a
    contiguous float64 [width] tensor on `device`; ValueError unless every entry is finite and > 0 (>= 0 when not `positive`)."""
    import torch
    v = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    if v.dtype.kind not in "biuf" or v.shape not in ((), (width,)):
        raise ValueError("%s must be a scalar or of shape (%d,), got %s %s" % (name, width, v.dtype, v.shape))
    v = np.broadcast_to(v.astype(np.float64), (width,))
    if not np.all(np.isfinite(v) & ((v > 0) if positive else (v >= 0))):
        raise ValueError("%s must be finite and %s" % (name, "> 0" if positive else ">= 0"))
    return torch.as_tensor(v.copy(), device=device)


def _state_width(m, time=True):
    """initial_state key -> trailing shape after [n] for model m (_initial_state's `width`); time only for the calls that take it."""
    width = dict(qpos=(m.nq,), qvel=(m.nv,), act=(m.na,), qacc_warmstart=(m.nv,))
    if time:
        width["time"] = ()
    return width


def _row0(out):
    """Row 0 of every tensor of `out` {field: tensor [n, ...]} as numpy, in one device-to-host copy: each field keeps its trailing shape and
    its dtype (int32, else float64), and a field with one value per env becomes a Python int or float."""
    import torch
    if not out:
        return {}
    flat = torch.cat([x[0].reshape(-1).double() for x in out.values()]).cpu().numpy()
    res, o = {}, 0
    for k, x in out.items():
        a = flat[o:o + x[0].numel()].reshape(tuple(x.shape[1:])); o += x[0].numel()
        a = a.astype(np.int32) if x.dtype == torch.int32 else a
        res[k] = a.item() if a.ndim == 0 else a
    return res


def _initial_state(initial_state, width, n, device):
    """The start-state fields (abi.ROLLOUT_STATE) of an `initial_state` dict: KeyError for a key not in `width` (key -> trailing shape
    after [n]), ValueError for a tensor that is not a contiguous float64 [n, width] on `device`; a None value is left out."""
    bufs = {}
    for k, v in (initial_state or {}).items():
        if k not in width:
            raise KeyError("unknown initial_state key %r (available: %s)" % (k, list(width)))
        if v is not None:
            _check_f64("initial_state[%r]" % k, v, (n,) + width[k], device)
            bufs[abi.ROLLOUT_STATE[k]] = v
    return bufs


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


def condition_model(m, muscle_condition):
    """The model a batch of `muscle_condition` simulates: sarcopenia halves the peak force of every muscle in a copy of m
    (base_v0.py:62-67: gainprm[:,2] *= 0.5, biasprm untouched); fatigue and reafferentation act on ctrl and keep m itself."""
    if muscle_condition == "sarcopenia":
        import copy
        m = copy.deepcopy(m)
        m.actuator_gainprm[:, 2] *= 0.5
    return m
stand_target_centre = tasks.stand_target_centre          # (importable from here as before)


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
        self.mj_model = m = model if model is not None else assets.load(_MODEL_OF_XML[kw["model_path"]])
        self.muscle_condition = kw.get("muscle_condition", "")
        self.mj_model = m = condition_model(m, self.muscle_condition)
        prog, self.prog_info = program.build_program(m)
        self.prog = prog
        self.I, self.D = blob.pack(m, prog)
        # everything task-specific is computed on the host by tasks.configure; what follows allocates and binds it
        c = tasks.configure(entry, m, self.prog_info, kw, self.max_episode_steps, auto_reset)
        self.task, self.torso, self.hold_random, self.cfg = c.task, c.torso, c.hold_random, c.cfg
        self.frame_skip, self.dt, self.n_frames = c.frame_skip, c.dt, c.n_frames
        self.init_qpos, self.init_qvel, self.tip_names, self.target_center = c.init_qpos, c.init_qvel, c.tip_names, c.target_center
        self.fatigue_reset_vec, self.reward_cfg = c.fatigue_reset_vec, c.reward_cfg
        # row_storage: "p48" (product: contact Jacobian rows held as the upper 48 bits of the f64 value -- 36 mantissa bits -- in shared memory,
        # 14 env-warps per SM on the hand) or "f64" (verification build of the same source, abi.lib("f64rows"): plain doubles, fewer warps)
        self.row_storage = kw.get("row_storage", "p48")
        if self.row_storage not in ("p48", "f64"):
            raise ValueError("row_storage must be 'p48' or 'f64'")
        self.dev_model = abi.DeviceModel(self.I, self.D, variant="f64rows" if self.row_storage == "f64" else None)
        cfg = self.cfg
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
        lay = c.layout
        self.obs_keys = [k_ for k_, _ in lay]
        self._obs_cols = None
        if kw.get("obs_keys") is not None and lay:
            keys = list(kw["obs_keys"])
            if m.na > 0 and "act" not in keys:
                keys.append("act")
            off, o = {}, 0
            for k_, w_ in lay:
                off[k_] = (o, w_); o += w_
            missing = [k_ for k_ in keys if k_ not in off]
            if missing:
                raise KeyError("obs_keys not available from this task's obs_dict: %s (available: %s)" % (missing, self.obs_keys))
            if keys != self.obs_keys:
                cols = np.concatenate([np.arange(off[k_][0], off[k_][0] + off[k_][1]) for k_ in keys])
                self._obs_cols, self._obs_cols_np = torch.as_tensor(cols, dtype=torch.int64, device=self.device), cols
                self.obs_dim = int(len(cols))
            self.obs_keys = keys
        t = dict(action=z(n, m.nu, dtype=f32), qpos=z(n, m.nq), qvel=z(n, m.nv), act=z(n, max(m.na, 1)), qacc_warmstart=z(n, m.nv),
                 time=z(n), target=z(n, m.nq), step_count=z(n, dtype=torch.int32), episode_count=z(n, dtype=torch.int64),
                 obs=z(n, self.full_obs_dim, dtype=f32), reward=z(n, dtype=f32), done=z(n, dtype=torch.uint8), truncated=z(n, dtype=torch.uint8),
                 ep_return=z(n, dtype=f32), last_return=z(n, dtype=f32), overflow=z(n, dtype=torch.int32))
        t["qpos"][:] = torch.as_tensor(m.qpos0, device=dv)
        t["target_range"] = torch.as_tensor(c.target_range, device=dv).contiguous()
        t["init_qpos"] = torch.as_tensor(self.init_qpos, device=dv).contiguous()
        t["init_qvel"] = torch.as_tensor(self.init_qvel, device=dv).contiguous()
        if c.env_prm is not None:
            t["env_prm"] = z(n, 8)
            t["env_prm"][:, :6] = torch.as_tensor(c.env_prm, device=dv)
        if cfg.muscle_condition == abi.COND_FATIGUE:
            t["fatigue"] = z(n, 3, m.nu)
            t["fatigue"][:, 1, :] = 1.0
            if self.fatigue_reset_vec is not None:
                t["fatigue_reset_vec"] = torch.as_tensor(self.fatigue_reset_vec, device=dv).contiguous()
        if cfg.task != abi.TASK_NONE:          # the observation each ended episode ended in (written by the step kernel; NaN until an env first ends)
            t["final_obs"] = torch.full((n, self.full_obs_dim), float("nan"), dtype=f32, device=dv)
        if taps:
            t.update(tap_qacc=z(n, m.nv), tap_actuator_force=z(n, m.nu), tap_ten_length=z(n, m.nu), tap_qfrc_smooth=z(n, m.nv),
                     tap_ncon=z(n, 4, dtype=torch.int32), tap_contact_pair=z(n, max(self.dims.maxcon, 1), dtype=torch.int32),
                     tap_contact_dist=z(n, max(self.dims.maxcon, 1)), tap_moment=z(n, max(self.dims.reserved[0], 1)), tap_qM=z(n, m.nM),
                     tap_phase_cycles=z(n, 20, dtype=torch.int64))
        self.t = t
        self.batch.bind(**t)
        t["obs_full"] = t["obs"]                                  # what the kernel writes (bound above); t["obs"] is what callers see
        if "final_obs" in t:
            t["final_obs_full"] = t["final_obs"]                  # likewise for final_obs
        if self._obs_cols is not None:
            t["obs"] = z(n, self.obs_dim, dtype=f32)
            t["final_obs"] = torch.full((n, self.obs_dim), float("nan"), dtype=f32, device=dv)
        self._h_action = None
        # mjData readout (data()): buffers allocated on first request; site_source places the sites the task moves per episode
        self._data, self._inv, self.state_version = {}, {}, 0         # (inverse(): its output tensors, likewise)
        src = tasks.site_sources(self.task, m, kw, self.tip_names)
        self._site_source = None if src is None else torch.as_tensor(src, device=dv).contiguous()

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
        self.state_version += 1
        self.batch.reset(mask=mask, seed=self.seed_value, env_offset=self.env_offset, stream=self._stream())
        self._sync_obs()
        return self.t["obs"], {}

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def step(self, action):
        """action: float32 CUDA tensor [num_envs, nu] (values as the reference's action_space: [-1, 1]).

        info["final_obs"] [num_envs, obs_dim] (the layout of obs) holds the observation of the state each episode that ended on this step
        ended in: with auto-reset, obs already belongs to the next episode.  A row is valid exactly where done | truncated of the same
        step is set; other rows keep what an earlier step wrote (NaN before an env first ends).  The tensor is reused by every step.
        None for the physics-only batch."""
        a = self.t["action"]
        if action.data_ptr() != a.data_ptr():
            if tuple(action.shape) != tuple(a.shape):
                raise ValueError("action must have shape %s, got %s" % (tuple(a.shape), tuple(action.shape)))
            a.copy_(action, non_blocking=True)
        self.batch.step(stream=self._stream())
        self.state_version += 1
        self._sync_obs()
        t = self.t
        if self._obs_cols is not None:
            self.torch.index_select(t["final_obs_full"], 1, self._obs_cols, out=t["final_obs"])
        return t["obs"], t["reward"], t["done"], t["truncated"], {"last_return": t["last_return"], "time": t["time"], "overflow": t["overflow"],
                                                                  "final_obs": t.get("final_obs")}

    def step_host(self, action_cpu_pinned):
        """End-to-end call with HOST buffers: H2D action copy, step, D2H of reward/done (the e2e bench path)."""
        torch = self.torch
        self.t["action"].copy_(action_cpu_pinned, non_blocking=True)
        self.batch.step(stream=self._stream())
        self.state_version += 1
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
        self.state_version += 1

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
        m = self.mj_model
        return tasks.info_from_obs(self.task, self.t["obs_full"], m.nq, m.nv, m.na, pose_thd=float(self.cfg.pose_thd), ntip=len(self.tip_names) or None)

    def final_task_info(self):
        """`rwd_sparse` / `solved` of the states the episodes ended in (task_info of info["final_obs"]): valid in the rows where done |
        truncated of the last step is set.  None for tasks without a distance-type success signal (walk), like task_info."""
        if "final_obs_full" not in self.t:
            return None
        m = self.mj_model
        return tasks.info_from_obs(self.task, self.t["final_obs_full"], m.nq, m.nv, m.na, pose_thd=float(self.cfg.pose_thd), ntip=len(self.tip_names) or None)

    def refresh_obs(self):
        """obs / reward / done of the current state (the reference's env.forward(), env_base.py:393-432)."""
        self.batch.observe(stream=self._stream())
        self.state_version += 1
        self._sync_obs()
        return self.t["obs"], self.t["reward"], self.t["done"]

    DATA_FIELDS = tuple(k for k in abi.DATA_FIELDS if k != "site_source")

    def data(self, *fields):
        """mjData of every env after mj_forward at its current state (the reference's env.unwrapped.mj_data after reset() / step()):
        {field: tensor [num_envs, ...]} for the requested fields of DATA_FIELDS (all when none is named), in MuJoCo ids and order.
        One launch computes only what the deepest requested group needs (pose < actuation < dynamics; myo_batch_data).  The tensors
        are allocated on first request (NaN / -1 until first written) and reused: a result is valid until the next state change.
        ctrl is the last step's ctrl (zeros before the first step); after an auto-reset the values describe the new episode's state."""
        fields = _check_fields("mjData", tuple(fields) or self.DATA_FIELDS, self.DATA_FIELDS)
        m, n = self.mj_model, self.num_envs
        size = dict(nbody=m.nbody, nsite=m.nsite, nu=m.nu, nv=m.nv, maxcon=self.dims.maxcon)
        for f in fields:
            if f not in self._data:
                _, dt, shape = abi.DATA_SHAPES[f]
                self._data[f] = _output(self.device, (n,), shape, size, dt == "i32")
        bufs = {f: self._data[f] for f in fields}
        if "site_xpos" in bufs:
            bufs["site_source"] = self._site_source
        self.batch.data(stream=self._stream(), **bufs)
        return {f: self._data[f] for f in fields}

    INVERSE_FIELDS = tuple(abi.INVERSE_SHAPES)

    def inverse(self, qacc, constraints=True, discrete=False, fields=("qfrc_inverse",)):
        """MuJoCo's mj_inverse for every env at its current (qpos, qvel): the generalized force that produces the acceleration `qacc`
        (float64 CUDA tensor [num_envs, nv] on this batch's device), {field: tensor [num_envs, ...]} for the requested INVERSE_FIELDS:
        qfrc_inverse, qfrc_constraint, contact_force [maxcon, 6] (mj_contactForce) and the dense actuator_moment [nu, nv].
        constraints=False is mjDSBL_CONSTRAINT (no contacts, limits or equalities); discrete=True reads qacc as (qvel' - qvel) / h of one
        Euler substep (mjENBL_INVDISCRETE).  act, ctrl and the warm start do not enter.  One launch; the tensors are allocated on first
        request and reused, like data()'s.  Not a state change."""
        torch = self.torch
        fields = _check_fields("inverse", fields, self.INVERSE_FIELDS)
        m, n = self.mj_model, self.num_envs
        if not isinstance(qacc, torch.Tensor) or qacc.dtype != torch.float64 or qacc.device != self.device or tuple(qacc.shape) != (n, m.nv):
            raise ValueError("qacc must be a float64 tensor of shape (%d, %d) on %s, got %s" % (
                n, m.nv, self.device, (type(qacc).__name__, getattr(qacc, "dtype", None), getattr(qacc, "device", None), tuple(getattr(qacc, "shape", ())))))
        size = dict(nu=m.nu, nv=m.nv, maxcon=self.dims.maxcon)
        outs = set(fields) | {"qfrc_inverse"}
        for f in outs:
            if f not in self._inv:
                self._inv[f] = _output(self.device, (n,), abi.INVERSE_SHAPES[f], size)
        self.batch.inverse(stream=self._stream(), flags=_flags(constraints, discrete), qacc=qacc.contiguous(), **{f: self._inv[f] for f in outs})
        return {f: self._inv[f] for f in fields}

    ROLLOUT_FIELDS = tuple(abi.ROLLOUT_SHAPES) + ("overflow",)

    def rollout(self, ctrl, qfrc_applied=None, substeps=1, initial_state=None, fields=("qpos", "qvel", "act", "qacc", "time")):
        """MuJoCo's mj_step for every env: nstep intervals of `substeps` mj_steps each, with the MuJoCo ctrl row ctrl[:, t] held for the
        substeps of interval t.  ctrl is mjData.ctrl, NOT the env's action: it is clipped to ctrlrange as mj_step does, and neither the
        action sigmoid (normalize_act), fatigue nor reafferentation is applied; a caller who starts from actions applies the remap itself
        (1 / (1 + exp(-5 (a - 0.5))) when normalize_act is set).  qfrc_applied [num_envs, nstep, nv] (mjData.qfrc_applied, None = zero)
        is added to qfrc_smooth.  Both are float64 CUDA tensors on this batch's device, contiguous, ctrl [num_envs, nstep, nu].
        initial_state: {"qpos", "qvel", "act", "qacc_warmstart", "time": float64 tensor [num_envs, width] ([num_envs] for time)}; a key
        left out is taken from the env's current state.  Returns {field: tensor [num_envs, nstep, ...]} of ROLLOUT_FIELDS, mjData after
        the last mj_step of each interval: qpos, qvel, act, qacc (also the next warm start: a rollout resumes exactly from row t with
        initial_state = its qpos, qvel, act, time and qacc as qacc_warmstart), time; overflow [num_envs] int32 is set where a substep
        dropped contacts.  The tensors are allocated per call.  Per-env overrides (env_prm) apply; the task layer, counters and auto-reset
        do not run, and the env's own state and episode are left as they were: not a state change.  One launch per interval."""
        torch = self.torch
        fields = _check_fields("rollout", fields, self.ROLLOUT_FIELDS)
        m, n = self.mj_model, self.num_envs
        substeps = _check_substeps(substeps)
        nstep = int(ctrl.shape[1]) if isinstance(ctrl, torch.Tensor) and ctrl.dim() == 3 else 0
        if nstep < 1:
            raise ValueError("ctrl must be a float64 tensor [num_envs, nstep >= 1, nu], got %s" % (tuple(getattr(ctrl, "shape", ())),))
        _check_f64("ctrl", ctrl, (n, nstep, m.nu), self.device)
        bufs = {"ctrl": ctrl}
        if qfrc_applied is not None:
            _check_f64("qfrc_applied", qfrc_applied, (n, nstep, m.nv), self.device)
            bufs["qfrc_applied"] = qfrc_applied
        bufs.update(_initial_state(initial_state, _state_width(m), n, self.device))
        out = _outputs(self.device, fields, (n, nstep), abi.ROLLOUT_SHAPES, dict(nq=m.nq, nv=m.nv, na=m.na))
        self.batch.rollout(nstep, substeps, stream=self._stream(), **bufs, **out)
        return out

    IK_FIELDS = tuple(abi.IK_SHAPES)
    # defaults of ik(): tol in metres and radians; at these, targets from forward kinematics of random in-range configurations are
    # reached from init_qpos at the rates DESIGN.md section 2 lists
    IK_DEFAULTS = dict(max_iter=200, tol=1e-6, damping=1e-3, max_step=0.5, posture=0.0, eq_weight=1.0)

    def ik(self, sites, target_pos, target_quat=None, qpos_init=None, qpos_ref=None, dofs=None, site_weight=None,
           max_iter=IK_DEFAULTS["max_iter"], tol=IK_DEFAULTS["tol"], damping=IK_DEFAULTS["damping"], max_step=IK_DEFAULTS["max_step"],
           posture=IK_DEFAULTS["posture"], eq_weight=IK_DEFAULTS["eq_weight"], fields=("qpos", "niter", "converged", "err")):
        """Damped least-squares inverse kinematics of every env (myo_batch_ik; include/myo_b200.h states the iteration): sites (names or
        ids, 1..16 of them) toward target_pos [num_envs, ns, 3] and, when given, target_quat [num_envs, ns, 4] (w x y z), from qpos_init
        [num_envs, nq] (None: the current qpos), with the posture term pulling hinge and slide joints toward qpos_ref [num_envs, nq] (None:
        the start) at weight `posture`, the joint equalities at weight eq_weight and per-site (position, orientation) weights site_weight
        [ns, 2].  dofs: joint names or a bool mask [nv] of the dofs that may move (None: all).  Joint limits hold by clamping after each
        step.  Tensors are contiguous float64 CUDA tensors on this batch's device.  Returns {field: tensor [num_envs, ...]} of IK_FIELDS:
        qpos, niter, converged (int32), err [ns, 2] (|position error|, |rotation error|), site_xpos [ns, 3], site_xmat [ns, 9],
        jacp / jacr [ns, 3, nv], all at the returned qpos; allocated per call.  One launch; not a state change (adopt a solution with
        set_state(qpos=...)).  A trajectory of T frames is one call on a batch of T envs."""
        torch, m, n = self.torch, self.mj_model, self.num_envs
        fields = _check_fields("ik", fields, self.IK_FIELDS)
        sid = [m.name2id("site", x) if isinstance(x, str) else int(x) for x in ([sites] if isinstance(sites, (str, int)) else sites)]
        ns = len(sid)
        if not 1 <= ns <= abi.IK_MAXSITE or any(not 0 <= x < m.nsite for x in sid):
            raise ValueError("sites must be 1..%d site names or ids in [0, %d), got %s" % (abi.IK_MAXSITE, m.nsite, sites))
        _check_f64("target_pos", target_pos, (n, ns, 3), self.device)
        bufs = {"target_pos": target_pos}
        for name, x, shape in (("target_quat", target_quat, (n, ns, 4)), ("qpos0", qpos_init, (n, m.nq)), ("qpos_ref", qpos_ref, (n, m.nq)),
                               ("site_weight", site_weight, (ns, 2))):
            if x is not None:
                _check_f64("qpos_init" if name == "qpos0" else name, x, shape, self.device)
                bufs[name] = x
        if dofs is not None:
            if isinstance(dofs, torch.Tensor) or isinstance(dofs, np.ndarray):
                mask = np.asarray(dofs.cpu() if isinstance(dofs, torch.Tensor) else dofs)
                if mask.dtype != np.bool_ or mask.shape != (m.nv,):
                    raise ValueError("dofs must be joint names or a bool mask of shape (%d,), got %s %s" % (m.nv, mask.dtype, mask.shape))
            else:
                mask = np.zeros(m.nv, bool)
                for j in [m.name2id("joint", x) for x in ([dofs] if isinstance(dofs, str) else dofs)]:
                    nd = {0: 6, 1: 3}.get(int(m.jnt_type[j]), 1)
                    mask[m.jnt_dofadr[j]:m.jnt_dofadr[j] + nd] = True
            bufs["dof_mask"] = torch.as_tensor(mask.astype(np.uint8), device=self.device)
        params = abi.MyoIkParams(nsite=ns, max_iter=int(max_iter), tol=float(tol), damping=float(damping), max_step=float(max_step),
                                 posture_weight=float(posture), eq_weight=float(eq_weight))
        if not (params.max_iter >= 0 and params.tol >= 0 and params.damping > 0 and params.max_step > 0 and params.posture_weight >= 0
                and params.eq_weight >= 0 and np.all(np.isfinite([tol, damping, max_step, posture, eq_weight]))):
            raise ValueError("ik needs max_iter >= 0, tol >= 0, damping > 0, max_step > 0, posture >= 0 and eq_weight >= 0, all finite")
        bufs["site_id"] = torch.as_tensor(np.asarray(sid, np.int32), device=self.device)
        bufs["site_quat"] = torch.as_tensor(np.ascontiguousarray(m.site_quat[sid], dtype=np.float64), device=self.device)
        out = _outputs(self.device, set(fields) | {"qpos"}, (n,), abi.IK_SHAPES, dict(nq=m.nq, nv=m.nv, ns=ns))
        self.batch.ik(params, stream=self._stream(), **bufs, **out)
        return {f: out[f] for f in fields}

    def jac_site(self, sites, qpos=None):
        """mj_jacSite of every env: (jacp, jacr [num_envs, ns, 3, nv], site_xpos [num_envs, ns, 3], site_xmat [num_envs, ns, 9]) at qpos
        [num_envs, nq] (None: the current qpos).  The same launch as ik() with max_iter = 0."""
        n = self.num_envs
        ns = 1 if isinstance(sites, (str, int)) else len(sites)
        r = self.ik(sites, self.torch.zeros((n, ns, 3), dtype=self.torch.float64, device=self.device), qpos_init=qpos, max_iter=0,
                    fields=("jacp", "jacr", "site_xpos", "site_xmat"))
        return r["jacp"], r["jacr"], r["site_xpos"], r["site_xmat"]

    FD_FIELDS = ("A", "B", "overflow")

    def transition_fd(self, ctrl, eps=1e-6, centered=False, substeps=1, qfrc_applied=None, initial_state=None, fields=("A", "B")):
        """MuJoCo's mjd_transitionFD for every env, over one interval of `substeps` mj_steps with ctrl held (substeps = 1 is
        mjd_transitionFD itself; substeps = frame_skip linearises the env's control interval, whose B is not zero in qpos / qvel since ctrl
        enters the muscles only through act_dot).  x' ~ x'0 + A dx + B du with x = [dq (nv, tangent space), qvel (nv), act (na)], nx =
        2 nv + na: A [num_envs, nx, nx], B [num_envs, nx, nu], A[i][j] = d x'_i / d x_j.  Forward differences, or centred ones with
        centered=True; ctrl columns at a ctrlrange end take the one side that stays in range (mjd_stepFD's rule, include/myo_b200.h).
        ctrl [num_envs, nu] is mjData.ctrl (as rollout(): no action remap), qfrc_applied [num_envs, nv] or None, both float64 CUDA
        tensors on this batch's device, contiguous.  initial_state: {"qpos", "qvel", "act", "qacc_warmstart": float64 tensor
        [num_envs, width]}; a key left out is taken from the env's current state.  The nominal x'0 is exactly rollout(ctrl[:, None],
        substeps=substeps) from the same start, and every perturbed interval starts with the start's warm start.
        Returns {field: tensor} of FD_FIELDS (overflow [num_envs] int32: set where a substep of the nominal or a perturbed interval
        dropped contacts).  The outputs are allocated per call: A takes num_envs * nx^2 * 8 bytes (359 MB for 2048 legs envs, 320 MB for
        661 torso envs), B num_envs * nx * nu * 8.  Not a state change: the call advances nothing and writes no env buffer.  With the
        iterative solver each column carries solver noise of order solver_tolerance / eps, as in MuJoCo; MyoVecEnv(...,
        solver_tolerance=...) tightens it.  Two launches (the nominal interval, then one warp per (env, column))."""
        fields = _check_fields("transition_fd", fields, self.FD_FIELDS)
        if "A" not in fields and "B" not in fields:
            raise ValueError("transition_fd needs at least one of the fields A and B")
        m, n = self.mj_model, self.num_envs
        substeps, eps = _check_substeps(substeps), float(eps)
        if not (np.isfinite(eps) and eps > 0):
            raise ValueError("eps must be finite and > 0, got %r" % eps)
        if centered not in (0, 1, False, True):
            raise ValueError("centered must be a bool, got %r" % (centered,))
        _check_f64("ctrl", ctrl, (n, m.nu), self.device)
        bufs = {"ctrl": ctrl}
        if qfrc_applied is not None:
            _check_f64("qfrc_applied", qfrc_applied, (n, m.nv), self.device)
            bufs["qfrc_applied"] = qfrc_applied
        bufs.update(_initial_state(initial_state, _state_width(m, time=False), n, self.device))
        out = _outputs(self.device, fields, (n,), dict(A=("nx", "nx"), B=("nx", "nu")), dict(nx=2 * m.nv + m.na, nu=m.nu))
        params = abi.MyoFdParams(eps=eps, centered=int(bool(centered)), substeps=substeps)
        self.batch.transition_fd(params, stream=self._stream(), **bufs, **out)
        return out

    INVERSE_FD_FIELDS = tuple(abi.INVERSE_FD_SHAPES) + ("overflow",)

    def inverse_fd(self, qacc, eps=1e-6, actuation=False, constraints=True, discrete=False, initial_state=None, fields=("DfDq", "DfDv", "DfDa")):
        """MuJoCo's mjd_inverseFD for every env (myo_batch_inverse_fd; include/myo_b200.h states it in full): forward-difference
        Jacobians of f = qfrc_inverse, or of qfrc_inverse - qfrc_actuator with actuation=True (flg_actuation: the generalized force the
        muscles at the current act do not supply), in qpos (through mj_integratePos), qvel and qacc, at the start state and the acceleration
        qacc [num_envs, nv] (a contiguous float64 CUDA tensor on this batch's device).  constraints and discrete as inverse()'s.
        initial_state: {"qpos", "qvel", "act": float64 tensor [num_envs, width]}; a key left out is taken from the env's current state.
        Returns {field: tensor [num_envs, ...]} of INVERSE_FD_FIELDS: DfDq, DfDv, DfDa [nv, nv] in MuJoCo's layout, DfDq[e, i, j] =
        d f_j / d q_i (transposed with respect to transition_fd()'s A), qfrc_inverse [nv] (the nominal f) and overflow [num_envs] int32 (set
        where the nominal or a perturbed pass dropped contacts).  Allocated per call: each block takes num_envs * nv^2 * 8 bytes.  Two
        launches (the nominal, then one warp per (env, column)); not a state change."""
        fields = _check_fields("inverse_fd", fields, self.INVERSE_FD_FIELDS)
        if not {"DfDq", "DfDv", "DfDa"} & set(fields):
            raise ValueError("inverse_fd needs at least one of the fields DfDq, DfDv and DfDa")
        m, n = self.mj_model, self.num_envs
        eps = float(eps)
        if not (np.isfinite(eps) and eps > 0):
            raise ValueError("eps must be finite and > 0, got %r" % eps)
        if actuation not in (0, 1, False, True):
            raise ValueError("actuation must be a bool, got %r" % (actuation,))
        _check_f64("qacc", qacc, (n, m.nv), self.device)
        width = _state_width(m, time=False)
        del width["qacc_warmstart"]            # (no pass reads the warm start)
        bufs = {"qacc": qacc}
        bufs.update(_initial_state(initial_state, width, n, self.device))
        out = _outputs(self.device, fields, (n,), abi.INVERSE_FD_SHAPES, dict(nv=m.nv))
        params = abi.MyoInverseFdParams(eps=eps, actuation=int(bool(actuation)))
        self.batch.inverse_fd(params, stream=self._stream(), flags=_flags(constraints, discrete), **bufs, **out)
        return out

    STATIC_OPT_FIELDS = tuple(abi.STATIC_OPT_SHAPES)
    STATIC_OPT_DEFAULTS = dict(max_iter=50, tol=1e-12)

    def static_opt(self, qacc, reserve, weight=None, constraints=True, discrete=False, warmstart=None, max_iter=STATIC_OPT_DEFAULTS["max_iter"],
                   tol=STATIC_OPT_DEFAULTS["tol"], fields=("act", "reserve_force", "ctrl")):
        """Muscle static optimisation of every env at its current (qpos, qvel, act) (myo_batch_static_opt; include/myo_b200.h states the
        problem and the solver): the activations a in [0, 1] and reserve generalized forces r of least 1/2 sum w a^2 + 1/2 sum (r / reserve)^2
        whose muscle and reserve forces produce the acceleration qacc, i.e. G a + r = qfrc_inverse(qacc) - AM' bias.  qacc [num_envs, nv]
        as inverse() takes it, with its constraints and discrete flags; reserve: the reserve strengths rho > 0, a scalar or [nv] (no
        default: the right scale differs by orders of magnitude between models); weight: muscle weights > 0, a scalar or [nu] (None: 1);
        warmstart: the dual lambda [num_envs, nv] of an earlier call (None: 0).  reserve and weight may be numbers, arrays or tensors of
        any numeric dtype, device and layout (copied to this batch's device as float64); qacc and warmstart are contiguous float64 CUDA
        tensors on this batch's device.
        Returns {field: tensor [num_envs, ...]} of STATIC_OPT_FIELDS: act, reserve_force [nv], ctrl (the excitation that takes the current
        act to a in one mj_step, clipped to ctrlrange), actuator_force, muscle_gain, muscle_bias [nu], qfrc_inverse, lambda [nv], niter,
        converged (int32) and residual (|G a + r - t|_inf, converged when <= tol max(1, |t|_inf)); allocated per call.  One launch; not a
        state change."""
        m, n = self.mj_model, self.num_envs
        fields = _check_fields("static_opt", fields, self.STATIC_OPT_FIELDS)
        _check_f64("qacc", qacc, (n, m.nv), self.device)
        bufs = {"qacc": qacc, "reserve": _vector("reserve", reserve, m.nv, self.device)}
        if weight is not None:
            bufs["weight"] = _vector("weight", weight, m.nu, self.device)
        if warmstart is not None:
            _check_f64("warmstart", warmstart, (n, m.nv), self.device)
            bufs["lambda0"] = warmstart
        params = _check_solver("static_opt", abi.MyoStaticOptParams(max_iter=int(max_iter), tol=float(tol)), max_iter, tol)
        out = _outputs(self.device, set(fields) | {"act"}, (n,), abi.STATIC_OPT_SHAPES, dict(nu=m.nu, nv=m.nv))
        self.batch.static_opt(params, stream=self._stream(), flags=_flags(constraints, discrete), **bufs, **out)
        return {f: out[f] for f in fields}

    CMC_FIELDS = tuple(abi.CMC_SHAPES) + ("overflow",)

    def cmc(self, ref_qpos, ref_qvel, ref_qacc, kp, kv, reserve, weight=None, substeps=1, constraints=True, discrete=False, initial_state=None,
            warmstart=None, max_iter=STATIC_OPT_DEFAULTS["max_iter"], tol=STATIC_OPT_DEFAULTS["tol"],
            fields=("qpos", "qvel", "act", "ctrl", "act_opt", "reserve_force", "niter", "converged")):
        """Computed muscle control of every env along its own reference motion (myo_batch_cmc; include/myo_b200.h states the loop): for
        each frame t, the desired acceleration qacc_des = ref_qacc[:, t] + kv (ref_qvel[:, t] - qvel) + kp (ref_qpos[:, t] (-) qpos) ((-):
        mj_differentiatePos), the static optimisation of static_opt() for it (reserve, weight, constraints, discrete, max_iter and tol as
        there, warm-started from the previous frame's lambda, frame 0 from `warmstart` [num_envs, nv] or 0), the excitation that brings act
        to the optimal activations at the end of `substeps` mj_steps with ctrl held, and that interval of rollout() with qfrc_applied = the
        reserve forces.  ref_qpos [num_envs, T, nq], ref_qvel and ref_qacc [num_envs, T, nv] are contiguous float64 CUDA tensors on this
        batch's device; kp and kv are gains >= 0, reserve and weight strengths > 0, each a scalar or a vector ([nv], weight [nu]) given
        as in static_opt(): a number, array or tensor of any numeric dtype, device and layout.
        initial_state as rollout()'s.  Returns {field: tensor [num_envs, T, ...]} of CMC_FIELDS: qacc_des, ctrl, act_opt (a*),
        reserve_force, lambda [nv or nu], niter, converged (int32), residual, and the state after the frame's interval qpos, qvel, act,
        qacc, time (rollout()'s rows); overflow [num_envs] int32.  Row t equals static_opt() and rollout() run from row t - 1's state, bit
        for bit.  The tensors are allocated per call; the frames run on the device without a host synchronisation.  Not a state change."""
        torch, m, n = self.torch, self.mj_model, self.num_envs
        fields = _check_fields("cmc", fields, self.CMC_FIELDS)
        substeps = _check_substeps(substeps)
        T = int(ref_qpos.shape[1]) if isinstance(ref_qpos, torch.Tensor) and ref_qpos.dim() == 3 else 0
        if T < 1:
            raise ValueError("ref_qpos must be a float64 tensor [num_envs, T >= 1, nq], got %s" % (tuple(getattr(ref_qpos, "shape", ())),))
        _check_f64("ref_qpos", ref_qpos, (n, T, m.nq), self.device)
        _check_f64("ref_qvel", ref_qvel, (n, T, m.nv), self.device)
        _check_f64("ref_qacc", ref_qacc, (n, T, m.nv), self.device)
        bufs = {"ref_qpos": ref_qpos, "ref_qvel": ref_qvel, "ref_qacc": ref_qacc, "kp": _vector("kp", kp, m.nv, self.device, positive=False),
                "kv": _vector("kv", kv, m.nv, self.device, positive=False), "reserve": _vector("reserve", reserve, m.nv, self.device)}
        if weight is not None:
            bufs["weight"] = _vector("weight", weight, m.nu, self.device)
        if warmstart is not None:
            _check_f64("warmstart", warmstart, (n, m.nv), self.device)
            bufs["lambda0"] = warmstart
        bufs.update(_initial_state(initial_state, _state_width(m), n, self.device))
        params = _check_solver("cmc", abi.MyoCmcParams(max_iter=int(max_iter), substeps=substeps, tol=float(tol)), max_iter, tol)
        out = _outputs(self.device, fields, (n, T), abi.CMC_SHAPES, dict(nq=m.nq, nv=m.nv, nu=m.nu, na=m.na))
        self.batch.cmc(params, T, stream=self._stream(), flags=_flags(constraints, discrete), **bufs, **out)
        return out

    def examine_policy(self, policy, horizon=None, mode="exploration", seed=None, generator=None, keep_obs=True):
        """Batched MujocoEnv.examine_policy_new (env_base.py:853-969): one episode per env, observations / actions stay on the device;
        returns (Trace with one "Trial<k>" group per env, summary dict).  See myosuite_b200/rollout.py."""
        from . import rollout
        return rollout.examine_policy(self, policy, horizon=horizon, mode=mode, seed=seed, generator=generator, keep_obs=keep_obs)

    def forward_debug(self, ctrl, n_substeps=0):
        c = self.torch.as_tensor(np.asarray(ctrl), dtype=self.torch.float64, device=self.device).contiguous()
        self._dbg_ctrl = c
        self.batch.forward_debug(c, n_substeps, stream=self._stream())
        self.state_version += 1


class _Named:
    """One named element of mj_data, as MuJoCo's data.body(name) / site / actuator / joint accessors return it."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def __repr__(self):
        return "<%s>" % ", ".join("%s=%r" % kv for kv in self.__dict__.items())


class _DataView:
    """`env.mj_data`-like read access to the single env: qpos, qvel, act, time and every field of the mjData readout (MyoVecEnv.data)
    as numpy arrays, with MuJoCo's named views body(name), site(name), actuator(name), joint(name) and the contact list.  Lazy: the
    first access after a state change runs one readout launch and one device-to-host copy; later accesses read the host copy."""

    def __init__(self, vec):
        self._vec, self._version, self._d = vec, None, None

    def _fetch(self):
        v = self._vec
        if self._version != v.state_version:
            out = v.data()
            self._d = _row0(dict(qpos=v.t["qpos"], qvel=v.t["qvel"], act=v.t["act"][:, :v.mj_model.na], time=v.t["time"], **out))
            self._version = v.state_version
        return self._d

    def __getattr__(self, k):
        if k.startswith("_") or k not in ("qpos", "qvel", "act", "time") + self._vec.DATA_FIELDS:
            raise AttributeError(k)
        x = self._fetch()[k]
        return x.copy() if isinstance(x, np.ndarray) else x

    def _id(self, kind, key):
        return int(key) if isinstance(key, (int, np.integer)) else self._vec.mj_model.name2id(kind, key)

    def body(self, key):
        i, d = self._id("body", key), self._fetch()
        return _Named(id=i, xpos=d["xpos"][i].copy(), xquat=d["xquat"][i].copy(), xmat=d["xmat"][i].copy())

    def site(self, key):
        i = self._id("site", key)
        return _Named(id=i, xpos=self._fetch()["site_xpos"][i].copy())

    def actuator(self, key):
        i, d = self._id("actuator", key), self._fetch()
        return _Named(id=i, length=d["actuator_length"][i:i + 1].copy(), velocity=d["actuator_velocity"][i:i + 1].copy(), force=d["actuator_force"][i:i + 1].copy())

    def joint(self, key):
        from . import mjcf
        m, d = self._vec.mj_model, self._fetch()
        i = self._id("joint", key); t = int(m.jnt_type[i])
        nq_, nv_ = {mjcf.JNT_FREE: (7, 6), mjcf.JNT_BALL: (4, 3)}.get(t, (1, 1))
        q, dv = int(m.jnt_qposadr[i]), int(m.jnt_dofadr[i])
        return _Named(id=i, qpos=d["qpos"][q:q + nq_].copy(), qvel=d["qvel"][dv:dv + nv_].copy(), qacc=d["qacc"][dv:dv + nv_].copy())

    @property
    def contact(self):
        """The first ncon contacts (geom1, geom2, dist, pos, frame; arrays over the contacts, like MuJoCo's data.contact)."""
        d = self._fetch(); n = d["ncon"]
        return _Named(geom1=d["contact_geom"][:n, 0].copy(), geom2=d["contact_geom"][:n, 1].copy(), dist=d["contact_dist"][:n].copy(),
                      pos=d["contact_pos"][:n].copy(), frame=d["contact_frame"][:n].copy())


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
        self._ntip = len(v.tip_names)
        self.obs_keys = list(v.obs_keys)
        self.rwd_keys_wt = dict(v.kwargs.get("weighted_reward_keys") or tasks.DEFAULT_WEIGHTS[v.task])
        self._task_cfg = v.reward_cfg                     # host reward constants (tasks.configure)
        self.rwd_mode = "dense"
        self.obs_dict, self.rwd_dict, self.proprio_dict, self.visual_dict = {}, {}, {}, {}
        self._reseed = True
        self.reset()

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

    def _dev(self, x, shape):
        """An array-like input as a contiguous float64 tensor of `shape` on the env's device; None stays None."""
        v = self.vec
        return None if x is None else v.torch.as_tensor(np.asarray(x, dtype=np.float64).reshape(shape), device=v.device).contiguous()

    def _state(self, initial_state):
        """An initial_state {key: array} as {key: [1, width] tensor} ([1] for time); None stays None."""
        return None if initial_state is None else {k: self._dev(x, (1,) if k == "time" else (1, -1)) for k, x in initial_state.items()}

    def mj_inverse(self, qacc, constraints=True, discrete=False):
        """mujoco.mj_inverse for this env at its current state: {field: numpy array} of MyoVecEnv.inverse's INVERSE_FIELDS (qfrc_inverse,
        qfrc_constraint, contact_force [maxcon, 6], actuator_moment [nu, nv]) for the acceleration qacc [nv].  One launch, one
        device-to-host copy."""
        v = self.vec
        return _row0(v.inverse(self._dev(qacc, (1, -1)), constraints=constraints, discrete=discrete, fields=v.INVERSE_FIELDS))

    def mj_rollout(self, ctrl, qfrc_applied=None, substeps=1, initial_state=None):
        """mujoco.mj_step rollout of this env (MyoVecEnv.rollout): ctrl [nstep, nu] is MuJoCo's ctrl, not the action (no sigmoid remap:
        apply normalize_act's 1 / (1 + exp(-5 (a - 0.5))) yourself when starting from actions), qfrc_applied [nstep, nv] or None,
        initial_state {key: array} or None (the current state).  Returns {field: numpy array [nstep, ...]} of qpos, qvel, act, qacc, time
        and the int overflow flag.  The env's own state is left as it was.  One device-to-host copy."""
        v = self.vec
        nstep = np.asarray(ctrl, dtype=np.float64).reshape(-1, self.mj_model.nu).shape[0]
        return _row0(v.rollout(self._dev(ctrl, (1, nstep, -1)), qfrc_applied=self._dev(qfrc_applied, (1, nstep, self.mj_model.nv)), substeps=substeps,
                               initial_state=self._state(initial_state), fields=v.ROLLOUT_FIELDS))

    def mj_ik(self, sites, target_pos, target_quat=None, qpos_init=None, qpos_ref=None, dofs=None, site_weight=None,
              fields=("qpos", "niter", "converged", "err"), **params):
        """Inverse kinematics of this env (MyoVecEnv.ik): target_pos [ns, 3], target_quat [ns, 4] or None, qpos_init / qpos_ref [nq] or
        None, dofs and site_weight as there; params: max_iter, tol, damping, max_step, posture, eq_weight.  Returns {field: numpy array}
        (niter and converged as ints).  Not a state change.  One device-to-host copy."""
        ns = 1 if isinstance(sites, (str, int)) else len(sites)
        return _row0(self.vec.ik(sites, self._dev(target_pos, (1, ns, 3)), target_quat=self._dev(target_quat, (1, ns, 4)),
                                 qpos_init=self._dev(qpos_init, (1, -1)), qpos_ref=self._dev(qpos_ref, (1, -1)), dofs=dofs,
                                 site_weight=self._dev(site_weight, (ns, 2)), fields=fields, **params))

    def static_opt(self, qacc, reserve, weight=None, constraints=True, discrete=False, warmstart=None, fields=("act", "reserve_force", "ctrl"),
                   **params):
        """Muscle static optimisation of this env at its current state (MyoVecEnv.static_opt): qacc [nv], reserve (scalar or [nv]),
        weight [nu] or None, warmstart [nv] or None; params: max_iter, tol.  Returns {field: numpy array} (niter and converged as ints,
        residual as a float).  Not a state change.  One device-to-host copy."""
        return _row0(self.vec.static_opt(self._dev(qacc, (1, -1)), reserve if np.ndim(reserve) == 0 else self._dev(reserve, (-1,)),
                                         weight=self._dev(weight, (-1,)), constraints=constraints, discrete=discrete,
                                         warmstart=self._dev(warmstart, (1, -1)), fields=fields, **params))

    def cmc(self, ref_qpos, ref_qvel, ref_qacc, kp, kv, reserve, weight=None, initial_state=None, warmstart=None,
            fields=("qpos", "qvel", "act", "ctrl", "act_opt", "reserve_force", "niter", "converged"), **params):
        """Computed muscle control of this env along a reference motion (MyoVecEnv.cmc): ref_qpos [T, nq], ref_qvel and ref_qacc [T, nv],
        kp, kv, reserve (scalars or [nv]), weight [nu] or None, initial_state {key: array} or None (the current state), warmstart [nv] or
        None; params: substeps, constraints, discrete, max_iter, tol.  Returns {field: numpy array [T, ...]} (overflow as an int).  Not a
        state change.  One device-to-host copy."""
        T = np.asarray(ref_qpos).reshape(-1, self.mj_model.nq).shape[0]
        return _row0(self.vec.cmc(self._dev(ref_qpos, (1, T, -1)), self._dev(ref_qvel, (1, T, -1)), self._dev(ref_qacc, (1, T, -1)), kp, kv, reserve,
                                  weight=weight, initial_state=self._state(initial_state), warmstart=self._dev(warmstart, (1, -1)), fields=fields,
                                  **params))

    def mj_jacSite(self, site):
        """mujoco.mj_jacSite at the current state: (jacp [3, nv], jacr [3, nv]) as numpy arrays."""
        jp, jr, _, _ = self.vec.jac_site([site])
        return jp[0, 0].cpu().numpy(), jr[0, 0].cpu().numpy()

    def mjd_transitionFD(self, ctrl, eps=1e-6, flg_centered=False, substeps=1, qfrc_applied=None, initial_state=None):
        """mujoco.mjd_transitionFD of this env (MyoVecEnv.transition_fd) over one interval of `substeps` mj_steps: ctrl [nu] is MuJoCo's
        ctrl, qfrc_applied [nv] or None, initial_state {key: array} or None (the current state).  Returns numpy (A [nx, nx], B [nx, nu]),
        nx = 2 nv + na.  Not a state change.  One device-to-host copy."""
        r = _row0(self.vec.transition_fd(self._dev(ctrl, (1, self.mj_model.nu)), eps=eps, centered=flg_centered, substeps=substeps,
                                         qfrc_applied=self._dev(qfrc_applied, (1, self.mj_model.nv)), initial_state=self._state(initial_state)))
        return r["A"], r["B"]

    def mjd_inverseFD(self, qacc, eps=1e-6, flg_actuation=False, constraints=True, discrete=False, initial_state=None):
        """mujoco.mjd_inverseFD of this env (MyoVecEnv.inverse_fd) at the acceleration qacc [nv]: initial_state {key: array} of qpos,
        qvel, act or None (the current state).  Returns numpy (DfDq, DfDv, DfDa), each [nv, nv] in MuJoCo's layout (DfDq[i, j] =
        d f_j / d q_i).  Not a state change.  One device-to-host copy."""
        r = _row0(self.vec.inverse_fd(self._dev(qacc, (1, self.mj_model.nv)), eps=eps, actuation=flg_actuation, constraints=constraints,
                                      discrete=discrete, initial_state=self._state(initial_state)))
        return r["DfDq"], r["DfDv"], r["DfDa"]

    # ---- dicts (env_base.py:409-432, task get_obs_dict / get_reward_dict)
    def get_obs_dict(self, *sim_args):
        """obs_dict of the current observation.  (The reference signature takes (mj_model, mj_data); the state lives on the device here, so
        any arguments are ignored.)"""
        m = self.mj_model
        return tasks.obs_dict_from_vec(self.vec.task, self._last["obs_full"], np.array([self._last["time"]]), m.nq, m.nv, m.na, self._ntip)

    def get_reward_dict(self, obs_dict):
        r = tasks.reward_dict(self.vec.task, obs_dict, self.rwd_keys_wt, self._task_cfg)
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
        m = self.mj_model
        w = dict(tasks.obs_layout(self.vec.task, m.nq, m.nv, m.na, self._ntip))
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
            if tasks.task_of(entry) is None:
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
