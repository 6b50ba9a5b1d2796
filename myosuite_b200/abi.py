"""ctypes binding of the C-ABI in include/myo_b200.h (libmyo_b200.so, built in-tree by myosuite_b200.build).

Host code stays Python over torch tensors: tensors are passed as ``data_ptr()`` only; no torch types
cross the ABI.  There is NO CPU fallback: if the library or a CUDA device is missing the calls raise.
"""
import ctypes
import os

import numpy as np

from . import build as _build

_LIB = None

c_i32, c_i64, c_u64, c_f64, c_vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_double, ctypes.c_void_p

TASK_NONE, TASK_POSE, TASK_WALK, TASK_HOLD, TASK_REACH = 0, 1, 2, 3, 4
COND_NONE, COND_FATIGUE = 0, 2


class MyoDims(ctypes.Structure):
    _fields_ = [(n, c_i32) for n in ("nq", "nv", "nu", "na", "nbody", "njnt", "ntendon", "nM", "npair", "nta", "maxcon",
                                      "maxefc", "smem_bytes_per_env")] + [("reserved", c_i32 * 3)]


class MyoTaskCfg(ctypes.Structure):
    _fields_ = [(n, c_i32) for n in ("task", "frame_skip", "max_episode_steps", "normalize_act", "muscle_condition",
                                      "auto_reset", "reset_random", "maxcon", "reaf_dst", "reaf_src", "barrier_mode", "reserved_i", "fatigue_reset")] + \
               [("pose_thd", c_f64), ("weights", c_f64 * 8), ("solver_tolerance", c_f64), ("task_i", c_i32 * 16), ("task_d", c_f64 * 24), ("reserved", c_f64 * 2),
                ("reach_shape", c_f64 * 4), ("joint_random", c_f64 * 2)]


BUFFER_FIELDS = ["action", "qpos", "qvel", "act", "qacc_warmstart", "time", "fatigue", "target", "target_range", "init_qpos", "init_qvel", "env_prm",
                 "step_count", "episode_count", "obs", "reward", "done", "truncated", "ep_return", "last_return",
                 "tap_qacc", "tap_actuator_force", "tap_ten_length", "tap_qfrc_smooth", "tap_ncon", "tap_contact_pair",
                 "tap_contact_dist", "tap_moment", "tap_qM", "tap_phase_cycles", "fatigue_reset_vec", "overflow"]


class MyoBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in BUFFER_FIELDS]


EXPORTS = ["myo_last_error", "myo_version", "myo_model_from_blob", "myo_model_dims", "myo_model_destroy", "myo_batch_create",
           "myo_batch_bind", "myo_batch_destroy", "myo_batch_obs_dim", "myo_batch_reset", "myo_batch_step",
           "myo_batch_forward_debug", "myo_batch_launch_count", "myo_batch_observe", "myo_debug_chol_solve",
           "myo_batch_launch_info", "myo_batch_debug_perm"]


class MyoError(RuntimeError):
    pass


def lib_path():
    return _build.LIB


def lib(variant=None):
    """The product library, or (variant="f64rows") the verification build of the same source whose contact rows are stored in f64."""
    global _LIB
    if variant:
        if variant not in _VARIANTS:
            if variant not in _build.VARIANTS:
                raise MyoError("unknown library variant %r" % (variant,))
            path = _build.variant_path(variant)
            if not os.path.exists(path):          # (mtimes need not survive a copy of the tree: existence only, like the product library)
                path = _build.build_variant(variant, _build.VARIANTS[variant])
            _VARIANTS[variant] = _bind(ctypes.CDLL(path))
        return _VARIANTS[variant]
    if _LIB is None:
        path = os.environ.get("MYO_B200_LIB") or _build.LIB      # MYO_B200_LIB: a variant build (developer experiments)
        if not os.path.exists(path):
            path = _build.build()
        _LIB = _bind(ctypes.CDLL(path))
    return _LIB


_VARIANTS = {}


def _bind(L):
    L.myo_last_error.restype = ctypes.c_char_p
    L.myo_model_from_blob.argtypes = [c_vp, c_i64, c_vp, c_i64, ctypes.POINTER(c_vp)]
    L.myo_model_dims.argtypes = [c_vp, ctypes.POINTER(MyoTaskCfg), ctypes.POINTER(MyoDims)]
    L.myo_model_destroy.argtypes = [c_vp]
    L.myo_model_destroy.restype = None
    L.myo_batch_create.argtypes = [c_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(MyoTaskCfg), ctypes.POINTER(c_vp)]
    L.myo_batch_bind.argtypes = [c_vp, ctypes.POINTER(MyoBuffers)]
    L.myo_batch_destroy.argtypes = [c_vp]
    L.myo_batch_destroy.restype = None
    L.myo_batch_obs_dim.argtypes = [c_vp]
    L.myo_batch_reset.argtypes = [c_vp, c_vp, c_u64, c_i64, c_vp]
    L.myo_batch_step.argtypes = [c_vp, c_vp]
    L.myo_batch_observe.argtypes = [c_vp, c_vp]
    L.myo_batch_forward_debug.argtypes = [c_vp, c_vp, ctypes.c_int, c_vp]
    L.myo_batch_launch_count.argtypes = [c_vp]
    L.myo_batch_launch_count.restype = c_i64
    L.myo_debug_chol_solve.argtypes = [ctypes.c_int, c_vp, c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.myo_batch_launch_info.argtypes = [c_vp, c_vp, ctypes.c_int]
    L.myo_batch_debug_perm.argtypes = [c_vp, c_vp, ctypes.c_int]
    return L


def _check(rc, L=None):
    if rc != 0:
        raise MyoError((L or lib()).myo_last_error().decode())


class DeviceModel:
    """Host handle of a packed model (myo_model*)."""

    def __init__(self, I, D, variant=None):
        self.I = np.ascontiguousarray(I, dtype=np.int32)
        self.D = np.ascontiguousarray(D, dtype=np.float64)
        self.L = lib(variant)
        h = c_vp()
        _check(self.L.myo_model_from_blob(self.I.ctypes.data, self.I.size, self.D.ctypes.data, self.D.size, ctypes.byref(h)), self.L)
        self.handle = h

    def dims(self, cfg=None):
        d = MyoDims()
        _check(self.L.myo_model_dims(self.handle, ctypes.byref(cfg) if cfg is not None else None, ctypes.byref(d)), self.L)
        return d

    def __del__(self):
        if getattr(self, "handle", None):
            self.L.myo_model_destroy(self.handle)
            self.handle = None


class Batch:
    """myo_batch*: n_env envs of one model on one CUDA device, driven through bound torch tensors."""

    def __init__(self, model, device, n_env, cfg):
        self.model, self.cfg, self.n_env, self.device, self.L = model, cfg, n_env, device, model.L
        h = c_vp()
        _check(self.L.myo_batch_create(model.handle, device, n_env, ctypes.byref(cfg), ctypes.byref(h)), self.L)
        self.handle = h
        self.tensors = {}

    @property
    def obs_dim(self):
        return self.L.myo_batch_obs_dim(self.handle)

    def bind(self, **tensors):
        """tensors: name -> torch CUDA tensor (contiguous) for the fields of myo_buffers."""
        self.tensors.update(tensors)
        b = MyoBuffers()
        for k, t in self.tensors.items():
            if k not in BUFFER_FIELDS:
                raise KeyError(k)
            if t is None:
                continue
            if not t.is_contiguous():
                raise ValueError("%s must be contiguous" % k)
            setattr(b, k, t.data_ptr())
        _check(self.L.myo_batch_bind(self.handle, ctypes.byref(b)), self.L)

    def reset(self, mask=None, seed=0, env_offset=0, stream=None):
        _check(self.L.myo_batch_reset(self.handle, mask.data_ptr() if mask is not None else None, seed, env_offset, stream), self.L)

    def step(self, stream=None):
        _check(self.L.myo_batch_step(self.handle, stream), self.L)

    def observe(self, stream=None):
        _check(self.L.myo_batch_observe(self.handle, stream), self.L)

    def forward_debug(self, ctrl, n_substeps=0, stream=None):
        _check(self.L.myo_batch_forward_debug(self.handle, ctrl.data_ptr(), n_substeps, stream), self.L)

    @property
    def launches(self):
        return self.L.myo_batch_launch_count(self.handle)

    LAUNCH_INFO_KEYS = ("use_w14", "warps_per_cta", "grid", "rounds", "regroup", "balanced", "smem_bytes", "perm_slots")

    def launch_info(self):
        """How env steps are launched: product kernel (use_w14), warps per CTA, grid, rounds per CTA, slot -> env map (regroup / balanced)."""
        out = np.zeros(len(self.LAUNCH_INFO_KEYS), dtype=np.int32)
        _check(self.L.myo_batch_launch_info(self.handle, out.ctypes.data, out.size), self.L)
        return {k: int(v) for k, v in zip(self.LAUNCH_INFO_KEYS, out)}

    def perm(self):
        """Slot -> env map of the last env step (numpy int32 [perm_slots], -1 = idle slot); raises when regroup is off."""
        out = np.full(max(self.launch_info()["perm_slots"], 1), -1, dtype=np.int32)
        _check(self.L.myo_batch_debug_perm(self.handle, out.ctypes.data, out.size), self.L)
        return out

    def __del__(self):
        if getattr(self, "handle", None):
            self.L.myo_batch_destroy(self.handle)
            self.handle = None


def debug_chol_solve(H_packed, rhs, mode=1, device=0):
    """Solve count SPD systems with the kernel's dense solver (unit-test hook).  H_packed: [count, n(n+1)/2] lower triangles; rhs: [count, n]."""
    H = np.ascontiguousarray(H_packed, dtype=np.float64); x = np.ascontiguousarray(rhs, dtype=np.float64).copy()
    count, n = x.shape
    _check(lib().myo_debug_chol_solve(device, H.ctypes.data, x.ctypes.data, n, count, mode))
    return x
