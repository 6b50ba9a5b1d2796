"""ctypes binding of the C-ABI in include/myo_b200.h (libmyo_b200.so, built in-tree by myosuite_b200.build).

Host code stays Python over torch tensors: tensors are passed as ``data_ptr()`` only; no torch types
cross the ABI.  There is NO CPU fallback: if the library or a CUDA device is missing the calls raise.
"""
import ctypes
import operator
import os

import numpy as np

from . import build as _build

_LIB = None

c_i32, c_i64, c_u64, c_f64, c_vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_double, ctypes.c_void_p

TASK_NONE, TASK_POSE, TASK_WALK, TASK_HOLD, TASK_REACH = 0, 1, 2, 3, 4
RESET_ENV_LIMIT = 1 << 47           # MYO_RESET_ENV_LIMIT: global env ids below it key distinct reset streams
COND_NONE, COND_FATIGUE = 0, 2
ABI_VERSION = 2                     # myo_version() of the header this binding mirrors (MyoBuffers ends with final_obs since 2)


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
                 "tap_contact_dist", "tap_moment", "tap_qM", "tap_phase_cycles", "fatigue_reset_vec", "overflow", "final_obs"]


class MyoBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in BUFFER_FIELDS]


# myo_data_buffers (include/myo_b200.h): the mjData readout of myo_batch_data, field -> (group, dtype, trailing shape in the model's sizes)
DATA_FIELDS = ["xpos", "xquat", "xmat", "site_xpos", "site_source", "actuator_length", "actuator_velocity", "actuator_force", "qfrc_actuator",
               "qacc", "ncon", "contact_geom", "contact_dist", "contact_pos", "contact_frame", "contact_force"]
DATA_SHAPES = {"xpos": ("pose", "f64", ("nbody", 3)), "xquat": ("pose", "f64", ("nbody", 4)), "xmat": ("pose", "f64", ("nbody", 9)),
               "site_xpos": ("pose", "f64", ("nsite", 3)),
               "actuator_length": ("actuation", "f64", ("nu",)), "actuator_velocity": ("actuation", "f64", ("nu",)),
               "actuator_force": ("actuation", "f64", ("nu",)), "qfrc_actuator": ("actuation", "f64", ("nv",)),
               "qacc": ("dynamics", "f64", ("nv",)), "ncon": ("dynamics", "i32", ()), "contact_geom": ("dynamics", "i32", ("maxcon", 2)),
               "contact_dist": ("dynamics", "f64", ("maxcon",)), "contact_pos": ("dynamics", "f64", ("maxcon", 3)),
               "contact_frame": ("dynamics", "f64", ("maxcon", 9)), "contact_force": ("dynamics", "f64", ("maxcon", 6))}
SITE_MODEL, SITE_TARGET, SITE_ENV_PRM, SITE_AT_TARGET_POSE = 0, 1, 2, 3       # myo_data_buffers.site_source kinds


class MyoDataBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in DATA_FIELDS]


# myo_inverse_buffers (include/myo_b200.h): inverse dynamics of myo_batch_inverse, output -> trailing shape in the model's sizes
INVERSE_FIELDS = ["qacc", "qfrc_inverse", "qfrc_constraint", "contact_force", "actuator_moment"]
INVERSE_SHAPES = {"qfrc_inverse": ("nv",), "qfrc_constraint": ("nv",), "contact_force": ("maxcon", 6), "actuator_moment": ("nu", "nv")}
INV_NOCONSTRAINT, INV_DISCRETE = 1, 2           # MYO_INV_* flags


class MyoInverseBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in INVERSE_FIELDS]


# myo_rollout_buffers (include/myo_b200.h): mj_step rollouts of myo_batch_rollout.  Inputs, start state, then the outputs -> trailing shape
# after [n, nstep] in the model's sizes (overflow is [n], int32)
ROLLOUT_FIELDS = ["ctrl", "qfrc_applied", "qpos0", "qvel0", "act0", "qacc_warmstart0", "time0", "qpos", "qvel", "act", "qacc", "time", "overflow"]
ROLLOUT_SHAPES = {"qpos": ("nq",), "qvel": ("nv",), "act": ("na",), "qacc": ("nv",), "time": ()}
ROLLOUT_STATE = {"qpos": "qpos0", "qvel": "qvel0", "act": "act0", "qacc_warmstart": "qacc_warmstart0", "time": "time0"}     # initial_state key -> field


class MyoRolloutBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in ROLLOUT_FIELDS]


# myo_ik_buffers / myo_ik_params (include/myo_b200.h): inverse kinematics of myo_batch_ik.  Inputs, then the outputs -> trailing shape
# after [n] in the call's sizes (ns sites)
IK_FIELDS = ["site_id", "site_quat", "site_weight", "target_pos", "target_quat", "qpos0", "qpos_ref", "dof_mask",
             "qpos", "niter", "converged", "err", "site_xpos", "site_xmat", "jacp", "jacr"]
IK_SHAPES = {"qpos": ("nq",), "niter": (), "converged": (), "err": ("ns", 2), "site_xpos": ("ns", 3), "site_xmat": ("ns", 9),
             "jacp": ("ns", 3, "nv"), "jacr": ("ns", 3, "nv")}
IK_MAXSITE = 16                                 # MYO_IK_MAXSITE


class MyoIkBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in IK_FIELDS]


class MyoIkParams(ctypes.Structure):
    _fields_ = [("nsite", c_i32), ("max_iter", c_i32)] + [(n, c_f64) for n in ("tol", "damping", "max_step", "posture_weight", "eq_weight")]


# myo_fd_buffers / myo_fd_params (include/myo_b200.h): finite-difference transition Jacobians of myo_batch_transition_fd.  Inputs, start
# state, then the outputs (A [n, nx, nx], B [n, nx, nu], overflow [n] int32; nx = 2 nv + na)
FD_FIELDS = ["ctrl", "qfrc_applied", "qpos0", "qvel0", "act0", "qacc_warmstart0", "A", "B", "overflow"]


class MyoFdBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in FD_FIELDS]


class MyoFdParams(ctypes.Structure):
    _fields_ = [("eps", c_f64), ("centered", c_i32), ("substeps", c_i32)]


# myo_static_opt_buffers / myo_static_opt_params (include/myo_b200.h): muscle static optimisation of myo_batch_static_opt.  Inputs, then
# the outputs -> trailing shape after [n] in the model's sizes
STATIC_OPT_FIELDS = ["qacc", "weight", "reserve", "lambda0", "act", "reserve_force", "ctrl", "actuator_force", "muscle_gain", "muscle_bias",
                     "qfrc_inverse", "lambda", "niter", "converged", "residual"]
STATIC_OPT_SHAPES = {"act": ("nu",), "reserve_force": ("nv",), "ctrl": ("nu",), "actuator_force": ("nu",), "muscle_gain": ("nu",),
                     "muscle_bias": ("nu",), "qfrc_inverse": ("nv",), "lambda": ("nv",), "niter": (), "converged": (), "residual": ()}


class MyoStaticOptBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in STATIC_OPT_FIELDS]


class MyoStaticOptParams(ctypes.Structure):
    _fields_ = [("max_iter", c_i32), ("tol", c_f64)]


# myo_cmc_buffers / myo_cmc_params (include/myo_b200.h): computed muscle control of myo_batch_cmc.  Inputs, start state, then the outputs
# -> trailing shape after [n, nstep] in the model's sizes (niter and converged int32; overflow is [n], int32)
CMC_FIELDS = ["ref_qpos", "ref_qvel", "ref_qacc", "kp", "kv", "weight", "reserve", "lambda0", "qpos0", "qvel0", "act0", "qacc_warmstart0", "time0",
              "qacc_des", "ctrl", "act_opt", "reserve_force", "lambda", "niter", "converged", "residual", "qpos", "qvel", "act", "qacc", "time",
              "overflow"]
CMC_SHAPES = {"qacc_des": ("nv",), "ctrl": ("nu",), "act_opt": ("nu",), "reserve_force": ("nv",), "lambda": ("nv",), "niter": (), "converged": (),
              "residual": (), "qpos": ("nq",), "qvel": ("nv",), "act": ("na",), "qacc": ("nv",), "time": ()}


class MyoCmcBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in CMC_FIELDS]


class MyoCmcParams(ctypes.Structure):
    _fields_ = [("max_iter", c_i32), ("substeps", c_i32), ("tol", c_f64)]


# myo_inverse_fd_buffers / myo_inverse_fd_params (include/myo_b200.h): finite-difference Jacobians of the inverse dynamics of
# myo_batch_inverse_fd.  Inputs, start state, then the outputs -> trailing shape after [n] in the model's sizes (overflow is [n], int32)
INVERSE_FD_FIELDS = ["qacc", "qpos0", "qvel0", "act0", "DfDq", "DfDv", "DfDa", "qfrc_inverse", "overflow"]
INVERSE_FD_SHAPES = {"DfDq": ("nv", "nv"), "DfDv": ("nv", "nv"), "DfDa": ("nv", "nv"), "qfrc_inverse": ("nv",)}


class MyoInverseFdBuffers(ctypes.Structure):
    _fields_ = [(n, c_vp) for n in INVERSE_FD_FIELDS]


class MyoInverseFdParams(ctypes.Structure):
    _fields_ = [("eps", c_f64), ("actuation", c_i32)]


EXPORTS = ["myo_last_error", "myo_version", "myo_model_from_blob", "myo_model_dims", "myo_model_destroy", "myo_batch_create",
           "myo_batch_bind", "myo_batch_destroy", "myo_batch_obs_dim", "myo_batch_reset", "myo_batch_step",
           "myo_batch_forward_debug", "myo_batch_launch_count", "myo_batch_observe", "myo_debug_chol_solve",
           "myo_batch_launch_info", "myo_batch_debug_perm", "myo_model_layout", "myo_batch_data", "myo_batch_inverse", "myo_batch_rollout",
           "myo_batch_ik", "myo_batch_transition_fd", "myo_batch_static_opt", "myo_batch_cmc", "myo_batch_inverse_fd"]

# myo_model_layout slots (include/myo_b200.h): persistent offsets and sizes, scratch offsets and sizes, then the scalars
LAYOUT_PERSISTENT = ("qpos", "qvel", "act", "qws", "dax", "dan", "qM", "fsm", "eprm", "wz", "cnt", "scr")
LAYOUT_SCRATCH = ("xpos", "xmat", "U", "PL", "mom", "tlen", "tvel", "tfrc", "cin", "crb", "bf", "conJ", "efD", "efA", "eqJ", "icon", "con", "clist",
                  "gpose", "efR", "efV", "va", "vg", "vp", "vMa", "vMp", "H", "Hs", "LD", "Dinv")
LAYOUT_SCALARS = ("head", "afterK", "extNonSolve", "solveEnd", "arefInH", "qwsInH", "n_per_warp", "maxcon", "maxefc")
LAYOUT_N = 2 * len(LAYOUT_PERSISTENT) + 2 * len(LAYOUT_SCRATCH) + len(LAYOUT_SCALARS)


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
        path = _build.LIB
        if not os.path.exists(path):
            path = _build.build()
        _LIB = _bind(ctypes.CDLL(path))
    return _LIB


_VARIANTS = {}


def _bind(L):
    L.myo_last_error.restype = ctypes.c_char_p
    L.myo_model_from_blob.argtypes = [c_vp, c_i64, c_vp, c_i64, ctypes.POINTER(c_vp)]
    L.myo_model_dims.argtypes = [c_vp, ctypes.POINTER(MyoTaskCfg), ctypes.POINTER(MyoDims)]
    L.myo_model_layout.argtypes = [c_vp, ctypes.POINTER(MyoTaskCfg), c_vp, ctypes.c_int]
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
    L.myo_batch_data.argtypes = [c_vp, ctypes.POINTER(MyoDataBuffers), c_vp]
    L.myo_batch_inverse.argtypes = [c_vp, ctypes.POINTER(MyoInverseBuffers), ctypes.c_int, c_vp]
    L.myo_batch_rollout.argtypes = [c_vp, ctypes.POINTER(MyoRolloutBuffers), ctypes.c_int, ctypes.c_int, c_vp]
    L.myo_batch_ik.argtypes = [c_vp, ctypes.POINTER(MyoIkBuffers), ctypes.POINTER(MyoIkParams), c_vp]
    L.myo_batch_transition_fd.argtypes = [c_vp, ctypes.POINTER(MyoFdBuffers), ctypes.POINTER(MyoFdParams), c_vp]
    L.myo_batch_static_opt.argtypes = [c_vp, ctypes.POINTER(MyoStaticOptBuffers), ctypes.POINTER(MyoStaticOptParams), ctypes.c_int, c_vp]
    L.myo_batch_cmc.argtypes = [c_vp, ctypes.POINTER(MyoCmcBuffers), ctypes.POINTER(MyoCmcParams), ctypes.c_int, ctypes.c_int, c_vp]
    L.myo_batch_inverse_fd.argtypes = [c_vp, ctypes.POINTER(MyoInverseFdBuffers), ctypes.POINTER(MyoInverseFdParams), ctypes.c_int, c_vp]
    L.myo_batch_launch_count.argtypes = [c_vp]
    L.myo_batch_launch_count.restype = c_i64
    L.myo_debug_chol_solve.argtypes = [ctypes.c_int, c_vp, c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.myo_batch_launch_info.argtypes = [c_vp, c_vp, ctypes.c_int]
    L.myo_batch_debug_perm.argtypes = [c_vp, c_vp, ctypes.c_int]
    if L.myo_version() != ABI_VERSION:
        raise MyoError("%s has ABI version %d, this binding needs %d: rebuild it (python -m myosuite_b200.build)" % (L._name, L.myo_version(), ABI_VERSION))
    return L


def _buffers(cls, tensors):
    """A cls (a struct of device pointers) with each tensor's data pointer in the field of its name; None leaves the field null."""
    s = cls()
    names = {n for n, _ in cls._fields_}
    for k, t in tensors.items():
        if k not in names:
            raise KeyError(k)
        if t is None:
            continue
        if not t.is_contiguous():
            raise ValueError("%s must be contiguous" % k)
        setattr(s, k, t.data_ptr())
    return s


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

    def layout(self, cfg=None):
        """Shared-memory layout of one env's slice (myo_model_layout; no device needed), in doubles from the slice start:
        {"o": {persistent region: offset}, "o_size": {...}, "s": {scratch region: offset}, "s_size": {...}, and the scalars}."""
        v = np.zeros(LAYOUT_N, dtype=np.int32)
        _check(self.L.myo_model_layout(self.handle, ctypes.byref(cfg) if cfg is not None else None, v.ctypes.data, v.size), self.L)
        v = [int(x) for x in v]
        npr, nsc = len(LAYOUT_PERSISTENT), len(LAYOUT_SCRATCH)
        out = {"o": dict(zip(LAYOUT_PERSISTENT, v[:npr])), "o_size": dict(zip(LAYOUT_PERSISTENT, v[npr:2 * npr])),
               "s": dict(zip(LAYOUT_SCRATCH, v[2 * npr:2 * npr + nsc])), "s_size": dict(zip(LAYOUT_SCRATCH, v[2 * npr + nsc:2 * npr + 2 * nsc]))}
        out.update(zip(LAYOUT_SCALARS, v[2 * npr + 2 * nsc:]))
        return out

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
        b = _buffers(MyoBuffers, self.tensors)
        _check(self.L.myo_batch_bind(self.handle, ctypes.byref(b)), self.L)

    def reset(self, mask=None, seed=0, env_offset=0, stream=None):
        """Reset the masked envs (all when mask is None) from the Philox streams of (seed, env_offset + env, episode_count): seed in
        [0, 2^64), global env ids in [0, 2^47) (RESET_ENV_LIMIT), where distinct keys give distinct streams.  Checked here, before ctypes
        would wrap an out-of-range integer into another key."""
        seed, env_offset = operator.index(seed), operator.index(env_offset)
        if not 0 <= seed < 1 << 64:
            raise ValueError("reset seed must be in [0, 2**64), got %d" % seed)
        if env_offset < 0 or env_offset + self.n_env > RESET_ENV_LIMIT:
            raise ValueError("env_offset must be in [0, 2**47 - n_env] = [0, %d], got %d" % (RESET_ENV_LIMIT - self.n_env, env_offset))
        _check(self.L.myo_batch_reset(self.handle, mask.data_ptr() if mask is not None else None, seed, env_offset, stream), self.L)

    def step(self, stream=None):
        _check(self.L.myo_batch_step(self.handle, stream), self.L)

    def observe(self, stream=None):
        _check(self.L.myo_batch_observe(self.handle, stream), self.L)

    def forward_debug(self, ctrl, n_substeps=0, stream=None):
        _check(self.L.myo_batch_forward_debug(self.handle, ctrl.data_ptr(), n_substeps, stream), self.L)

    def data(self, stream=None, **tensors):
        """mjData readout (myo_batch_data) into the given torch CUDA tensors (names of DATA_FIELDS; only these are computed)."""
        d = _buffers(MyoDataBuffers, tensors)
        _check(self.L.myo_batch_data(self.handle, ctypes.byref(d), stream), self.L)

    def inverse(self, stream=None, flags=0, **tensors):
        """Inverse dynamics (myo_batch_inverse) into the given torch CUDA tensors (names of INVERSE_FIELDS: qacc in, the others out; qacc and
        qfrc_inverse are required).  flags: INV_NOCONSTRAINT | INV_DISCRETE."""
        d = _buffers(MyoInverseBuffers, tensors)
        _check(self.L.myo_batch_inverse(self.handle, ctypes.byref(d), flags, stream), self.L)

    def rollout(self, nstep, substeps, stream=None, **tensors):
        """mj_step rollout (myo_batch_rollout) of nstep intervals of `substeps` mj_steps with the given torch CUDA tensors (names of
        ROLLOUT_FIELDS: ctrl [n, nstep, nu] required, qfrc_applied and the start state *0 in, the others out)."""
        d = _buffers(MyoRolloutBuffers, tensors)
        _check(self.L.myo_batch_rollout(self.handle, ctypes.byref(d), nstep, substeps, stream), self.L)

    def ik(self, params, stream=None, **tensors):
        """Inverse kinematics (myo_batch_ik) with the given torch CUDA tensors (names of IK_FIELDS: site_id, target_pos and qpos are
        required) and a MyoIkParams."""
        d = _buffers(MyoIkBuffers, tensors)
        _check(self.L.myo_batch_ik(self.handle, ctypes.byref(d), ctypes.byref(params), stream), self.L)

    def transition_fd(self, params, stream=None, **tensors):
        """Finite-difference transition Jacobians (myo_batch_transition_fd) with the given torch CUDA tensors (names of FD_FIELDS: ctrl
        [n, nu] and at least one of A, B are required) and a MyoFdParams."""
        d = _buffers(MyoFdBuffers, tensors)
        _check(self.L.myo_batch_transition_fd(self.handle, ctypes.byref(d), ctypes.byref(params), stream), self.L)

    def static_opt(self, params, stream=None, flags=0, **tensors):
        """Muscle static optimisation (myo_batch_static_opt) with the given torch CUDA tensors (names of STATIC_OPT_FIELDS: qacc, reserve
        and act are required), a MyoStaticOptParams and MYO_INV_* flags."""
        d = _buffers(MyoStaticOptBuffers, tensors)
        _check(self.L.myo_batch_static_opt(self.handle, ctypes.byref(d), ctypes.byref(params), flags, stream), self.L)

    def cmc(self, params, nstep, stream=None, flags=0, **tensors):
        """Computed muscle control (myo_batch_cmc) over nstep frames with the given torch CUDA tensors (names of CMC_FIELDS: ref_qpos,
        ref_qvel, ref_qacc, kp, kv and reserve are required), a MyoCmcParams and MYO_INV_* flags."""
        d = _buffers(MyoCmcBuffers, tensors)
        _check(self.L.myo_batch_cmc(self.handle, ctypes.byref(d), ctypes.byref(params), nstep, flags, stream), self.L)

    def inverse_fd(self, params, stream=None, flags=0, **tensors):
        """Finite-difference Jacobians of the inverse dynamics (myo_batch_inverse_fd) with the given torch CUDA tensors (names of
        INVERSE_FD_FIELDS: qacc and at least one of DfDq, DfDv, DfDa are required), a MyoInverseFdParams and MYO_INV_* flags."""
        d = _buffers(MyoInverseFdBuffers, tensors)
        _check(self.L.myo_batch_inverse_fd(self.handle, ctypes.byref(d), ctypes.byref(params), flags, stream), self.L)

    @property
    def launches(self):
        return self.L.myo_batch_launch_count(self.handle)

    LAUNCH_INFO_KEYS = ("use_w14", "warps_per_cta", "grid", "rounds", "regroup", "balanced", "smem_bytes", "perm_slots", "hand_shape")

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
