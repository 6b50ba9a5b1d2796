"""mjData.qfrc_applied on the CPU oracle (tests/rollout_oracle.c): the oracle library's source plus a forward pass and a step with an
applied generalized force, compiled once per process into a temporary directory (the source tree may be read-only)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from oracle.oracle_py import Oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="myo_rollout_oracle_"), "libmyo_rollout_oracle.so")
        # the flags of oracle/Makefile
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-shared", "-o", so, os.path.join(_HERE, "rollout_oracle.c"), "-lm"])
        L = ctypes.CDLL(so)
        L.oracle_create.restype = ctypes.c_void_p
        L.oracle_create.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.oracle_field.restype = ctypes.POINTER(ctypes.c_double)
        L.oracle_field.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
        L.oracle_ifield.restype = ctypes.POINTER(ctypes.c_int)
        L.oracle_ifield.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
        for f in ("oracle_forward", "oracle_step", "oracle_reset", "oracle_destroy"):
            getattr(L, f).argtypes = [ctypes.c_void_p]
            getattr(L, f).restype = None
        L.oracle_step_n.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.oracle_step_n.restype = None
        L.oracle_info.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.oracle_info.restype = ctypes.c_int
        for f in ("oracle_forward_applied", "oracle_step_applied"):
            getattr(L, f).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
            getattr(L, f).restype = None
        _LIB = L
    return _LIB


class AppliedOracle(Oracle):
    """The oracle with mjData.qfrc_applied: f("qfrc_applied") is a field like the others (so set(qfrc_applied=...) works), zero at
    creation and after reset() like mj_resetData, and forward() / step() add it to qfrc_smooth."""

    def __init__(self, I, D):
        self._I = np.ascontiguousarray(I, dtype=np.int32)
        self._D = np.ascontiguousarray(D, dtype=np.float64)
        self._L = lib()
        self._h = self._L.oracle_create(self._I.ctypes.data, self._D.ctypes.data)
        if not self._h:
            raise RuntimeError("oracle_create failed (blob magic/version)")
        self._applied = np.zeros(len(super().f("qvel")))

    def f(self, name):
        return self._applied if name == "qfrc_applied" else super().f(name)

    def reset(self):
        super().reset()
        self._applied[:] = 0

    def forward(self):
        self._L.oracle_forward_applied(self._h, self._applied.ctypes.data)

    def step(self, n=1):
        for _ in range(n):
            self._L.oracle_step_applied(self._h, self._applied.ctypes.data)
