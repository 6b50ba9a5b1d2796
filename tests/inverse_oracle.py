"""mj_inverse on the CPU oracle (tests/inverse_oracle.c): the oracle library's source plus oracle_inverse, compiled once per process
into a temporary directory (the source tree may be read-only)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from oracle.oracle_py import Oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
INV_NOCONSTRAINT, INV_DISCRETE = 1, 2
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="myo_inverse_oracle_"), "libmyo_inverse_oracle.so")
        # the flags of oracle/Makefile
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-shared", "-o", so, os.path.join(_HERE, "inverse_oracle.c"), "-lm"])
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
        L.oracle_inverse.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.oracle_inverse.restype = None
        _LIB = L
    return _LIB


class InvOracle(Oracle):
    """The oracle with mj_inverse: inverse(qacc, flags) -> qfrc_inverse; f("qfrc_constraint") and f("efc_force") are then the inverse's."""

    def __init__(self, I, D):
        self._I = np.ascontiguousarray(I, dtype=np.int32)
        self._D = np.ascontiguousarray(D, dtype=np.float64)
        self._L = lib()
        self._h = self._L.oracle_create(self._I.ctypes.data, self._D.ctypes.data)
        if not self._h:
            raise RuntimeError("oracle_create failed (blob magic/version)")

    def inverse(self, qacc, flags=0):
        self.f("qacc")[:] = qacc
        out = np.zeros(len(self.f("qvel")))
        self._L.oracle_inverse(self._h, int(flags), out.ctypes.data)
        return out
