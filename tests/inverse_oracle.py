"""mj_inverse on the CPU oracle (tests/inverse_oracle.c): the oracle library's source plus oracle_inverse, compiled once per process
into a temporary directory (the source tree may be read-only)."""
import ctypes
import functools
import os

import numpy as np

from oracle.oracle_py import Oracle, build_extension

_HERE = os.path.dirname(os.path.abspath(__file__))
INV_NOCONSTRAINT, INV_DISCRETE = 1, 2


@functools.cache
def lib():
    L = build_extension(os.path.join(_HERE, "inverse_oracle.c"))
    L.oracle_inverse.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    L.oracle_inverse.restype = None
    return L


class InvOracle(Oracle):
    """The oracle with mj_inverse: inverse(qacc, flags) -> qfrc_inverse; f("qfrc_constraint") and f("efc_force") are then the inverse's."""

    def __init__(self, I, D):
        super().__init__(I, D, lib())

    def inverse(self, qacc, flags=0):
        self.f("qacc")[:] = qacc
        out = np.zeros(len(self.f("qvel")))
        self._L.oracle_inverse(self._h, int(flags), out.ctypes.data)
        return out
