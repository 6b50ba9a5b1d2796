"""mjData.qfrc_applied on the CPU oracle (tests/rollout_oracle.c): the oracle library's source plus a forward pass and a step with an
applied generalized force, compiled once per process into a temporary directory (the source tree may be read-only)."""
import ctypes
import functools
import os

import numpy as np

from oracle.oracle_py import Oracle, build_extension

_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def lib():
    L = build_extension(os.path.join(_HERE, "rollout_oracle.c"))
    for f in ("oracle_forward_applied", "oracle_step_applied"):
        getattr(L, f).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        getattr(L, f).restype = None
    return L


class AppliedOracle(Oracle):
    """The oracle with mjData.qfrc_applied: f("qfrc_applied") is a field like the others (so set(qfrc_applied=...) works), zero at
    creation and after reset() like mj_resetData, and forward() / step() add it to qfrc_smooth.  `L`: a library built from
    rollout_oracle.c's source (None: lib())."""

    def __init__(self, I, D, L=None):
        super().__init__(I, D, L or lib())
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
