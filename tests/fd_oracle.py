"""MuJoCo's mjd_transitionFD on the CPU oracle (tests/fd_oracle.c): the rollout oracle's source plus integratePos, differentiatePos and
oracle_transition_fd, compiled once per process into a temporary directory (the source tree may be read-only)."""
import ctypes
import functools
import os

import numpy as np

from oracle.oracle_py import build_extension
from rollout_oracle import AppliedOracle

_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def lib():
    L = build_extension(os.path.join(_HERE, "fd_oracle.c"))
    vp, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    for f in ("oracle_forward_applied", "oracle_step_applied"):
        getattr(L, f).argtypes = [vp, vp]
        getattr(L, f).restype = None
    L.oracle_integrate_pos.argtypes = [vp, vp, vp, d]
    L.oracle_differentiate_pos.argtypes = [vp, vp, d, vp, vp]
    L.oracle_transition_fd.argtypes = [vp, vp, vp, d, i, i, vp, vp]
    for f in ("oracle_integrate_pos", "oracle_differentiate_pos", "oracle_transition_fd"):
        getattr(L, f).restype = None
    return L


def _arr(x, n):
    a = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
    assert a.size == n, (a.size, n)
    return a


class FdOracle(AppliedOracle):
    """AppliedOracle (mjData.qfrc_applied) with mjd_transitionFD over one interval of `substeps` steps, mj_integratePos and
    mj_differentiatePos.  The state set on it is the start; transition_fd leaves it as it was."""

    def __init__(self, I, D):
        super().__init__(I, D, lib())

    def integrate_pos(self, qpos, v, scale):
        q = _arr(qpos, len(self.f("qpos"))).copy()
        self._L.oracle_integrate_pos(self._h, q.ctypes.data, _arr(v, len(self.f("qvel"))).ctypes.data, float(scale))
        return q

    def differentiate_pos(self, q1, q2, dt=1.0):
        nq, nv = len(self.f("qpos")), len(self.f("qvel"))
        v = np.zeros(nv)
        self._L.oracle_differentiate_pos(self._h, v.ctypes.data, float(dt), _arr(q1, nq).ctypes.data, _arr(q2, nq).ctypes.data)
        return v

    def transition_fd(self, ctrl, qfrc_applied=None, eps=1e-6, centered=False, substeps=1, A=True, B=True):
        """(A [nx, nx], B [nx, nu]) from the current state (None for a block not asked for), nx = 2 nv + na."""
        nv, na, nu = len(self.f("qvel")), len(self.f("act")), len(self.f("ctrl"))
        nx = 2 * nv + na
        c = _arr(ctrl, nu)
        f = None if qfrc_applied is None else _arr(qfrc_applied, nv)
        Ao = np.full((nx, nx), np.nan) if A else None
        Bo = np.full((nx, nu), np.nan) if B else None
        self._L.oracle_transition_fd(self._h, c.ctypes.data, None if f is None else f.ctypes.data, float(eps), int(bool(centered)), int(substeps),
                                     None if Ao is None else Ao.ctypes.data, None if Bo is None else Bo.ctypes.data)
        return Ao, Bo
