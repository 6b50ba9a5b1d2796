"""mj_jacSite and inverse kinematics on the CPU oracle (tests/ik_oracle.c): the oracle library's source plus oracle_jac_site and oracle_ik,
compiled once per process into a temporary directory (the source tree may be read-only)."""
import ctypes
import functools
import os

import numpy as np

from oracle.oracle_py import Oracle, build_extension

_HERE = os.path.dirname(os.path.abspath(__file__))
# the defaults of MyoVecEnv.ik (myosuite_b200/vec_env.py: MyoVecEnv.IK_DEFAULTS)
DEFAULTS = dict(max_iter=200, tol=1e-6, damping=1e-3, max_step=0.5, posture=0.0, eq_weight=1.0)


@functools.cache
def lib():
    L = build_extension(os.path.join(_HERE, "ik_oracle.c"))
    L.oracle_jac_site.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 5
    L.oracle_jac_site.restype = None
    L.oracle_ik.argtypes = ([ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_int] + [ctypes.c_double] * 5
                            + [ctypes.c_void_p] * 7)
    L.oracle_ik.restype = None
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data


class IkOracle(Oracle):
    """The oracle with mj_jacSite and oracle_ik.  `site_quat` is the model's mjModel.site_quat (the blob carries no site frames)."""

    def __init__(self, I, D, site_quat):
        super().__init__(I, D, lib())
        self.site_quat = np.ascontiguousarray(site_quat, dtype=np.float64)
        self.nv = len(self.f("qvel"))

    def jac_site(self, site, qpos=None):
        """(jacp [3, nv], jacr [3, nv], site_xpos [3], site_xmat [9]) at qpos (default: the oracle's)."""
        if qpos is not None:
            self.set(qpos=qpos)
        jp, jr, p, R = np.zeros((3, self.nv)), np.zeros((3, self.nv)), np.zeros(3), np.zeros(9)
        sq = np.ascontiguousarray(self.site_quat[site])
        self._L.oracle_jac_site(self._h, int(site), sq.ctypes.data, jp.ctypes.data, jr.ctypes.data, p.ctypes.data, R.ctypes.data)
        return jp, jr, p, R

    def ik(self, sites, target_pos, qpos0, target_quat=None, qpos_ref=None, dof_mask=None, site_weight=None, **params):
        """oracle_ik from qpos0: dict of qpos, niter, converged, err [ns, 2], site_xpos, site_xmat, jacp, jacr [ns, 3, nv]."""
        p = dict(DEFAULTS, **params)
        sites = np.ascontiguousarray(sites, dtype=np.int32)
        ns = len(sites)
        sq = np.ascontiguousarray(self.site_quat[sites])
        tp = np.ascontiguousarray(target_pos, dtype=np.float64).reshape(ns, 3)
        tq = None if target_quat is None else np.ascontiguousarray(target_quat, dtype=np.float64).reshape(ns, 4)
        ref = None if qpos_ref is None else np.ascontiguousarray(qpos_ref, dtype=np.float64)
        mask = None if dof_mask is None else np.ascontiguousarray(dof_mask, dtype=np.uint8)
        sw = None if site_weight is None else np.ascontiguousarray(site_weight, dtype=np.float64).reshape(ns, 2)
        self.set(qpos=qpos0)
        niter, conv = ctypes.c_int(0), ctypes.c_int(0)
        out = {"err": np.zeros((ns, 2)), "site_xpos": np.zeros((ns, 3)), "site_xmat": np.zeros((ns, 9)),
               "jacp": np.zeros((ns, 3, self.nv)), "jacr": np.zeros((ns, 3, self.nv))}
        self._L.oracle_ik(self._h, ns, sites.ctypes.data, sq.ctypes.data, _ptr(sw), tp.ctypes.data, _ptr(tq), _ptr(ref), _ptr(mask),
                          int(p["max_iter"]), float(p["tol"]), float(p["damping"]), float(p["max_step"]), float(p["posture"]), float(p["eq_weight"]),
                          ctypes.byref(niter), ctypes.byref(conv), *(out[k].ctypes.data for k in ("err", "site_xpos", "site_xmat", "jacp", "jacr")))
        out.update(qpos=self.f("qpos").copy(), niter=niter.value, converged=conv.value)
        return out
