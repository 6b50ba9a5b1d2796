"""CPU reference of one frame of computed muscle control (myo_batch_cmc), in float64 from the oracle alone and sharing no code with the
device: the desired acceleration from FdOracle.differentiate_pos, the static optimisation of static_opt_ref (the problem from InvOracle,
solved by bounded least squares), the excitation over the k-step map of static_opt_ref.act_next (vectorised over the muscles), and the
interval on AppliedOracle with ctrl and qfrc_applied held for k steps.

A state is {qpos, qvel, act, qacc_warmstart, time} of one env, as rollout()'s initial_state rows."""
import numpy as np

import static_opt_ref as R
from fd_oracle import FdOracle
from inverse_oracle import INV_DISCRETE, INV_NOCONSTRAINT, InvOracle
from parity_helpers import Oracles, _in_regime

STATE = ("qpos", "qvel", "act", "qacc_warmstart", "time")


def flags(constraints=True, discrete=False):
    return (0 if constraints else INV_NOCONSTRAINT) | (INV_DISCRETE if discrete else 0)


def act_next(m, ctrl, act):
    """static_opt_ref.act_next of every muscle at once: act after one mj_step of the activation dynamics with MuJoCo ctrl `ctrl`"""
    lim = np.asarray(m.actuator_ctrllimited).astype(bool)
    cr, dyn = np.asarray(m.actuator_ctrlrange), np.asarray(m.actuator_dynprm)
    c = np.where(lim, np.minimum(np.maximum(ctrl, cr[:, 0]), cr[:, 1]), ctrl)
    cc, ac = np.minimum(np.maximum(c, 0.0), 1.0), np.minimum(np.maximum(act, 0.0), 1.0)
    ta, td, dctrl = dyn[:, 0] * (0.5 + 1.5 * ac), dyn[:, 1] / (0.5 + 1.5 * ac), cc - act
    sharp = dyn[:, 2] < 1e-15
    x = np.minimum(np.maximum(dctrl / np.where(sharp, 1.0, dyn[:, 2]) + 0.5, 0.0), 1.0)
    tau = np.where(sharp, np.where(dctrl > 0, ta, td), td + (ta - td) * x * x * x * (3 * x * (2 * x - 5) + 10))
    return act + m.opt_timestep * dctrl / np.maximum(1e-15, tau)


def act_after(m, ctrl, act, k):
    for _ in range(k):
        act = act_next(m, ctrl, act)
    return act


def ctrl_bounds(m):
    b = np.array([R.ctrl_range(m, i) for i in range(m.nu)]).reshape(-1, 2)
    return b[:, 0], b[:, 1]


def excitation(m, act, a, k):
    """the ctrl of every muscle that, held for k steps, takes act to a: static_opt_ref.excitation at k = 1, otherwise a bisection over the
    k-step map run on all muscles at once (each muscle stops where test_cmc.excitation_k's loop would), clipped to the control range"""
    act, a = np.asarray(act, dtype=np.float64), np.asarray(a, dtype=np.float64)
    if k == 1:
        return np.array([R.excitation(m, i, act[i], a[i]) for i in range(m.nu)])
    lo, hi = ctrl_bounds(m)
    top, bot = act_after(m, hi, act, k) <= a, act_after(m, lo, act, k) >= a
    l, u = lo.copy(), hi.copy()
    live = ~(top | bot)
    for _ in range(200):
        mid = 0.5 * (l + u)
        live &= (l < mid) & (mid < u)
        if not live.any():
            break
        below = act_after(m, mid, act, k) < a
        l, u = np.where(live & below, mid, l), np.where(live & ~below, mid, u)
    pick = np.where(np.abs(act_after(m, l, act, k) - a) <= np.abs(act_after(m, u, act, k) - a), l, u)
    return np.where(top, hi, np.where(bot, lo, pick))


class OraclePair:
    """(InvOracle, FdOracle) of each env's model, built once per env: the hold task's object size is the env's own (parity_helpers.Oracles)"""

    def __init__(self, env):
        self.inv, self.fd = Oracles(env), Oracles(env)
        self.inv.Oracle, self.inv.base = InvOracle, InvOracle(env.I, env.D)
        self.fd.Oracle, self.fd.base = FdOracle, FdOracle(env.I, env.D)
        self.cache = {}

    def get(self, e, prm=None):
        if e not in self.cache:
            self.cache[e] = (self.inv.get(prm), self.fd.get(prm))
        return self.cache[e]


class CmcRef:
    """One env's CMC frame on the CPU.  kp, kv and rho are scalars or [nv], w [nu]; fl the inverse flags of the call; k its substeps."""

    def __init__(self, m, io, fo, kp, kv, rho, w=None, fl=0, k=1):
        self.m, self.io, self.fo, self.fl, self.k = m, io, fo, fl, k
        self.kp, self.kv = np.broadcast_to(np.float64(kp), (m.nv,)), np.broadcast_to(np.float64(kv), (m.nv,))
        self.rho = np.broadcast_to(np.float64(rho), (m.nv,)).copy()
        self.w = np.ones(m.nu) if w is None else np.broadcast_to(np.float64(w), (m.nu,)).copy()

    def qacc_des(self, s, ref_q, ref_v, ref_a):
        return ref_a + self.kv * (ref_v - s["qvel"]) + self.kp * self.fo.differentiate_pos(s["qpos"], ref_q)

    def solve(self, s, qdes):
        """the static optimisation at state s: {t, G, AM, g, b, act_opt, reserve_force, lambda} (lambda = r / rho^2)"""
        m = self.m
        t, G, AM, g, b, _ = R.problem(self.io, m, s["qpos"], s["qvel"], s["act"][:m.na], qdes, self.fl)
        a, r = R.solve_lsq(t, G, self.w, self.rho)
        return dict(t=t, G=G, AM=AM, g=g, b=b, act_opt=a, reserve_force=r, **{"lambda": r / self.rho ** 2})

    def excitation(self, act, a):
        return excitation(self.m, act[:self.m.na], a, self.k)

    def interval(self, s, ctrl, reserve):
        """k steps with ctrl and qfrc_applied held from state s (its warm start and time; the inverse-wrap roots cold, as at the start of
        every rollout launch): (the state after it, whether every substep's contacts stayed in the parity regime, the largest ncon)"""
        o, m = self.fo, self.m
        o.reset()
        o.set(qpos=s["qpos"], qvel=s["qvel"], act=s["act"][:m.na], qacc_warmstart=s["qacc_warmstart"])
        o.f("time")[:] = s["time"]
        o.f("wrap_warm")[:] = 1
        o.f("wrap_z")[:] = -1
        o.set(ctrl=ctrl, qfrc_applied=reserve)
        ok, ncon = True, 0
        for _ in range(self.k):
            o.step(1)
            ok = ok and _in_regime(o, m)
            ncon = max(ncon, o.ncon)
        out = {k: o.f(k).copy() for k in ("qpos", "qvel", "act", "time")}
        out["qacc_warmstart"] = o.f("qacc").copy()
        return out, ok, ncon

    def frame(self, s, ref_q, ref_v, ref_a):
        """the whole frame on the CPU from state s: {qacc_des, act_opt, reserve_force, lambda, ctrl, next, regime, ncon}"""
        qd = self.qacc_des(s, ref_q, ref_v, ref_a)
        S = self.solve(s, qd)
        c = self.excitation(s["act"], S["act_opt"])
        nxt, ok, ncon = self.interval(s, c, S["reserve_force"])
        return dict(qacc_des=qd, ctrl=c, next=nxt, regime=ok, ncon=ncon, **{k: S[k] for k in ("act_opt", "reserve_force", "lambda")})


def kkt_error(S, w):
    """the lsq solution's optimality on its own data: |a - clip(G' lambda / w, 0, 1)| relative to max(|G|' |lambda| / w, 1), and
    |G a + r - t| relative to max(|t|, 1) (zero up to rounding: r = t - G a by construction)"""
    G, lam, a = S["G"], S["lambda"], S["act_opt"]
    ref = np.clip(G.T @ lam / w, 0.0, 1.0)
    scale = np.maximum(np.abs(G).T @ np.abs(lam) / w, 1.0)
    F = G @ a + S["reserve_force"] - S["t"]
    return float(np.max(np.abs(a - ref) / scale)), float(np.abs(F).max() / max(1.0, np.abs(S["t"]).max()))
