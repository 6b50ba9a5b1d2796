"""CPU reference of muscle static optimisation (myo_batch_static_opt): the problem's data from the oracle, its solution by bounded least
squares, a numpy restatement of the device's dual Newton, and one step of MuJoCo's muscle activation dynamics.

    min_{a, r}  1/2 sum_m w_m a_m^2 + 1/2 sum_i (r_i / rho_i)^2   s.t.   G a + r = t,   0 <= a_m <= 1

with t = qfrc_inverse(qacc) - AM' b and G = AM' diag(g).  Eliminating r = t - G a leaves [W^1/2; diag(1/rho) G] a ~ [0; t / rho] over the
box, which scipy's lsq_linear(method="bvls") solves by an active-set method that shares nothing with the dual Newton."""
import numpy as np


def problem(o, m, qpos, qvel, act, qacc, flags=0):
    """(t, G, AM, g, b, tau) of one state from the oracle o: tau from its mj_inverse, AM = gear x ten_J of each muscle's tendon, and the
    muscle gain and bias from two forward passes (act = 0 gives actuator_force = b, act = 1 gives g + b)."""
    o.reset(); o.set(qpos=qpos, qvel=qvel, act=act, ctrl=np.zeros(m.nu))
    tau = o.inverse(qacc, flags).copy()
    o.reset(); o.set(qpos=qpos, qvel=qvel, act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
    b = o.f("actuator_force").copy()
    AM = o.f("ten_J").reshape(-1, m.nv)[m.actuator_trnid[:, 0]] * m.actuator_gear[:, 0, None]
    o.reset(); o.set(qpos=qpos, qvel=qvel, act=np.ones(m.na), ctrl=np.zeros(m.nu)); o.forward()
    g = o.f("actuator_force") - b
    t = tau - AM.T @ b
    return t, AM.T * g[None, :], AM, g, b, tau


def solve_lsq(t, G, w, rho):
    """a of the eliminated problem by lsq_linear(method="bvls"), and r = t - G a"""
    from scipy.optimize import lsq_linear
    nu = G.shape[1]
    A = np.vstack([np.diag(np.sqrt(w)), G / rho[:, None]])
    rhs = np.concatenate([np.zeros(nu), t / rho])
    res = lsq_linear(A, rhs, bounds=(0.0, 1.0), method="bvls", tol=1e-15, max_iter=10 * nu + 100)
    a = np.clip(res.x, 0.0, 1.0)
    return a, t - G @ a


def _phi(s, w):
    return np.where(s <= 0, 0.0, np.where(s < w, 0.5 * s * s / w, s - 0.5 * w))


def solve_dual_newton(t, G, w, rho, tol=1e-12, max_iter=50, lam=None):
    """The device's iteration (include/myo_b200.h: myo_static_opt_buffers), restated in numpy: (a, r, lambda, niter, converged, |F|_inf)."""
    nv = len(t)
    lam = np.zeros(nv) if lam is None else np.array(lam, dtype=np.float64)
    r2 = rho * rho
    thr = tol * max(1.0, np.abs(t).max())
    it = 0
    while True:
        s = G.T @ lam
        a = np.clip(s / w, 0.0, 1.0)
        F = G @ a + r2 * lam - t
        fn = np.abs(F).max()
        if fn <= thr or it >= max_iter:
            return a, r2 * lam, lam, it, fn <= thr, fn
        free = ((s / w > 0) | (s == 0)) & (s / w < 1)          # strictly inside the box, or at the kink s = 0
        H = (G[:, free] / w[free]) @ G[:, free].T + np.diag(r2)
        x = np.linalg.solve(H, -F)
        sd = G.T @ x
        A1, A2, slope = x @ (t - r2 * lam), r2 @ (x * x), -F @ x
        al = 1.0
        for _ in range(60):
            dpsi = al * A1 - 0.5 * al * al * A2 - np.sum(_phi(s + al * sd, w) - _phi(s, w))
            if dpsi >= 1e-4 * al * slope:
                break
            al *= 0.5
        lam = lam + al * x
        it += 1


def act_next(m, i, ctrl, act):
    """act after one mj_step of muscle i's activation dynamics with MuJoCo ctrl `ctrl` (mju_muscleDynamics, Euler)"""
    c = ctrl
    if m.actuator_ctrllimited[i]:
        c = min(max(c, m.actuator_ctrlrange[i, 0]), m.actuator_ctrlrange[i, 1])
    dyn = m.actuator_dynprm[i]
    cc, ac = min(max(c, 0.0), 1.0), min(max(act, 0.0), 1.0)
    ta, td, dctrl = dyn[0] * (0.5 + 1.5 * ac), dyn[1] / (0.5 + 1.5 * ac), cc - act
    if dyn[2] < 1e-15:
        tau = ta if dctrl > 0 else td
    else:
        x = min(max(dctrl / dyn[2] + 0.5, 0.0), 1.0)
        tau = td + (ta - td) * x * x * x * (3 * x * (2 * x - 5) + 10)
    return act + m.opt_timestep * dctrl / max(1e-15, tau)


def ctrl_range(m, i):
    """the controls that reach the activation dynamics: ctrlrange (when limited) intersected with [0, 1]"""
    if m.actuator_ctrllimited[i]:
        return max(m.actuator_ctrlrange[i, 0], 0.0), min(m.actuator_ctrlrange[i, 1], 1.0)
    return 0.0, 1.0


def excitation(m, i, act, a):
    """the ctrl of muscle i that takes act to a in one step: closed form with tausmooth = 0, bisection otherwise"""
    lo, hi = ctrl_range(m, i)
    dyn = m.actuator_dynprm[i]
    if dyn[2] < 1e-15:
        ac = min(max(act, 0.0), 1.0)
        tau = dyn[0] * (0.5 + 1.5 * ac) if a > act else dyn[1] / (0.5 + 1.5 * ac)
        return min(max(act + (a - act) * tau / m.opt_timestep, lo), hi)
    if act_next(m, i, hi, act) <= a:
        return hi
    if act_next(m, i, lo, act) >= a:
        return lo
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if not lo < mid < hi:
            break
        lo, hi = (mid, hi) if act_next(m, i, mid, act) < a else (lo, mid)
    return lo if abs(act_next(m, i, lo, act) - a) <= abs(act_next(m, i, hi, act) - a) else hi
