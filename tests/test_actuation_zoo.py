"""Tendon wraps, muscle actuation, joint limits, joint equalities and the in-kernel solver sizes against plain numpy references and
the CPU oracle, on synthetic models.

The shipped models reach a narrow slice of this code: every muscle has tausmooth = 0, gear = 1 and ctrllimited = 1; every limited
joint has margin 0 and one solref / solimp; every equality has solimp[0] == solimp[1] (impedance's early exit); inside wraps,
side-site-free wraps and world-fixed wrap geoms exist only on one or two models; the tree-sparse integrator runs on a branched tree
nowhere.  The zoo here is four kinds of model, each written as MJCF, compiled by `mjcf.compile_mjcf` and run as a physics-only batch:

- WRAP: nine tendons across a branched hinge chain, one muscle each: sphere and cylinder wraps outside without a side site, outside
  with one, and inside; wrap geoms on the world, on a moving body and on the body of one endpoint; one tendon with two wrap elements
  and a constant same-body segment; a cylinder side site with |s_xy| < r <= |s| (the 3-D norm makes it an outside wrap); a sphere
  whose ends and centre are collinear (a tie: only length and finiteness are meaningful there).
- MUSCLE: six muscles on a hinge-hinge-slide chain with tausmooth 0 and > 0, gear 0.5 / 1 / 2.5, ctrllimited true and false and
  several (lmin, lmax, vmax, fpmax, fvmax) and dynprm sets; configurations put every force-length, force-velocity and passive piece in
  reach, with ctrl outside [0, 1] and outside ctrlrange and act outside [0, 1].
- LIM_TREE / LIM_CROSS: hinge and slide limits with margin 0 and > 0, a range narrower than twice the margin (two rows), a range of
  exactly twice the margin, solimp powers 1, 2 and 2.5 with a 1 cm width, solimp[0] == solimp[1], several solrefs; joint equalities
  with five non-zero polycoefs, ref != 0 on both joints, one without joint2, one inactive and non-degenerate solimp.  In LIM_TREE
  every equality stays inside one chain (PD_EQ_TREE = 1), in LIM_CROSS one crosses branches (PD_EQ_TREE = 0).
- SWEEP_<nv>: branched hinge trees at nv = 7 (sparse integrator), 16, 24, 28, 35, 36, 37 and 40 (dense Newton / Euler sizes around
  the register Cholesky's bordered cases and its > 36 row fallback) with a few limits, one equality and one capsule-plane pair.

The plain references (numpy, f64) restate MuJoCo's documented formulas and elementary geometry; none reads the oracle's code."""
import os

import numpy as np
import pytest

from parity_helpers import relerr

ROWS = ["p48", "f64"]
FWD_QACC = 1e-7                        # one forward pass (test_gpu_parity.py's bound for the hand)
REL = 1e-12                            # actuator lengths, forces and moments against the oracle (relative to the largest entry)
ROLL_QPOS, ROLL_QVEL = 1e-7, 1e-5      # 10 chained substeps
MID = dict(qpos=2e-7, qvel=1e-5, qacc=1e-6)     # product kernels: the mid-episode bounds of test_product_parity.py
MINVAL = 1e-15
FD_H = 1e-6                            # central difference step of the moment check (rad or m)
SWEEP_NV = [7, 16, 24, 28, 35, 36, 37, 40]
REPORT = {}


# ----------------------------------------------------------------------------- plain references
def solparam(solimp):
    """MuJoCo's clamping of solimp (getsolparam)."""
    si = np.array(solimp, float)
    si[0], si[1], si[3] = (np.clip(si[k], 1e-4, 0.9999) for k in (0, 1, 3))
    si[2], si[4] = max(0.0, si[2]), max(1.0, si[4])
    return si


def impedance(solimp, pos, margin):
    """MuJoCo's constraint impedance d(r): solimp[0] at r = 0 to solimp[1] at |r| >= width, r = pos - margin, a power-p sigmoid
    through solimp[3] (documentation, "Solver parameters")."""
    d0, d1, width, mid, p = solparam(solimp)
    if d0 == d1 or width <= MINVAL:
        return 0.5 * (d0 + d1)
    x = abs(pos - margin) / width
    if x >= 1 or x <= 0:
        return d1 if x >= 1 else d0
    if p == 1:
        y = x
    elif x <= mid:
        y = mid * (x / mid) ** p
    else:
        y = 1 - (1 - mid) * ((1 - x) / (1 - mid)) ** p
    return d0 + y * (d1 - d0)


def kb(solref, solimp, h):
    """stiffness K and damping B of the reference acceleration aref = -B v - K imp (pos - margin) (refsafe: time constant >= 2 h)"""
    dmax = solparam(solimp)[1]
    tc, dr = max(solref[0], 2 * h), solref[1]
    return 1 / (dmax * dmax * tc * tc * dr * dr), 2 / (dmax * tc)


def fl_piece(L, lmin, lmax):
    a, b = 0.5 * (lmin + 1), 0.5 * (1 + lmax)
    return "FL<lmin" if L < lmin else "FL>lmax" if L > lmax else "FL1" if L <= a else "FL2" if L <= 1 else "FL3" if L <= b else "FL4"


def muscle_gain(length, vel, lr, g):
    """MuJoCo's muscle gain -F * FL(L) * FV(V) (documentation, "Muscles"): g = gainprm (range0, range1, force, scale, lmin, lmax, vmax,
    fpmax, fvmax).  FL is two quadratic bumps joined at L = 1 and zero outside [lmin, lmax]; FV rises quadratically from 0 at V = -1 to 1
    at V = 0 and saturates at fvmax at V = fvmax - 1.  Returns (gain, FL piece, FV piece)."""
    r0, r1, F, _, lmin, lmax, vmax, _, fvmax = g[:9]
    L0 = (lr[1] - lr[0]) / (r1 - r0)
    L, V = r0 + (length - lr[0]) / L0, vel / (L0 * vmax)
    a, b = 0.5 * (lmin + 1), 0.5 * (1 + lmax)
    if L < lmin or L > lmax:
        FL = 0.0
    elif L <= a:
        FL = 0.5 * ((L - lmin) / (a - lmin)) ** 2
    elif L <= 1:
        FL = 1 - 0.5 * ((1 - L) / (1 - a)) ** 2
    elif L <= b:
        FL = 1 - 0.5 * ((L - 1) / (b - 1)) ** 2
    else:
        FL = 0.5 * ((lmax - L) / (lmax - b)) ** 2
    y = fvmax - 1
    if V <= -1:
        FV, fv = 0.0, "FV<=-1"
    elif V <= 0:
        FV, fv = (V + 1) ** 2, "FV(-1,0]"
    elif V <= y:
        FV, fv = fvmax - (y - V) ** 2 / y, "FV(0,y]"
    else:
        FV, fv = fvmax, "FV>y"
    return -F * FL * FV, fl_piece(L, lmin, lmax), fv


def muscle_bias(length, lr, bp):
    """MuJoCo's passive muscle force: 0 up to L = 1, a quadratic to L = b = (1 + lmax) / 2, then linear with slope fpmax / (b - 1)."""
    r0, r1, F, _, _, lmax, _, fpmax = bp[:8]
    L = r0 + (length - lr[0]) / ((lr[1] - lr[0]) / (r1 - r0))
    b = 0.5 * (1 + lmax)
    if L <= 1:
        return 0.0, "FP<=1"
    if L <= b:
        return -F * fpmax * 0.5 * ((L - 1) / (b - 1)) ** 2, "FP(1,b]"
    return -F * fpmax * (0.5 + (L - b) / (b - 1)), "FP>b"


def muscle_dynamics(ctrl, act, dynprm):
    """MuJoCo's muscle activation: act_dot = (clip(ctrl, 0, 1) - act) / tau with Millard's activation / deactivation time constants and,
    for tausmooth > 0, a quintic smoothstep between them over dctrl in [-tausmooth / 2, tausmooth / 2]."""
    c, a = min(max(ctrl, 0.0), 1.0), min(max(act, 0.0), 1.0)
    ta, td = dynprm[0] * (0.5 + 1.5 * a), dynprm[1] / (0.5 + 1.5 * a)
    dctrl = c - act
    if dynprm[2] < MINVAL:
        tau = ta if dctrl > 0 else td
    else:
        x = min(max(dctrl / dynprm[2] + 0.5, 0.0), 1.0)
        tau = td + (ta - td) * (6 * x ** 5 - 15 * x ** 4 + 10 * x ** 3)
    return dctrl / max(MINVAL, tau)


def _rot2(v, ang):
    c, s = np.cos(ang), np.sin(ang)
    return np.array([c * v[0] - s * v[1], s * v[0] + c * v[1]])


def _segs_cross(a, b, c, d):
    """do the 2-D segments ab and cd meet?"""
    def orient(p, q, r):
        return (q[0] - p[0]) * (r[1] - p[1]) - (q[1] - p[1]) * (r[0] - p[0])
    o1, o2, o3, o4 = orient(a, b, c), orient(a, b, d), orient(c, d, a), orient(c, d, b)
    return o1 * o2 <= 0 and o3 * o4 <= 0


def wrap_outside_2d(a0, a1, r, sd):
    """Shortest path a0 -> circle -> a1 hugging the circle on one side: (2-D length, arc angle, branch).  Each end leaves along a
    tangent of length sqrt(|a|^2 - r^2) touching the circle at angle +-acos(r / |a|) from its own direction; the two senses give two
    candidate paths.  Without a side site the path wraps only when the straight segment meets the disc, on the side whose tangent points
    are closer; with a side site it also wraps when the segment passes on the far side of the site, on the side the site faces.  A
    candidate whose two straight pieces cross is not a path."""
    if np.dot(a0, a0) < r * r or np.dot(a1, a1) < r * r:
        return None, None, "endpoint-inside"
    dif = a1 - a0
    c = a0 + np.clip(-np.dot(dif, a0) / np.dot(dif, dif), 0, 1) * dif
    crosses = np.dot(c, c) <= r * r
    if not crosses and (sd is None or np.dot(c, sd) >= 0):
        return None, None, "clear"
    cands = []
    for sg in (1, -1):
        t0 = r * _rot2(a0 / np.linalg.norm(a0), -sg * np.arccos(r / np.linalg.norm(a0)))
        t1 = r * _rot2(a1 / np.linalg.norm(a1), sg * np.arccos(r / np.linalg.norm(a1)))
        if sd is not None:
            mdir = t0 + t1
            score = np.dot(mdir / np.linalg.norm(mdir), sd) if np.linalg.norm(mdir) >= MINVAL else sd[0]
        else:
            score = -np.dot(t0 - t1, t0 - t1)
        bad = _segs_cross(a0, t0, a1, t1)
        cands.append((-10000 if bad else score, t0, t1, bad))
    score, t0, t1, bad = cands[0] if cands[0][0] > cands[1][0] else cands[1]
    if bad:
        return None, None, "seg-reject"
    ang = np.arccos(np.clip(np.dot(t0, t1) / (r * r), -1, 1))
    tie = abs(cands[0][0] - cands[1][0]) < 1e-9
    L = np.sqrt(np.dot(a0, a0) - r * r) + r * ang + np.sqrt(np.dot(a1, a1) - r * r)
    return L, ang, ("tie" if tie else "side-forced" if not crosses else "wrap")


def wrap_inside_2d(a0, a1, r):
    """Inverse (inside) wrap: the path a0 -> c -> a1 through one point c of the circle, the stationary point of |a0 - c| + |c - a1| on
    the arc facing both ends (Alhazen's problem), found by bounded 1-D minimisation of the angle of c refined to 1e-14.  Straight when an
    end lies inside the circle or the segment crosses the disc.  (2-D legs of the path, branch)"""
    from scipy.optimize import minimize_scalar
    n0, n1 = np.linalg.norm(a0), np.linalg.norm(a1)
    if n0 <= r or n1 <= r:
        return None, "endpoint-inside"
    dif = a1 - a0
    t = -np.dot(dif, a0) / np.dot(dif, dif)
    if 0 < t < 1 and np.linalg.norm(a0 + t * dif) <= r:
        return None, "crosses"
    th0, th1 = np.arctan2(a0[1], a0[0]), np.arctan2(a1[1], a1[0])
    dth = (th1 - th0 + np.pi) % (2 * np.pi) - np.pi
    G = abs(dth)
    # MuJoCo's Newton solve from z = 1 - 1e-7 gives up when its residual is already positive there: the end directions are within about
    # 1e-3 rad of the tangent limit.  It then keeps the point in the direction of the ends' midpoint, which is what the reference does.
    A, B, z = r / n0, r / n1, 1 - 1e-7
    if np.cos(G) < 1 - MINVAL and np.arcsin(A * z) + np.arcsin(B * z) - 2 * np.arcsin(z) + G > 0:
        mdir = 0.5 * (a0 + a1)
        c = r * mdir / np.linalg.norm(mdir)
        return (np.linalg.norm(a0 - c), np.linalg.norm(a1 - c)), "no-solution"
    f = lambda ph: np.linalg.norm(a0 - r * np.array([np.cos(ph), np.sin(ph)])) + np.linalg.norm(a1 - r * np.array([np.cos(ph), np.sin(ph)]))
    lo, hi = sorted((th0, th0 + dth))
    res = minimize_scalar(f, bounds=(lo, hi), method="bounded", options=dict(xatol=1e-14, maxiter=500))
    ph = res.x
    for _ in range(3):      # Newton refinement of the stationary point
        e = 1e-6
        d1, d2 = (f(ph + e) - f(ph - e)) / (2 * e), (f(ph + e) - 2 * f(ph) + f(ph - e)) / (e * e)
        if d2 > 0 and lo <= ph - d1 / d2 <= hi:
            ph -= d1 / d2
    c = r * np.array([np.cos(ph), np.sin(ph)])
    return (np.linalg.norm(a0 - c), np.linalg.norm(a1 - c)), ("collinear" if np.cos(G) >= 1 - MINVAL else "alhazen")


def wrap_ref(x0, x1, gpos, gmat, r, cyl, side, inside):
    """(length of the path x0 -> wrap geom -> x1, branch).  Spheres wrap in the plane of the centre and both ends (any plane through a
    collinear pair: the length does not depend on it); cylinders in their xy plane, the height spread along the unrolled 2-D path, so
    the 3-D length is hypot(2-D length, dz) (the helix)."""
    p0, p1 = gmat.T @ (x0 - gpos), gmat.T @ (x1 - gpos)
    s = None if side is None else gmat.T @ (side - gpos)
    straight = float(np.linalg.norm(x1 - x0))
    if np.linalg.norm(p0) < MINVAL or np.linalg.norm(p1) < MINVAL:
        return straight, "at-centre"
    if cyl:
        e0, e1, dz, tag = np.array([1.0, 0, 0]), np.array([0, 1.0, 0]), p1[2] - p0[2], "cyl"
    else:
        e0 = p0 / np.linalg.norm(p0)
        n = np.cross(p0, p1)
        collinear = np.linalg.norm(n) < MINVAL
        if collinear:
            n = np.cross(e0, [0.0, 0.0, 1.0] if abs(e0[2]) < 0.9 else [1.0, 0.0, 0.0])
        e1 = np.cross(n / np.linalg.norm(n), e0)
        dz, tag = 0.0, "sph-collinear" if collinear else "sph"
    a0, a1 = np.array([p0 @ e0, p0 @ e1]), np.array([p1 @ e0, p1 @ e1])
    if inside:
        legs, br = wrap_inside_2d(a0, a1, r)
        if legs is None:
            return straight, "in-" + br
        return float(np.hypot(legs[0] + legs[1], dz)), "in-" + br + ("-" + tag if tag != "cyl" else "")
    sd = None
    if s is not None:
        sd = np.array([s @ e0, s @ e1])
        sd = np.array([r, 0.0]) if np.linalg.norm(sd) < MINVAL else r * sd / np.linalg.norm(sd)
    L2, ang, br = wrap_outside_2d(a0, a1, r, sd)
    if L2 is None:
        return straight, "out-" + br
    return float(np.hypot(L2, dz)), "out-" + br + ("-" + tag if tag == "sph-collinear" else "")


def tendon_ref(m, kin, t):
    """(length of tendon t from the host kinematics, [(wrap geom, side site, branch)])"""
    from myosuite_b200 import mjcf, mjmath as mm
    def site(s):
        b = m.site_bodyid[s]
        return kin["xpos"][b] + kin["xmat"][b] @ m.site_pos[s]
    adr, num = int(m.tendon_adr[t]), int(m.tendon_num[t])
    L, branches, j = 0.0, [], 0
    while j < num - 1:
        s0 = int(m.wrap_objid[adr + j])
        if m.wrap_type[adr + j + 1] == mjcf.WRAP_SITE:
            L += float(np.linalg.norm(site(int(m.wrap_objid[adr + j + 1])) - site(s0))); j += 1
            continue
        g, s1, ss = int(m.wrap_objid[adr + j + 1]), int(m.wrap_objid[adr + j + 2]), int(m.wrap_prm[adr + j + 1])
        b = m.geom_bodyid[g]
        gpos, gmat = kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g], kin["xmat"][b] @ mm.quat2mat(m.geom_quat[g])
        side = site(ss) if ss >= 0 else None
        inside = side is not None and np.linalg.norm(side - gpos) < m.geom_size[g][0]     # the 3-D norm decides, for cylinders too
        l, br = wrap_ref(site(s0), site(s1), gpos, gmat, float(m.geom_size[g][0]), m.wrap_type[adr + j + 1] == mjcf.WRAP_CYLINDER, side, inside)
        L += l; branches.append((g, ss, br)); j += 2
    return L, branches


def gauss_qacc(M, qacc_smooth, rows):
    """Exact minimiser of the Gauss cost 1/2 (a - a0)' M (a - a0) + sum_eq D/2 (J a - aref)^2 + sum_lim D/2 min(0, J a - aref)^2, by
    enumerating the active set of the (few) inequality rows: the cost is convex and piecewise quadratic, and exactly one active set
    is consistent with its own minimiser (up to ties on a kink, where the candidates agree)."""
    import itertools
    ineq = [k for k, r in enumerate(rows) if not r[3]]
    best = None
    for nact in range(len(ineq) + 1):
        for S in itertools.combinations(ineq, nact):
            H, g = M.copy(), M @ qacc_smooth
            for k, (J, aref, D, eq) in enumerate(rows):
                if eq or k in S:
                    H += D * np.outer(J, J); g += D * J * aref
            a = np.linalg.solve(H, g)
            ok = all(((J @ a - aref) <= 1e-12 * max(1, abs(aref))) == (k in S) or abs(J @ a - aref) <= 1e-12 * max(1, abs(aref))
                     for k, (J, aref, D, eq) in enumerate(rows) if not eq)
            if ok:
                c = 0.5 * (a - qacc_smooth) @ M @ (a - qacc_smooth) + sum(0.5 * D * min(0.0, J @ a - aref) ** 2 if not eq else 0.5 * D * (J @ a - aref) ** 2
                                                                          for J, aref, D, eq in rows)
                if best is None or c < best[0]:
                    best = (c, a)
    return best[1]


def constraint_rows(m, qpos, qvel):
    """The joint equality and limit rows of a state from MuJoCo's definitions: [(J, aref, D, is_equality)], D = imp / ((1 - imp) *
    invweight0), aref = -B v - K imp (pos - margin).  Equality rows: pos = q1 - q1_0 - poly(q2 - q2_0), margin 0.  Limit rows: pos = the
    distance to the range end, active when pos < margin (strict)."""
    h, rows = m.opt_timestep, []
    for e in range(m.neq):
        if not m.eq_active0[e]:
            continue
        j1, j2 = int(m.eq_obj1id[e]), int(m.eq_obj2id[e])
        q1, d1 = m.jnt_qposadr[j1], m.jnt_dofadr[j1]
        J = np.zeros(m.nv); J[d1] = 1.0
        pos, iw = qpos[q1] - m.qpos0[q1], m.dof_invweight0[d1]
        c = m.eq_data[e]
        if j2 >= 0:
            q2, d2 = m.jnt_qposadr[j2], m.jnt_dofadr[j2]
            x = qpos[q2] - m.qpos0[q2]
            pos -= sum(c[k] * x ** k for k in range(5))
            J[d2] = -sum(k * c[k] * x ** (k - 1) for k in range(1, 5))
            iw += m.dof_invweight0[d2]
        else:
            pos -= c[0]
        imp = impedance(m.eq_solimp[e], pos, 0.0)
        K, B = kb(m.eq_solref[e], m.eq_solimp[e], h)
        rows.append((J, -B * (J @ qvel) - K * imp * pos, imp / ((1 - imp) * iw), True))
    for j in range(m.njnt):
        if not m.jnt_limited[j]:
            continue
        q, d, mg = qpos[m.jnt_qposadr[j]], m.jnt_dofadr[j], m.jnt_margin[j]
        for sg, dist in ((1.0, q - m.jnt_range[j, 0]), (-1.0, m.jnt_range[j, 1] - q)):
            if dist < mg:
                J = np.zeros(m.nv); J[d] = sg
                imp = impedance(m.jnt_solimp[j], dist, mg)
                K, B = kb(m.jnt_solref[j], m.jnt_solimp[j], h)
                rows.append((J, -B * (J @ qvel) - K * imp * (dist - mg), imp / ((1 - imp) * m.dof_invweight0[d]), False))
    return rows


# ----------------------------------------------------------------------------- models
def _g(name, typ, size, pos="0 0 0", extra=""):
    return '<geom name="%s" type="%s" size="%s" pos="%s" contype="0" conaffinity="0" %s/>' % (name, typ, size, pos, extra)


def _muscle(name, tendon, lr=(0.01, 1.0), **kw):
    kw.setdefault("force", 5)
    return '<muscle name="%s" tendon="%s" lengthrange="%.17g %.17g" %s/>' % (name, tendon, lr[0], lr[1], " ".join('%s="%s"' % kv for kv in sorted(kw.items())))


# WRAP: world W, body A (hinge z at the origin) with children B (hinge z) -> D (hinge y) and C (hinge tilted)
WRAP_TENDONS = {     # tendon -> path (sites and (geom, side site or None))
    "t_sph_out": ["W0", ("wsph", None), "B0"],              # world sphere, no side site
    "t_sph_side": ["C0", ("asph", "as_out"), "B1"],         # moving sphere, side site
    "t_sph_in": ["B0", ("asph", "as_in"), "C1"],            # moving sphere, inside
    "t_cyl_out": ["W1", ("wcyl", None), "A1"],              # world cylinder, no side site
    "t_cyl_side": ["W0", ("wcyl", "wc_out"), "D0"],         # world cylinder, side site with |s_xy| < r <= |s|
    "t_cyl_in": ["C0", ("acyl", "ac_in"), "D0"],            # moving cylinder, inside
    "t_same": ["A0", ("asph", None), "D1"],                 # wrap geom on the body of the first end
    "t_seq": ["W0", ("wsph", "ws_out"), "A0", ("acyl", None), "B1", "B0"],     # two wraps and a constant same-body segment
    "t_tie": ["W2", ("wsph", None), "B2"],                 # ends and centre on one line at qA = qB = 0: the fallback plane, a tie
}


def wrap_xml():
    ten = ""
    for t, path in WRAP_TENDONS.items():
        el = "".join('<site site="%s"/>' % p if isinstance(p, str) else '<geom geom="%s"%s/>' % (p[0], ' sidesite="%s"' % p[1] if p[1] else "")
                     for p in path)
        ten += '<spatial name="%s">%s</spatial>' % (t, el)
    acts = "".join(_muscle("m_" + t, t, force=5) for t in WRAP_TENDONS)
    return ('<mujoco model="wrapzoo"><compiler angle="radian"/><option timestep="0.002"/><worldbody>'
            + _g("wsph", "sphere", "0.02", "-0.07 0.01 0") + _g("wcyl", "cylinder", "0.018 0.04", "0.02 -0.09 0", 'euler="0.2 0 0"')
            + '<site name="W0" pos="-0.16 0 0.02"/><site name="W1" pos="0.06 -0.17 -0.02"/><site name="W2" pos="-0.16 0.01 0"/>'
            '<site name="ws_out" pos="-0.07 0.05 0"/><site name="wc_out" pos="0.03 -0.09 0.031"/>'
            '<body name="A"><joint name="jA" axis="0 0 1" damping="0.02"/>' + _g("ca", "capsule", "0.01", extra='fromto="0 0 0 0.1 0 0"')
            + _g("asph", "sphere", "0.015", "0.07 0.012 0") + _g("acyl", "cylinder", "0.012 0.03", "0.02 0.06 0", 'euler="0 0.3 0"')
            + '<site name="A0" pos="0.05 0.035 0.01"/><site name="A1" pos="0.05 -0.035 0"/><site name="as_out" pos="0.07 0.04 0"/>'
            '<site name="as_in" pos="0.072 0.012 0.003"/><site name="ac_in" pos="0.02 0.063 0.002"/>'
            '<body name="B" pos="0.12 0 0"><joint name="jB" axis="0 0 1" damping="0.02"/>' + _g("cb", "capsule", "0.01", extra='fromto="0 0 0 0.08 0 0"')
            + '<site name="B0" pos="0.06 0.012 0.015"/><site name="B1" pos="0.05 -0.02 -0.01"/><site name="B2" pos="0 0.01 0"/>'
            '<body name="D" pos="0.09 0 0"><joint name="jD" axis="0 1 0"/>' + _g("cd", "capsule", "0.008", extra='fromto="0 0 0 0.05 0 0"')
            + '<site name="D0" pos="0.04 0.01 -0.01"/><site name="D1" pos="0.03 -0.01 0.012"/></body></body>'
            '<body name="C" pos="0 0.13 0"><joint name="jC" axis="0.3 0 1" damping="0.02"/>' + _g("cc", "capsule", "0.01", extra='fromto="0 0 0 0 0.08 0"')
            + '<site name="C0" pos="0.012 0.06 0.012"/><site name="C1" pos="-0.015 0.05 -0.008"/></body></body>'
            '</worldbody><tendon>%s</tendon><actuator>%s</actuator></mujoco>' % (ten, acts))


# MUSCLE: world site -> hinge A (z) -> hinge B (y) -> slide S (x); one straight tendon per muscle from a world site to a distal site
MUSCLES = [  # (end body, gear, parameters); the lengthrange is fitted to the configurations (fit_lengthranges)
    ("A", 1.0, dict(ctrllimited="true", ctrlrange="0.1 0.8", force=30)),
    ("B", 0.5, dict(ctrllimited="false", tausmooth="0.3", force=40, lmin="0.6", lmax="1.4", vmax="2", fpmax="1.1", fvmax="1.5")),
    ("S", 2.5, dict(ctrllimited="true", ctrlrange="-0.2 0.7", tausmooth="0.05", timeconst="0.02 0.06", force=20, range="0.6 1.2")),
    ("B", 1.0, dict(ctrllimited="false", tausmooth="1.2", timeconst="0.005 0.08", force=25, lmin="0.3", lmax="1.8", vmax="1",
                    fpmax="0.5", fvmax="1.9")),
    ("S", 0.5, dict(ctrllimited="true", ctrlrange="0.3 1", force=15, lmin="0.55", lmax="1.5", vmax="3", fpmax="2", fvmax="1.2")),
    ("A", 2.5, dict(ctrllimited="false", tausmooth="0.1", timeconst="0.015 0.03", force=35, range="0.8 1.1", fvmax="1.4")),
]
MUSCLE_SITES = {"A": "0.09 0.02 0.01", "B": "0.07 -0.02 0.015", "S": "0.05 0.015 -0.01"}


def muscle_xml(lrs):
    sites = "".join('<site name="w%d" pos="%s"/>' % (i, "-0.2 %g %g" % (0.03 * (i % 3 - 1), 0.02 * (i % 2))) for i in range(len(MUSCLES)))
    body_sites = {k: "".join('<site name="e%d" pos="%s"/>' % (i, MUSCLE_SITES[k]) for i, (b, _, _) in enumerate(MUSCLES) if b == k) for k in "ABS"}
    ten = "".join('<spatial name="t%d"><site site="w%d"/><site site="e%d"/></spatial>' % (i, i, i) for i in range(len(MUSCLES)))
    acts = "".join(_muscle("m%d" % i, "t%d" % i, lrs[i], gear=gear, **p) for i, (_, gear, p) in enumerate(MUSCLES))
    return ('<mujoco model="musclezoo"><compiler angle="radian"/><option timestep="0.002"/><worldbody>%s'
            '<body name="A"><joint name="jA" axis="0 0 1" damping="0.05"/>%s%s'
            '<body name="B" pos="0.1 0 0"><joint name="jB" axis="0 1 0"/>%s%s'
            '<body name="S" pos="0.08 0 0"><joint name="jS" type="slide" axis="1 0 0" damping="1"/>%s%s'
            '</body></body></body></worldbody><tendon>%s</tendon><actuator>%s</actuator></mujoco>'
            % (sites, _g("ga", "capsule", "0.015", extra='fromto="0 0 0 0.1 0 0"'), body_sites["A"],
               _g("gb", "capsule", "0.012", extra='fromto="0 0 0 0.08 0 0"'), body_sites["B"],
               _g("gs", "sphere", "0.02", "0.04 0 0"), body_sites["S"], ten, acts))


# LIM: root hinge j0 -> hinge j1 -> slide j2, and root -> hinge j3 -> slide j4.  Binary-exact ranges and margins so that the
# dist == margin and range == 2 margin poses are exact.
LIMITS = {   # joint: (type, range, margin, solref, solimp)
    "j0": ("hinge", (-0.5, 0.5), 0.0, (0.02, 1), (0.9, 0.95, 0.01, 0.5, 2)),
    "j1": ("hinge", (-0.25, 0.375), 0.0625, (0.03, 0.8), (0.8, 0.95, 0.01, 0.3, 1)),
    "j2": ("slide", (-0.015625, 0.03125), 0.03125, (0.02, 1.2), (0.85, 0.99, 0.01, 0.6, 2.5)),     # range < 2 margin: two rows
    "j3": ("hinge", (-0.25, 0.25), 0.25, (0.02, 1), (0.9, 0.9, 0.01, 0.5, 2)),                  # range == 2 margin; solimp[0] == solimp[1]
    "j4": ("slide", (-0.0625, 0.0625), 0.015625, (0.04, 0.7), (0.7, 0.98, 0.01, 0.4, 2.5)),
}
REFS = {"j0": 0.1, "j1": -0.05, "j2": 0.0, "j3": 0.07, "j4": 0.0}
EQS_TREE = [   # (joint1, joint2, polycoef, solref, solimp, active)
    ("j1", "j0", "0.01 0.5 -0.3 0.2 0.1", "0.02 1", "0.8 0.95 0.05 0.4 2", True),
    ("j2", "j1", "0.002 0.03 0.02 -0.01 0.01", "0.03 0.9", "0.85 0.97 0.02 0.5 2.5", True),
    ("j4", None, "0.004", "0.02 1", "0.7 0.9 0.01 0.3 1", True),
    ("j3", "j0", "0 1", "0.02 1", "0.9 0.95 0.01 0.5 2", False),
]
EQS_CROSS = EQS_TREE[:3] + [("j3", "j1", "-0.02 0.4 0.1 -0.1 0.05", "0.025 1", "0.75 0.96 0.05 0.5 2", True), EQS_TREE[3]]


def lim_xml(eqs):
    def jnt(n):
        t, r, mg, sr, si = LIMITS[n]
        ax = "0 0 1" if t == "hinge" else "1 0 0"
        return ('<joint name="%s" type="%s" axis="%s" range="%.17g %.17g" margin="%.17g" solreflimit="%g %g" solimplimit="%s" ref="%g" damping="0.01"/>'
                % (n, t, ax, r[0], r[1], mg, sr[0], sr[1], " ".join("%g" % v for v in si), REFS[n]))
    eq = "".join('<joint joint1="%s" %s polycoef="%s" solref="%s" solimp="%s" active="%s"/>'
                 % (a, 'joint2="%s"' % b if b else "", pc, sr, si, "true" if act else "false") for a, b, pc, sr, si, act in eqs)
    return ('<mujoco model="limzoo"><compiler angle="radian"/><option timestep="0.002"/><worldbody>'
            '<body name="b0" pos="0 0 0.5">%s%s<site name="ms0" pos="0 0 0.005"/><site name="ms1" pos="0 0 -0.005"/>'
            '<body name="b1" pos="0.1 0 0">%s%s<body name="b2" pos="0.08 0 0">%s%s</body></body>'
            '<body name="b3" pos="0 0.1 0">%s%s<body name="b4" pos="0 0.08 0">%s%s</body></body></body></worldbody>'
            '<tendon><spatial name="mt"><site site="ms0"/><site site="ms1"/></spatial></tendon>'
            '<actuator>%s</actuator><equality>%s</equality></mujoco>'
            % (jnt("j0"), _g("g0", "capsule", "0.01", extra='fromto="0 0 0 0.1 0 0"'), jnt("j1"), _g("g1", "capsule", "0.01", extra='fromto="0 0 0 0.08 0 0"'),
               jnt("j2"), _g("g2", "sphere", "0.02"), jnt("j3"), _g("g3", "capsule", "0.01", extra='fromto="0 0 0 0 0.08 0"'),
               jnt("j4"), _g("g4", "sphere", "0.015"), _muscle("m0", "mt", (0.005, 0.02)), eq))


def sweep_xml(nv):
    """A branched hinge tree of nv bodies (parent of body k: (k - 1) // 3), three limits, one parent-child equality and one capsule
    (on the deepest body) against a world plane."""
    bodies = {k: [] for k in range(-1, nv)}
    for k in range(nv):
        bodies[(k - 1) // 3 if k else -1].append(k)
    depth = {0: 0}
    for k in range(1, nv):
        depth[k] = depth[(k - 1) // 3] + 1
    deep = max(range(nv), key=lambda k: (depth[k], k))

    def body(k):
        ax = ["0 0 1", "0 1 0", "1 0 0"][k % 3]
        lim = ' range="-0.6 0.7" margin="0.02"' if k in (1, 2, nv - 1) else ""
        ang = 2 * np.pi * (k % 3) / 3
        pos = "0 0 0.8" if k == 0 else "%.6f %.6f -0.04" % (0.06 * np.cos(ang), 0.06 * np.sin(ang))
        geom = _g("cap", "capsule", "0.01 0.02", "0 0 -0.03") if k == deep else _g("g%d" % k, "sphere", "0.012")
        sites = '<site name="ms0" pos="0 0 0.005"/><site name="ms1" pos="0 0 -0.005"/>' if k == 0 else ""
        return '<body name="b%d" pos="%s"><joint name="j%d" axis="%s" damping="0.02"%s/>%s%s%s</body>' % (
            k, pos, k, ax, lim, geom, sites, "".join(body(c) for c in bodies[k]))
    plane_z = 0.8 - 0.04 * depth[deep] - 0.05
    return ('<mujoco model="sweep%d"><compiler angle="radian"/><option timestep="0.002"/><worldbody>%s%s</worldbody>'
            '<tendon><spatial name="mt"><site site="ms0"/><site site="ms1"/></spatial></tendon>'
            '<actuator>%s</actuator><equality><joint joint1="j1" joint2="j0" polycoef="0 0.5" solref="0.02 1" solimp="0.8 0.95 0.02 0.5 2"/></equality>'
            '<contact><pair geom1="floor" geom2="cap" condim="3" margin="0.005"/></contact></mujoco>'
            % (nv, _g("floor", "plane", "0 0 1", "0 0 %.6f" % plane_z), body(0), _muscle("m0", "mt", (0.005, 0.02))))


def compile_xml(xml, tmp, name):
    from myosuite_b200 import mjcf
    path = os.path.join(str(tmp), name + ".xml")
    with open(path, "w") as f:
        f.write(xml)
    return mjcf.compile_mjcf(path)


def oracle_of(m):
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    return Oracle(*blob.pack(m))


# ----------------------------------------------------------------------------- configurations
def wrap_configs(m):
    """qpos rows: a grid over the hinges plus poses chosen for single branches"""
    rng = np.random.default_rng(11)
    q = [rng.uniform(-1.6, 1.6, m.nq) for _ in range(40)]
    q += [np.array([a, b, c, d]) for a in (-0.6, 0.0, 0.7) for b in (-1.2, 0.0, 1.0) for c, d in ((0.0, 0.0), (0.9, -0.8))]
    # (jA, jB, jD, jC) found by a seeded search: an end inside the sphere of t_sph_side, inside-wrap exits without a Newton root
    q += [np.array(v) for v in ([2.2456, -2.9306, 1.443, -2.0379], [1.9683, 2.5934, 0.67, 1.442], [0.8761, -1.6907, -0.8808, 1.4008],
                                [-2.7318, -1.9224, 2.2218, 0.9031])]
    return np.array(q)


def muscle_configs(m):
    rng = np.random.default_rng(12)
    n = 96
    qpos = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(-1.2, 1.2, n), rng.uniform(-0.05, 0.05, n)], 1)
    qvel = rng.normal(0, 1, (n, 3)) * np.array([4.0, 4.0, 0.4])
    act = rng.uniform(-0.3, 1.3, (n, m.na))
    ctrl = rng.uniform(-0.5, 1.5, (n, m.nu))
    return qpos, qvel, act, ctrl


def fit_lengthranges(tmp):
    """Each muscle's lengthrange maps the configurations' actuator lengths onto normalised lengths from 0.2 to 2.2 (every force-length
    and passive piece)."""
    from myosuite_b200 import mjcf
    m = compile_xml(muscle_xml([(0.01, 1.0)] * len(MUSCLES)), tmp, "muscle_fit")
    qpos = muscle_configs(m)[0]
    lens = np.array([[m.actuator_gear[i, 0] * tendon_ref(m, mjcf.kinematics(m, q), i)[0] for i in range(m.nu)] for q in qpos])
    lrs = []
    for i in range(m.nu):
        r0, r1 = m.actuator_gainprm[i, :2]
        lo, hi = lens[:, i].min(), lens[:, i].max()
        L0 = (hi - lo) / 2.0                           # normalised L spans 2.0
        lr0 = lo - (0.2 - r0) * L0
        lrs.append((lr0, lr0 + L0 * (r1 - r0)))
    return lrs


def lim_configs(m):
    """Random poses with 10 % overshoot of every range, then poses for single branches: every limit 3 mm and 7 mm past margin (either
    side of solimp[3] with a 1 cm width), exactly at dist == margin, j2 inside both margins, j3 at the midpoint of a range 2 margin wide"""
    rng = np.random.default_rng(13)
    jn = list(LIMITS)
    out = []
    for _ in range(40):
        out.append(np.array([rng.uniform(LIMITS[j][1][0] - 0.1 * np.diff(LIMITS[j][1])[0], LIMITS[j][1][1] + 0.1 * np.diff(LIMITS[j][1])[0]) for j in jn]))
    mid = np.array([0.5 * sum(LIMITS[j][1]) for j in jn])
    for k, j in enumerate(jn):
        t, r, mg, _, _ = LIMITS[j]
        for pen in (0.003, 0.007):
            for side in (0, 1):
                q = mid.copy(); q[k] = r[0] + mg - pen if side == 0 else r[1] - mg + pen; out.append(q)
        q = mid.copy(); q[k] = r[0] + mg; out.append(q)          # dist == margin: inactive (strict <)
    q = mid.copy(); q[jn.index("j2")] = 0.0078125; out.append(q)
    q = mid.copy(); q[jn.index("j3")] = 0.0; out.append(q)
    return np.array(out)


def sweep_configs(m, n=24):
    rng = np.random.default_rng(100 + m.nv)
    return rng.uniform(-0.6, 0.6, (n, m.nq))


# ----------------------------------------------------------------------------- the zoo
def build_zoo(tmp, names=None):
    """{name: dict(m, prog, info, qpos, qvel, act, ctrl)}"""
    from myosuite_b200 import program
    zoo = {}
    specs = ["WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS"] + ["SWEEP_%d" % nv for nv in SWEEP_NV]
    for name in specs:
        if names is not None and name not in names:
            continue
        if name == "WRAP":
            m = compile_xml(wrap_xml(), tmp, name); qpos = wrap_configs(m)
        elif name == "MUSCLE":
            m = compile_xml(muscle_xml(fit_lengthranges(tmp)), tmp, name)
        elif name.startswith("LIM"):
            m = compile_xml(lim_xml(EQS_TREE if name == "LIM_TREE" else EQS_CROSS), tmp, name); qpos = lim_configs(m)
        else:
            m = compile_xml(sweep_xml(int(name.split("_")[1])), tmp, name); qpos = sweep_configs(m)
        rng = np.random.default_rng(7 + len(zoo))
        if name == "MUSCLE":
            qpos, qvel, act, ctrl = muscle_configs(m)
        else:
            n = len(qpos)
            qvel, act, ctrl = rng.normal(0, 0.5, (n, m.nv)), rng.uniform(0, 1, (n, m.na)), rng.uniform(0, 1, (n, m.nu))
        prog, info = program.build_program(m)
        zoo[name] = dict(m=m, prog=prog, info=info, qpos=qpos, qvel=qvel, act=act, ctrl=ctrl)
    return zoo


def wrap_branches(z):
    """[[per config: [(tendon, geom, side site, branch)]]] and the numpy tendon lengths [n, ntendon]"""
    from myosuite_b200 import mjcf
    m = z["m"]
    br, lens = [], []
    for q in z["qpos"]:
        kin = mjcf.kinematics(m, q)
        row, lrow = [], []
        for t in range(m.ntendon):
            L, b = tendon_ref(m, kin, t)
            lrow.append(L); row += [(t,) + x for x in b]
        br.append(row); lens.append(lrow)
    return br, np.array(lens)


def muscle_ref(m, length, vel, act, ctrl):
    """(actuator force, act_dot, pieces) of actuator i from the numpy references; length / vel are actuator (gear-scaled) values"""
    out = []
    for i in range(m.nu):
        c = ctrl[i]
        if m.actuator_ctrllimited[i]:
            c = min(max(c, m.actuator_ctrlrange[i, 0]), m.actuator_ctrlrange[i, 1])
        lr = m.actuator_lengthrange[i]
        gain, fl, fv = muscle_gain(length[i], vel[i], lr, m.actuator_gainprm[i])
        bias, fp = muscle_bias(length[i], lr, m.actuator_biasprm[i])
        out.append((gain * act[i] + bias, muscle_dynamics(c, act[i], m.actuator_dynprm[i]), (fl, fv, fp)))
    return out


# ----------------------------------------------------------------------------- CPU: coverage and the references against the oracle
WRAP_BRANCHES = {"out-wrap", "out-clear", "out-side-forced", "out-endpoint-inside", "out-tie-sph-collinear", "in-alhazen", "in-alhazen-sph",
                 "in-crosses", "in-endpoint-inside", "in-no-solution", "in-no-solution-sph"}
MUSCLE_PIECES = {"FL<lmin", "FL1", "FL2", "FL3", "FL4", "FL>lmax", "FV<=-1", "FV(-1,0]", "FV(0,y]", "FV>y", "FP<=1", "FP(1,b]", "FP>b"}


def test_actuation_zoo_coverage(tmp_path):
    """The zoo's programs and configurations reach every branch the module is meant to test (counted with the numpy references)."""
    from myosuite_b200 import program as P
    zoo = build_zoo(tmp_path)
    # wraps: all four classes, world / moving / endpoint-body geoms, and every branch
    z = zoo["WRAP"]; m, prog = z["m"], z["prog"]
    d = prog["P_dims"]
    assert min(d[P.PD_NWE_SPH_OUT], d[P.PD_NWE_SPH_IN], d[P.PD_NWE_CYL_OUT], d[P.PD_NWE_CYL_IN]) > 0
    gb = prog["PWE"][:, 2]
    assert (gb < 0).any() and (gb >= 0).any()
    same = [t for t, path in WRAP_TENDONS.items() if any(not isinstance(p, str) and m.body_weldid[m.geom_bodyid[m.name2id("geom", p[0])]]
                                                         == m.body_weldid[m.site_bodyid[m.name2id("site", path[k - 1])]] for k, p in enumerate(path))]
    assert "t_same" in same and len(prog["PT_const"]) == m.ntendon and np.count_nonzero(prog["PT_const"]) >= 1
    g, s = m.name2id("geom", "wcyl"), m.name2id("site", "wc_out")
    sl = mjmath_local(m, g, s)
    assert np.hypot(sl[0], sl[1]) < m.geom_size[g][0] <= np.linalg.norm(sl)
    br, _ = wrap_branches(z)
    seen = {}
    for row in br:
        for t, gg, ss, b in row:
            seen[b] = seen.get(b, 0) + 1
    print("\nwrap branches over %d configs: %s" % (len(br), dict(sorted(seen.items()))))
    assert WRAP_BRANCHES <= set(seen), WRAP_BRANCHES - set(seen)
    # muscles: tausmooth 0 and > 0, gear 0.5 / 1 / 2.5, ctrllimited both ways, ctrl outside [0, 1] and ctrlrange, act outside [0, 1], and
    # every curve piece
    z = zoo["MUSCLE"]; m = z["m"]
    assert {0.0} < set(m.actuator_dynprm[:, 2]) and set(m.actuator_gear[:, 0]) == {0.5, 1.0, 2.5} and set(m.actuator_ctrllimited) == {0, 1}
    assert len({tuple(r) for r in z["prog"]["PA_d"]}) == m.nu
    assert (z["act"] < 0).any() and (z["act"] > 1).any() and (z["ctrl"] < 0).any() and (z["ctrl"] > 1).any()
    lim = m.actuator_ctrllimited == 1
    assert ((z["ctrl"][:, lim] < m.actuator_ctrlrange[lim, 0]) & (z["ctrl"][:, lim] >= 0)).any()
    o = oracle_of(m); pieces = {}
    for e in range(len(z["qpos"])):
        o.reset(); o.set(qpos=z["qpos"][e], qvel=z["qvel"][e], act=z["act"][e], ctrl=z["ctrl"][e]); o.forward()
        for i, (_, _, pc) in enumerate(muscle_ref(m, o.f("actuator_length"), o.f("actuator_velocity"), z["act"][e], z["ctrl"][e])):
            for p in pc:
                pieces[p] = pieces.get(p, 0) + 1
    print("muscle curve pieces over %d configs x %d muscles: %s" % (len(z["qpos"]), m.nu, dict(sorted(pieces.items()))))
    assert MUSCLE_PIECES <= set(pieces), MUSCLE_PIECES - set(pieces)
    # limits / equalities
    lim_seen = dict(two=0, at_margin=0, below_mid=0, above_mid=0, margin_rows=0, eq_interp=0)
    powers_lim, powers_eq = set(), set()
    for name, tree in (("LIM_TREE", 1), ("LIM_CROSS", 0)):
        z = zoo[name]; m, prog = z["m"], z["prog"]
        assert prog["P_dims"][P.PD_EQ_TREE] == tree and prog["P_dims"][P.PD_NEQ] == int(m.eq_active0.sum()) == m.neq - 1
        assert prog["P_dims"][P.PD_NLIMROW] == 6 and (m.eq_data != 0).all(axis=1).any()
        assert (m.qpos0 != 0).sum() >= 3
        powers_lim |= {float(si[4]) for si in m.jnt_solimp[m.jnt_limited == 1]}
        powers_eq |= {float(si[4]) for si, a in zip(m.eq_solimp, m.eq_active0) if a and si[0] != si[1]}
        for q, v in zip(z["qpos"], z["qvel"]):
            rows = constraint_rows(m, q, v)
            assert len(rows) <= int(m.eq_active0.sum()) + prog["P_dims"][P.PD_NLIMROW]
            for j in range(m.njnt):
                r, mg = m.jnt_range[j], m.jnt_margin[j]
                dl, dh = q[j] - r[0], r[1] - q[j]
                lim_seen["two"] += dl < mg and dh < mg
                lim_seen["at_margin"] += dl == mg and mg > 0
                si = solparam(m.jnt_solimp[j])
                for dist in (dl, dh):
                    if dist < mg:
                        x = abs(dist - mg) / si[2]
                        lim_seen["margin_rows"] += mg > 0
                        lim_seen["below_mid"] += 0 < x <= si[3] and si[0] != si[1]
                        lim_seen["above_mid"] += si[3] < x < 1 and si[0] != si[1]
            for e in range(m.neq):
                if m.eq_active0[e]:
                    lim_seen["eq_interp"] += 0 < abs(constraint_pos(m, q, e)) < solparam(m.eq_solimp[e])[2]
    print("limits / equalities: %s, limit solimp powers %s, equality solimp powers %s" % (lim_seen, sorted(powers_lim), sorted(powers_eq)))
    assert min(lim_seen.values()) > 0 and powers_lim == {1.0, 2.0, 2.5} and powers_eq == {1.0, 2.0, 2.5}
    # size sweep
    contacts = {}
    for nv in SWEEP_NV:
        z = zoo["SWEEP_%d" % nv]; m = z["m"]
        assert m.nv == nv and m.npair == 1 and m.neq == 1 and z["prog"]["P_dims"][P.PD_EQ_TREE] == 1
        assert max(np.bincount(m.body_parentid[1:])) >= 2          # branched
        o = oracle_of(m); nc = 0
        for q in z["qpos"]:
            o.reset(); o.set(qpos=q); o.forward(); nc += o.ncon > 0
        contacts[nv] = nc
    print("sweep: configs with a contact per nv %s" % contacts)
    assert all(c > 0 for c in contacts.values()) and contacts[7] < len(zoo["SWEEP_7"]["qpos"])


def mjmath_local(m, g, s):
    """site s in the frame of geom g at qpos0"""
    from myosuite_b200 import mjcf, mjmath as mm
    kin = mjcf.kinematics(m, m.qpos0)
    b, bs = m.geom_bodyid[g], m.site_bodyid[s]
    gpos, gmat = kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g], kin["xmat"][b] @ mm.quat2mat(m.geom_quat[g])
    return gmat.T @ (kin["xpos"][bs] + kin["xmat"][bs] @ m.site_pos[s] - gpos)


def constraint_pos(m, q, e):
    j1, j2 = int(m.eq_obj1id[e]), int(m.eq_obj2id[e])
    pos = q[m.jnt_qposadr[j1]] - m.qpos0[m.jnt_qposadr[j1]]
    if j2 < 0:
        return pos - m.eq_data[e][0]
    x = q[m.jnt_qposadr[j2]] - m.qpos0[m.jnt_qposadr[j2]]
    return pos - sum(m.eq_data[e][k] * x ** k for k in range(5))


def test_references_match_oracle(tmp_path):
    """The numpy references against the oracle on every config: tendon and actuator lengths (wraps), actuator force and act_dot
    (muscles), the constraint rows and qacc as the exact Gauss minimiser (limits / equalities)."""
    from myosuite_b200 import mjcf
    zoo = build_zoo(tmp_path, ["WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS"])
    worst = {}
    z = zoo["WRAP"]; m = z["m"]; o = oracle_of(m)
    br, lens = wrap_branches(z)
    w = dict(out=0.0, inside=0.0)
    for e, q in enumerate(z["qpos"]):
        o.reset(); o.set(qpos=q); o.forward()
        tl = o.f("ten_length")
        for t in range(m.ntendon):
            kinds = [b for tt, _, _, b in br[e] if tt == t]
            r = abs(lens[e, t] - tl[t]) / tl[t]
            k = "inside" if any(b.startswith("in-") and b not in ("in-crosses", "in-endpoint-inside") for b in kinds) else "out"
            w[k] = max(w[k], r)
            assert r < (1e-11 if k == "inside" else 1e-13), (e, t, kinds, lens[e, t], tl[t])
    worst["WRAP tendon length"] = w
    z = zoo["MUSCLE"]; m = z["m"]; o = oracle_of(m); wf = wa = 0.0
    for e in range(len(z["qpos"])):
        o.reset(); o.set(qpos=z["qpos"][e], qvel=z["qvel"][e], act=z["act"][e], ctrl=z["ctrl"][e]); o.forward()
        kin = mjcf.kinematics(m, z["qpos"][e])
        ln = np.array([m.actuator_gear[i, 0] * tendon_ref(m, kin, i)[0] for i in range(m.nu)])
        np.testing.assert_allclose(ln, o.f("actuator_length"), rtol=1e-13)
        ref = muscle_ref(m, o.f("actuator_length"), o.f("actuator_velocity"), z["act"][e], z["ctrl"][e])
        f, ad = np.array([r[0] for r in ref]), np.array([r[1] for r in ref])
        wf, wa = max(wf, relerr(o.f("actuator_force"), f)), max(wa, relerr(o.f("act_dot"), ad))
        assert relerr(o.f("actuator_force"), f) < 1e-13 and relerr(o.f("act_dot"), ad) < 1e-13, e
    worst["MUSCLE force / act_dot"] = (wf, wa)
    for name in ("LIM_TREE", "LIM_CROSS"):
        z = zoo[name]; m = z["m"]; o = oracle_of(m); wq = 0.0
        for e, (q, v) in enumerate(zip(z["qpos"], z["qvel"])):
            o.reset(); o.set(qpos=q, qvel=v, act=z["act"][e], ctrl=z["ctrl"][e]); o.forward()
            rows = constraint_rows(m, q, v)
            assert o.nefc == len(rows), (name, e)
            np.testing.assert_allclose(o.f("efc_aref"), [r[1] for r in rows], rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(o.f("efc_D"), [r[2] for r in rows], rtol=1e-12)
            M = mjcf.mass_matrix(m, mjcf.kinematics(m, q))
            a = gauss_qacc(M, np.linalg.solve(M, o.f("qfrc_smooth")), rows)
            r = relerr(o.f("qacc"), a); wq = max(wq, r)
            assert r < 1e-9, (name, e, r)
        worst["%s qacc" % name] = wq
    print("\nnumpy references vs oracle, worst: %s" % worst)


# ----------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def zoo(tmp_path_factory):
    z = build_zoo(tmp_path_factory.mktemp("actzoo"))
    yield z
    if REPORT:
        print("\nactuation zoo vs references and oracle:")
        for k in sorted(REPORT):
            print("  %-24s %s" % (k, REPORT[k]))


MODELS = ["WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS"] + ["SWEEP_%d" % nv for nv in SWEEP_NV]
FD_MODELS = ("WRAP", "MUSCLE")


def _numpy_lengths(z):
    """numpy actuator lengths [n, nu] and, per config, whether the moment is defined there (no tie, no branch change within +-FD_H)"""
    from myosuite_b200 import mjcf
    m = z["m"]
    out, smooth = [], []
    for q in z["qpos"]:
        rows = [[tendon_ref(m, mjcf.kinematics(m, q + s * FD_H * np.eye(m.nq)[d]), int(m.actuator_trnid[i, 0])) for i in range(m.nu)]
                for d in range(m.nv) for s in (-1, 1)]
        c = [tendon_ref(m, mjcf.kinematics(m, q), int(m.actuator_trnid[i, 0])) for i in range(m.nu)]
        out.append([m.actuator_gear[i, 0] * c[i][0] for i in range(m.nu)])
        brs = [[b for _, _, b in x[1]] for x in c]
        # at a tie the moment is discontinuous: only length and finiteness are compared there.  At the inverse wrap's no-solution exit the
        # touching point (the ends' midpoint direction) is not a stationary point of the path length, so the moment that the kernel and
        # MuJoCo form from the two straight pieces is not the length's derivative there: compared with the oracle only.
        smooth.append(all(not any("tie" in b or "no-solution" in b for b in bb) for bb in brs) and all([[b for _, _, b in x[1]] for x in r] == brs for r in rows))
    return np.array(out), np.array(smooth)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", MODELS)
def test_zoo_forward_and_rollout(zoo, name, rows):
    """One forward pass with taps on every config (actuator length and force against the numpy references and the oracle, tendon moments
    against the oracle's ten_J and a central difference of the kernel's own lengths, qfrc_smooth, nefc and qacc; qacc of the limit models
    also against the exact Gauss minimiser), then 10 chained substeps (qpos, qvel, act) against the oracle with warm-started inverse
    wraps."""
    import torch
    from myosuite_b200 import mjcf, vec_env
    z = zoo[name]; m = z["m"]
    qpos, qvel, act, ctrl = z["qpos"], z["qvel"], z["act"], z["ctrl"]
    n = len(qpos)
    fd = name in FD_MODELS
    qa = qpos
    if fd:      # extra envs at q +- h e_d for the central difference of the lengths
        qa = np.concatenate([qpos] + [qpos + s * FD_H * np.eye(m.nq)[d] for d in range(m.nv) for s in (-1, 1)])
    N = len(qa)
    rep = lambda x: np.concatenate([x] * (N // n))
    env = vec_env.MyoVecEnv(None, N, model=m, taps=True, row_storage=rows)
    env.set_state(qpos=qa, qvel=rep(qvel), act=rep(act)); env.forward_debug(rep(ctrl), 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_")}
    prog, info = env.prog, env.prog_info
    ten_of = [info["act_tendons"][k] for k in prog["PNZ_tendon"]]
    nzd = prog["PNZ_dof"]
    gear = m.actuator_gear[:, 0]
    nl, smooth = _numpy_lengths(z) if name in ("WRAP", "MUSCLE") else (None, None)
    o = oracle_of(m)
    worst = dict(len=0.0, len_np=0.0, force=0.0, force_np=0.0, mom=0.0, fd=0.0, smooth=0.0, qacc=0.0, gauss=0.0)
    for e in range(n):
        msg = "%s[%s] config %d" % (name, rows, e)
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        for k in ("tap_qacc", "tap_actuator_force", "tap_ten_length", "tap_qfrc_smooth", "tap_moment"):
            assert np.isfinite(t[k][e]).all(), msg + " " + k
        assert t["tap_ncon"][e, 1] == o.nefc and t["tap_ncon"][e, 0] == o.ncon, msg
        r = relerr(t["tap_ten_length"][e], o.f("actuator_length")); worst["len"] = max(worst["len"], r); assert r < REL, msg + ": length %.2e" % r
        r = relerr(t["tap_actuator_force"][e], o.f("actuator_force")); worst["force"] = max(worst["force"], r); assert r < REL, msg + ": force %.2e" % r
        if nl is not None:
            r = relerr(t["tap_ten_length"][e], nl[e]); worst["len_np"] = max(worst["len_np"], r)
            assert r < (1e-11 if name == "WRAP" else REL), msg + ": length vs numpy %.2e" % r
        if name == "MUSCLE":
            ref = np.array([x[0] for x in muscle_ref(m, o.f("actuator_length"), o.f("actuator_velocity"), act[e], ctrl[e])])
            r = relerr(t["tap_actuator_force"][e], ref); worst["force_np"] = max(worst["force_np"], r); assert r < REL, msg + ": force vs numpy %.2e" % r
        J = o.f("ten_J").reshape(m.ntendon, m.nv)
        mom = np.zeros_like(J); mom[ten_of, nzd] = t["tap_moment"][e][:len(nzd)]
        r = float(np.abs(mom - J).max() / max(1e-12, np.abs(J).max())); worst["mom"] = max(worst["mom"], r)
        assert r < REL, msg + ": moment %.2e" % r
        if fd and smooth[e]:
            L = t["tap_ten_length"]
            for d in range(m.nv):
                lm, lp = L[n * (1 + 2 * d) + e], L[n * (2 + 2 * d) + e]
                fdm = (lp - lm) / (2 * FD_H) / gear
                got = np.array([mom[int(m.actuator_trnid[i, 0]), d] for i in range(m.nu)])
                worst["fd"] = max(worst["fd"], float(np.abs(fdm - got).max()))
                np.testing.assert_allclose(got, fdm, rtol=0, atol=1e-7, err_msg=msg + " dof %d" % d)
        r = relerr(t["tap_qfrc_smooth"][e], o.f("qfrc_smooth")); worst["smooth"] = max(worst["smooth"], r); assert r < 1e-10, msg + ": qfrc_smooth %.2e" % r
        r = relerr(t["tap_qacc"][e], o.f("qacc")); worst["qacc"] = max(worst["qacc"], r); assert r < FWD_QACC, msg + ": qacc %.2e" % r
        if name.startswith("LIM"):
            M = mjcf.mass_matrix(m, mjcf.kinematics(m, qpos[e]))
            a = gauss_qacc(M, np.linalg.solve(M, o.f("qfrc_smooth")), constraint_rows(m, qpos[e], qvel[e]))
            r = relerr(t["tap_qacc"][e], a); worst["gauss"] = max(worst["gauss"], r); assert r < FWD_QACC, msg + ": qacc vs Gauss minimiser %.2e" % r
    # 10 chained substeps on a fresh batch (inverse wraps start cold, as the oracle's)
    env = vec_env.MyoVecEnv(None, n, model=m, taps=True, row_storage=rows)
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 10); torch.cuda.synchronize()
    gq, gv, ga = (env.t[k].cpu().numpy() for k in ("qpos", "qvel", "act"))
    assert np.isfinite(gq).all() and np.isfinite(gv).all() and np.isfinite(ga).all()
    wq = wv = wa = 0.0
    for e in range(n):
        msg = "%s[%s] config %d, 10 substeps" % (name, rows, e)
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.f("wrap_warm")[:] = 1; o.step(10)
        wq, wv = max(wq, float(np.abs(gq[e] - o.f("qpos")).max())), max(wv, relerr(gv[e], o.f("qvel")))
        wa = max(wa, float(np.abs(ga[e, :m.na] - o.f("act")).max()))
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=ROLL_QPOS, err_msg=msg)
        assert relerr(gv[e], o.f("qvel")) < ROLL_QVEL, msg
        np.testing.assert_allclose(ga[e, :m.na], o.f("act"), rtol=0, atol=1e-12, err_msg=msg)
    REPORT["%s[%s]" % (name, rows)] = ("%d configs%s; worst length %.1e (numpy %.1e), force %.1e (numpy %.1e), moment %.1e (FD %.1e), "
                                       "qfrc_smooth %.1e, qacc %.1e (Gauss %.1e); 10 substeps qpos %.1e qvel %.1e act %.1e"
                                       % (n, " (%d with FD moments)" % int(smooth.sum()) if fd else "", worst["len"], worst["len_np"],
                                          worst["force"], worst["force_np"], worst["mom"], worst["fd"], worst["smooth"], worst["qacc"],
                                          worst["gauss"], wq, wv, wa))
    print(REPORT["%s[%s]" % (name, rows)])


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", MODELS)
def test_zoo_product_step(zoo, name, rows):
    """The same states through env.step on a batch without taps, so that a product kernel runs, against oracle.step(frame_skip)."""
    import torch
    from myosuite_b200 import vec_env
    from oracle import env_oracle
    z = zoo[name]; m = z["m"]
    qpos, qvel, act = z["qpos"], z["qvel"], z["act"]
    n = len(qpos)
    env = vec_env.MyoVecEnv(None, n, model=m, row_storage=rows)
    assert not any(k.startswith("tap_") for k in env.t)
    li = env.batch.launch_info()
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    a = np.random.default_rng(8).uniform(-1, 1, (n, m.nu)).astype(np.float32)
    env.step(torch.as_tensor(a, device=env.device)); torch.cuda.synchronize()
    S = env.get_env_state()
    o = oracle_of(m); worst = dict(qpos=0.0, qvel=0.0, qacc=0.0)
    for e in range(n):
        msg = "%s[%s] config %d, product step" % (name, rows, e)
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=env_oracle.action_to_ctrl(a[e].astype(np.float64)))
        o.f("wrap_warm")[:] = 1
        o.step(env.n_frames)
        assert np.isfinite(S["qpos"][e]).all() and np.isfinite(S["qacc_warmstart"][e]).all(), msg
        worst["qpos"] = max(worst["qpos"], float(np.abs(S["qpos"][e] - o.f("qpos")).max()))
        worst["qvel"] = max(worst["qvel"], relerr(S["qvel"][e], o.f("qvel"))); worst["qacc"] = max(worst["qacc"], relerr(S["qacc_warmstart"][e], o.f("qacc")))
        np.testing.assert_allclose(S["qpos"][e], o.f("qpos"), rtol=0, atol=MID["qpos"], err_msg=msg)
        assert relerr(S["qvel"][e], o.f("qvel")) < MID["qvel"], msg
        assert relerr(S["qacc_warmstart"][e], o.f("qacc")) < MID["qacc"], msg
        np.testing.assert_allclose(S["act"][e][:m.na], o.f("act"), rtol=0, atol=1e-12, err_msg=msg)
    REPORT["%s[%s] product" % (name, rows)] = ("%s kernel, %d warps/CTA, grid %d; %d configs, %d substeps; worst qpos %.1e qvel %.1e qacc %.1e"
                                               % ("w14" if li["use_w14"] else "k320", li["warps_per_cta"], li["grid"], n, env.n_frames,
                                                  worst["qpos"], worst["qvel"], worst["qacc"]))
    print(REPORT["%s[%s] product" % (name, rows)])
