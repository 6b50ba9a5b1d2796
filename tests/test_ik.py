"""Inverse kinematics and site Jacobians (myo_batch_ik, MyoVecEnv.ik / jac_site, MyoEnv.mj_ik / mj_jacSite) against the CPU reference
tests/ik_oracle.c: mj_jacSite through the oracle's cdof and oracle_ik, the iteration of include/myo_b200.h restated on dense matrices.

CPU: the header matches abi.py; oracle_jac_site against central differences of the oracle's site pose; one oracle_ik iteration against a
numpy solve of the stated normal equations; properties and convergence rates of oracle_ik at the defaults (DESIGN.md section 2).
GPU: jac_site and the iterations against the oracle on every base task at reached states; convergence at the defaults equal to the
CPU reference's; properties; no side effects; batch and library independence; input checks; the single env."""
import ctypes
import os

import numpy as np
import pytest

from ik_oracle import DEFAULTS, IkOracle
from test_mj_data import CASES, ROWS, SEED, _header_struct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIPPED = ["myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso"]
TIPS = ["THtip", "IFtip", "MFtip", "RFtip", "LFtip"]
JAC_REL = 1e-12            # jac_site against the oracle, relative to the env's largest entry; site_xmat and site_xpos absolute
ITER_TOL = 1e-10           # qpos and err after K iterations against oracle_ik (tol = 0): worst measured 1.5e-12 (hold, orientation
                           # targets, K = 10) on an H100 80GB HBM3; the bound leaves room for more iterations' growth
REPORT = {}


def _setup(m):
    from myosuite_b200 import blob, program
    prog, _ = program.build_program(m)
    I, D = blob.pack(m, prog)
    return IkOracle(I, D, m.site_quat)


def _random_q(m, rng, n=None):
    """in-range random hinge and slide joints, free joints at qpos0"""
    q = np.tile(m.qpos0, (n or 1, 1))
    for j in range(m.njnt):
        if m.jnt_type[j] in (2, 3):
            lo, hi = m.jnt_range[j] if m.jnt_limited[j] else (-1.0, 1.0)
            q[:, m.jnt_qposadr[j]] = rng.uniform(lo, hi, n or 1)
    return q if n else q[0]


def _worst(a, b):
    """the larger of a and b, NaN if either is (the builtin max drops a NaN second argument)"""
    return float(np.max([a, b]))


def _sites(m):
    names = {k for k in m.names["site"]}
    for group in (TIPS + ["S_grasp", "object"], ["pelvis", "toe_r", "toe_l"], ["wrist"]):
        got = [m.name2id("site", s) for s in group if s in names]
        if got:
            return got
    return [0, m.nsite // 3, 2 * m.nsite // 3, m.nsite - 1]


# ----------------------------------------------------------------------------- CPU
def test_ik_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_ik_buffers")
    assert len(fields) == decls and abi.IK_FIELDS == fields
    assert [n for n, _ in abi.MyoIkBuffers._fields_] == fields and ctypes.sizeof(abi.MyoIkBuffers) == 8 * len(fields)
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    body = src[:src.index("} myo_ik_params;")]
    body = body[body.rindex("typedef struct {"):]
    import re
    names = re.findall(r"(\w+)\s*[,;]", re.sub(r"(int32_t|double)", "", body.split("{", 1)[1]))
    assert names == [n for n, _ in abi.MyoIkParams._fields_] == ["nsite", "max_iter", "tol", "damping", "max_step", "posture_weight", "eq_weight"]
    assert src.index("} myo_rollout_buffers;") < src.index("} myo_ik_buffers;") < src.index("} myo_ik_params;") < src.index("int myo_batch_ik(")
    assert "#define MYO_IK_MAXSITE %d" % abi.IK_MAXSITE in src and "myo_batch_ik" in abi.EXPORTS


def _sweeps(tmp):
    import test_actuation_zoo as AZ
    return {k: v["m"] for k, v in AZ.build_zoo(tmp, names=["SWEEP_%d" % nv for nv in AZ.SWEEP_NV]).items()}


def _fd_jac(o, site, q, m, h=1e-6):
    """central differences of the site position and rotation through q (+) h e_i"""
    nv = m.nv
    jp, jr = np.zeros((3, nv)), np.zeros((3, nv))
    for i in range(nv):
        out = []
        for sg in (1, -1):
            o.set(qpos=q)
            dq = np.zeros(nv); dq[i] = sg * h
            qq = _integrate(m, q, dq)
            _, _, p, R = o.jac_site(site, qq)
            out.append((p, R.reshape(3, 3)))
        jp[:, i] = (out[0][0] - out[1][0]) / (2 * h)
        _, _, _, R0 = o.jac_site(site, q)
        W = (out[0][1] - out[1][1]) / (2 * h) @ R0.reshape(3, 3).T            # skew(omega) = dR R'

        jr[:, i] = [W[2, 1], W[0, 2], W[1, 0]]
    return jp, jr


def _integrate(m, q, dq):
    from myosuite_b200 import mjmath as mm
    q = q.copy()
    for j in range(m.njnt):
        qa, da = m.jnt_qposadr[j], m.jnt_dofadr[j]
        if m.jnt_type[j] == 0:
            q[qa:qa + 3] += dq[da:da + 3]
            w = dq[da + 3:da + 6]; a = np.linalg.norm(w)
            ql = np.array([1.0, 0, 0, 0]) if a == 0 else np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * w / a])
            qn = mm.quat_mul(q[qa + 3:qa + 7], ql)
            q[qa + 3:qa + 7] = qn / np.linalg.norm(qn)
        else:
            q[qa] += dq[da]
    return q


def test_oracle_jac_site_finite_differences(models, tmp_path):
    """oracle_jac_site against central differences of the oracle's own site pose at random in-range q, on the shipped models (hinge
    columns; the hold object's and the legs' pelvis free joints) and the actuation zoo's SWEEP models.  Bound 1e-8: 13x the worst measured
    (7.6e-10, the truncation and cancellation error of the h = 1e-6 central difference)."""
    rng = np.random.default_rng(SEED)
    all_models = dict(models); all_models.update(_sweeps(str(tmp_path)))
    worst, free = 0.0, set()
    for name, m in all_models.items():
        o = _setup(m)
        sites = (_sites(m)[:3] if name in SHIPPED else [m.nsite - 1]) + ([m.name2id("site", "object")] if name == "myohand_hold" else [])
        for _ in range(2):
            q = _random_q(m, rng)
            for s in sites:
                jp, jr, _, _ = o.jac_site(s, q)
                fp, fr = _fd_jac(o, s, q, m)
                scale = max(np.abs(jp).max(), np.abs(jr).max(), 1e-300)
                worst = _worst(worst, max(np.abs(jp - fp).max(), np.abs(jr - fr).max()) / scale)
                if any(m.jnt_type[m.dof_jntid[d]] == 0 and jp[:, d].any() for d in range(m.nv)):
                    free.add(name)
    REPORT["jac_site_fd"] = "central differences (h = 1e-6), worst %.1e relative" % worst
    print("\noracle_jac_site vs central differences: worst relative %.1e over %d models, free-joint columns on %s" % (worst, len(all_models), sorted(free)))
    assert free == {"myohand_hold", "myolegs"} and worst < 1e-8, (worst, free)


def _numpy_step(o, m, sites, tp, q0, mask=None, tq=None, qref=None, **p):
    """one iteration of the stated semantics in numpy, from the oracle's Jacobians; the rotation error log(mat(Q) R') through scipy"""
    from scipy.spatial.transform import Rotation
    p = dict(DEFAULTS, **p)
    nv = m.nv
    H, g = np.zeros((nv, nv)), np.zeros(nv)
    for k, (s, t) in enumerate(zip(sites, tp)):
        jp, jr, x, R = o.jac_site(s, q0)
        H += jp.T @ jp; g += jp.T @ (t - x)
        if tq is not None:
            Q = tq[k] / np.linalg.norm(tq[k])
            w = Rotation.from_matrix(Rotation.from_quat(np.r_[Q[1:], Q[0]]).as_matrix() @ R.reshape(3, 3).T).as_rotvec()
            H += jr.T @ jr; g += jr.T @ w
    for e in range(m.neq):
        j1, j2, c = m.eq_obj1id[e], m.eq_obj2id[e], m.eq_data[e]
        row = np.zeros(nv); row[m.jnt_dofadr[j1]] = 1
        res = q0[m.jnt_qposadr[j1]] - m.qpos0[m.jnt_qposadr[j1]]
        if j2 < 0:
            res -= c[0]
        else:
            x = q0[m.jnt_qposadr[j2]] - m.qpos0[m.jnt_qposadr[j2]]
            res -= c[0] + c[1] * x + c[2] * x**2 + c[3] * x**3 + c[4] * x**4
            row[m.jnt_dofadr[j2]] = -(c[1] + 2 * c[2] * x + 3 * c[3] * x**2 + 4 * c[4] * x**3)
        H += p["eq_weight"] * np.outer(row, row); g -= p["eq_weight"] * row * res
    for j in range(m.njnt):
        if m.jnt_type[j] in (2, 3):
            d, qa = m.jnt_dofadr[j], m.jnt_qposadr[j]; H[d, d] += p["posture"]
            g[d] += p["posture"] * ((q0 if qref is None else qref)[qa] - q0[qa])
    H += p["damping"] * np.eye(nv)
    if mask is not None:
        for i in np.where(~mask)[0]:
            H[i, :] = 0; H[:, i] = 0; H[i, i] = 1; g[i] = 0
    dq = np.linalg.solve(H, g)
    if np.linalg.norm(dq) > p["max_step"]:
        dq *= p["max_step"] / np.linalg.norm(dq)
    q = _integrate(m, q0, dq)
    for j in range(m.njnt):
        if m.jnt_limited[j] and m.jnt_type[j] in (2, 3):
            q[m.jnt_qposadr[j]] = np.clip(q[m.jnt_qposadr[j]], *m.jnt_range[j])
    return q


def test_oracle_ik_one_iteration_matches_numpy(models):
    """one oracle_ik iteration equals the numpy solve of the stated H dq = g: position targets, the dof mask, the step cap, orientation
    targets (scipy's rotation log), the posture term toward a reference, the joint equalities, and the range clamp throughout"""
    rng = np.random.default_rng(SEED)
    worst = 0.0
    for name in SHIPPED:
        m = models[name]; o = _setup(m); sites = _sites(m)
        for trial in range(5):
            q0 = _random_q(m, rng); tp = np.array([o.jac_site(s, _random_q(m, rng))[2] for s in sites])
            mask = rng.uniform(size=m.nv) < 0.7 if trial == 1 else None
            step = 0.05 if trial == 2 else DEFAULTS["max_step"]
            tq = rng.normal(size=(len(sites), 4)) if trial == 3 else None
            qref, rho = (_random_q(m, rng), 0.3) if trial == 4 else (None, 0.0)
            ref = _numpy_step(o, m, sites, tp, q0, mask=mask, tq=tq, qref=qref, max_step=step, posture=rho)
            r = o.ik(sites, tp, q0, target_quat=tq, qpos_ref=qref, dof_mask=mask, max_iter=1, tol=0.0, max_step=step, posture=rho)
            assert r["niter"] == 1
            worst = _worst(worst, np.abs(r["qpos"] - ref).max())
    print("\none oracle_ik iteration vs numpy: worst %.1e" % worst)
    assert worst <= 1e-12, worst


def test_oracle_ik_properties(models):
    rng = np.random.default_rng(SEED + 1)
    for name in SHIPPED:
        m = models[name]; o = _setup(m); sites = _sites(m)
        q0 = _random_q(m, rng); tp = np.array([o.jac_site(s, _random_q(m, rng))[2] for s in sites]) + 0.05
        r0 = o.ik(sites, tp, q0, max_iter=0)
        assert r0["niter"] == 0 and np.array_equal(r0["qpos"], q0)
        mask = rng.uniform(size=m.nv) < 0.5
        r = o.ik(sites, tp, q0, dof_mask=mask, max_iter=20, tol=0.0)
        for j in range(m.njnt):
            qa, da = m.jnt_qposadr[j], m.jnt_dofadr[j]
            if m.jnt_type[j] == 0:
                assert abs(np.linalg.norm(r["qpos"][qa + 3:qa + 7]) - 1) < 1e-14
            elif not mask[da]:
                assert r["qpos"][qa] == q0[qa]
            if m.jnt_limited[j] and m.jnt_type[j] in (2, 3):
                assert m.jnt_range[j, 0] <= r["qpos"][qa] <= m.jnt_range[j, 1]


CONV = {"myohand_pose": TIPS, "myolegs": ["pelvis", "toe_r", "toe_l"], "myoelbow_1dof6muscles": ["wrist"]}


def test_oracle_ik_convergence(models):
    """oracle_ik at the defaults, targets from forward kinematics of random in-range configurations, start at qpos0 (init_qpos of
    these tasks): the converged fraction and worst error the GPU test reproduces (DESIGN.md section 2).  Each miss is also continued
    for 800 more iterations from where it stopped, and its joints pinned at a range end are counted: that separates iteration budget
    from stalls against the clamp."""
    rng = np.random.default_rng(SEED)
    lim_of = lambda m: np.where(m.jnt_limited.astype(bool) & (m.jnt_type >= 2))[0]
    for name, sn in CONV.items():
        m = models[name]; o = _setup(m); sites = [m.name2id("site", s) for s in sn]
        conv, worst, eqr, miss = [], 0.0, 0.0, []
        for _ in range(40):
            qt = _random_q(m, rng)
            tp = np.array([o.jac_site(s, qt)[2] for s in sites])
            r = o.ik(sites, tp, m.qpos0)
            conv.append(r["converged"]); worst = _worst(worst, r["err"][:, 0].max())
            if not r["converged"]:
                pinned = sum(r["qpos"][m.jnt_qposadr[j]] in tuple(m.jnt_range[j]) for j in lim_of(m))
                more = o.ik(sites, tp, r["qpos"], max_iter=800)
                miss.append((r["niter"] == DEFAULTS["max_iter"], pinned > 0, more["converged"]))
            for e in range(m.neq):
                q = r["qpos"]; j1, j2, c = m.eq_obj1id[e], m.eq_obj2id[e], m.eq_data[e]
                x = q[m.jnt_qposadr[j2]] - m.qpos0[m.jnt_qposadr[j2]]
                eqr = _worst(eqr, abs(q[m.jnt_qposadr[j1]] - m.qpos0[m.jnt_qposadr[j1]] - np.polyval(c[::-1], x)))
        mm = np.array(miss, float).reshape(-1, 3)
        REPORT["conv_" + name] = ("converged %.2f, worst error %.1e m, equality residual %.1e; of %d misses: %.2f at max_iter, %.2f with a joint "
                                  "at a range end, %.2f converge within 800 more iterations" % (np.mean(conv), worst, eqr, len(mm), *(mm.mean(0) if len(mm) else (0, 0, 0))))
        print("\n%s: %s" % (name, REPORT["conv_" + name]))
        if name == "myoelbow_1dof6muscles":
            assert np.mean(conv) == 1.0
        assert len(mm) == 0 or mm[:, 0].all()      # a miss always spends the whole budget: no early exit without convergence


# ----------------------------------------------------------------------------- GPU
def _warm(case, rows="p48", n=None):
    import torch
    from myosuite_b200 import vec_env
    eid, n0 = CASES[case]
    env = vec_env.MyoVecEnv(eid, n or n0, seed=SEED, row_storage=rows)
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(6):
        env.step((torch.rand(env.num_envs, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
    return env


def _checked(n):
    return sorted(set(range(0, n, 16)) | set(range(min(n, 32))))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_jac_site_vs_oracle(case):
    import torch
    env = _warm(case); m = env.mj_model; sites = _sites(m)
    jp, jr, xp, xm = (x.cpu().numpy() for x in env.jac_site(sites))
    ref_xpos = env.data("site_xpos")["site_xpos"].cpu().numpy()
    torch.cuda.synchronize()
    q = env.t["qpos"].cpu().numpy()
    assert all(np.isfinite(x).all() for x in (jp, jr, xp, xm))      # every output of every env written (they start as NaN)
    o = _setup(m)
    WJ, WX, WP = [], [], []
    for e in _checked(env.num_envs):
        ref = [o.jac_site(s, q[e]) for s in sites]
        scale = max(max(np.abs(rp).max(), np.abs(rr).max()) for rp, rr, _, _ in ref)      # the env's largest entry (a site on a static body: all 0)
        for k, (s, (rp, rr, p, R)) in enumerate(zip(sites, ref)):
            WJ.append(max(np.abs(jp[e, k] - rp).max(), np.abs(jr[e, k] - rr).max()) / scale)
            WX.append(np.abs(xm[e, k] - R).max())
            WP.append(np.abs(xp[e, k] - ref_xpos[e, s]).max())
    wj, wx, wp = (float(np.max(x)) for x in (WJ, WX, WP))      # (np.max propagates NaN, unlike the builtin max)
    REPORT["jac_" + case] = "jac %.1e rel, site_xmat %.1e, site_xpos vs readout %.1e" % (wj, wx, wp)
    print("\n%s: %s" % (case, REPORT["jac_" + case]))
    assert wj <= JAC_REL and wx <= 1e-12 and wp <= 1e-12, (wj, wx, wp)


IK_CASES = {"pos": {}, "pos_rot": {"rot": True}, "posture": {"posture": 0.1}, "mask": {"mask": True}, "eq": {"eq_weight": 10.0}}


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3, 10])
@pytest.mark.parametrize("kind", list(IK_CASES))
@pytest.mark.parametrize("case", list(CASES))
def test_ik_iterations_vs_oracle(case, kind, K):
    """K iterations with tol = 0 against oracle_ik per env: niter equal, qpos and err within ITER_TOL (worst measured in DESIGN.md)"""
    import torch
    spec = IK_CASES[kind]
    env = _warm(case, n=256); m = env.mj_model; sites = _sites(m); n, ns = env.num_envs, len(sites)
    if kind == "eq" and m.neq == 0:
        pytest.skip("no joint equalities")
    rng = np.random.default_rng(SEED + K)
    q = env.t["qpos"].cpu().numpy()
    o = _setup(m)
    tp = np.stack([[o.jac_site(s, _random_q(m, rng))[2] for s in sites] for _ in range(n)])
    tq = None
    if spec.get("rot"):
        tq = rng.normal(size=(n, ns, 4))
    mask = rng.uniform(size=m.nv) < 0.6 if spec.get("mask") else None
    ref = np.tile(m.qpos0, (n, 1)) if spec.get("posture") else None
    dev = lambda x: None if x is None else torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=env.device)
    params = dict(max_iter=K, tol=0.0, posture=spec.get("posture", 0.0), eq_weight=spec.get("eq_weight", DEFAULTS["eq_weight"]))
    r = env.ik(sites, dev(tp), target_quat=dev(tq), qpos_ref=dev(ref), dofs=mask, fields=("qpos", "niter", "converged", "err"), **params)
    R = {k: v.cpu().numpy() for k, v in r.items()}
    assert np.isfinite(R["qpos"]).all() and np.isfinite(R["err"]).all() and (R["niter"] >= 0).all() and (R["converged"] >= 0).all()
    WQ, WE = [], []
    for e in _checked(n):
        out = o.ik(sites, tp[e], q[e], target_quat=None if tq is None else tq[e], qpos_ref=None if ref is None else ref[e], dof_mask=mask, **params)
        # equal niter, except where the reference reached err = 0 exactly (the elbow's one dof): tol = 0 is then round-off away
        assert R["niter"][e] == out["niter"] == K or (out["converged"] and R["niter"][e] >= out["niter"]), (e, R["niter"][e], out["niter"])
        WQ.append(np.abs(R["qpos"][e] - out["qpos"]).max()); WE.append(np.abs(R["err"][e] - out["err"]).max())
    wq, we = float(np.max(WQ)), float(np.max(WE))
    key = "iter_%s_%s_%d" % (case, kind, K)
    REPORT[key] = "qpos %.1e, err %.1e" % (wq, we)
    print("\n%s: %s" % (key, REPORT[key]))
    assert wq <= ITER_TOL and we <= ITER_TOL, (wq, we)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", [("myohand_pose", 4096), ("myolegs", 2048)])
def test_convergence_matches_cpu(name, n):
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv.from_model(name, n)
    m = env.mj_model; sites = [m.name2id("site", s) for s in CONV[name]]
    rng = np.random.default_rng(SEED)
    qt = _random_q(m, rng, n)
    dev = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=env.device)
    tp = env.jac_site(sites, qpos=dev(qt))[2].contiguous()
    r = env.ik(sites, tp, qpos_init=dev(np.tile(m.qpos0, (n, 1))))
    R = {k: v.cpu().numpy() for k, v in r.items()}
    TP = tp.cpu().numpy()
    assert np.isfinite(TP).all() and np.isfinite(R["qpos"]).all() and np.isfinite(R["err"]).all() and (R["niter"] >= 0).all()
    o = _setup(m)
    conv = np.zeros(n, int); worst = np.zeros(n)
    for e in range(n):
        out = o.ik(sites, TP[e], m.qpos0)
        conv[e], worst[e] = out["converged"], out["err"][:, 0].max()
    differ = np.where(conv != R["converged"])[0]
    near = np.abs(worst[differ] - DEFAULTS["tol"]) < 1e-9
    gw, cw = float(R["err"][:, :, 0].max()), float(worst.max())
    REPORT["conv_gpu_" + name] = "GPU converged %.4f worst %.2e; CPU converged %.4f worst %.2e; %d flags differ (%d within round-off of tol)" % (
        R["converged"].mean(), gw, conv.mean(), cw, len(differ), int(near.sum()))
    print("\n%s: %s" % (name, REPORT["conv_gpu_" + name]))
    assert near.all(), differ[~near][:10]
    assert abs(gw - cw) <= 1e-6 * max(1.0, cw)


def _bits(t):
    import torch
    return t.view({torch.float64: torch.int64, torch.float32: torch.int32}[t.dtype]) if t.is_floating_point() else t


@pytest.mark.gpu
def test_properties_and_no_side_effects():
    import torch
    env = _warm("hand_pose", n=512); twin = _warm("hand_pose", n=512)
    m = env.mj_model; sites = _sites(m); n = env.num_envs
    q0 = env.t["qpos"].clone()
    lo, hi = np.full(m.nq, -np.inf), np.full(m.nq, np.inf)
    lim = m.jnt_limited.astype(bool) & (m.jnt_type >= 2)
    lo[m.jnt_qposadr[lim]], hi[m.jnt_qposadr[lim]] = m.jnt_range[lim, 0], m.jnt_range[lim, 1]
    lo, hi = torch.as_tensor(lo, device=env.device), torch.as_tensor(hi, device=env.device)
    qin = torch.minimum(torch.maximum(q0, lo), hi).contiguous()        # in range, so that the clamp leaves held dofs alone
    rng = np.random.default_rng(SEED)
    o = _setup(m)
    tp = torch.as_tensor(np.stack([[o.jac_site(s, _random_q(m, rng))[2] for s in sites] for _ in range(n)]), device=env.device)
    mask = rng.uniform(size=m.nv) < 0.5
    before = {k: v.clone() for k, v in env.t.items() if isinstance(v, torch.Tensor)}
    D0 = {k: v.clone() for k, v in env.data("site_xpos", "qacc").items()}
    r = env.ik(sites, tp, qpos_init=qin, dofs=mask, max_iter=30, tol=0.0)
    r0 = env.ik(sites, tp, qpos_init=qin, max_iter=0, fields=("qpos", "niter"))
    torch.cuda.synchronize()
    Q = r["qpos"]
    assert torch.equal(_bits(r0["qpos"]), _bits(qin)) and int(r0["niter"].abs().sum()) == 0
    assert bool((Q >= lo).all() and (Q <= hi).all())
    held = torch.as_tensor(~mask, device=env.device)
    assert torch.equal(_bits(Q[:, held]), _bits(qin[:, held]))
    for k, v in before.items():
        assert torch.equal(_bits(v), _bits(env.t[k])), k
    for k, v in env.data("site_xpos", "qacc").items():
        assert torch.equal(_bits(v), _bits(D0[k])), k
    g = torch.Generator(device="cpu").manual_seed(SEED + 5)
    for t in range(50):
        a = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device)
        env.step(a); twin.step(a)
        if t % 10 == 0:
            env.ik(sites, tp, max_iter=5)
    torch.cuda.synchronize()
    for k in ("qpos", "qvel", "act", "obs", "reward"):
        assert torch.equal(_bits(env.t[k]), _bits(twin.t[k])), k


@pytest.mark.gpu
def test_free_joint_quaternions_unit():
    import torch
    env = _warm("hold", n=256); m = env.mj_model
    sites = [m.name2id("site", "object")] + _sites(m)[:3]
    tp = env.jac_site(sites)[2] + 0.02
    r = env.ik(sites, tp.contiguous(), max_iter=20, tol=0.0)
    qa = int(m.jnt_qposadr[np.where(m.jnt_type == 0)[0][0]])
    nq = r["qpos"][:, qa + 3:qa + 7].norm(dim=1)
    assert float((nq - 1).abs().max()) < 1e-14


@pytest.mark.gpu
def test_batch_independence_and_libraries():
    import torch
    from myosuite_b200 import vec_env
    big = vec_env.MyoVecEnv.from_model("myolegs", 4096)
    m = big.mj_model; sites = [m.name2id("site", s) for s in CONV["myolegs"]]
    rng = np.random.default_rng(SEED)
    dev = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=big.device)
    qt, q0 = _random_q(m, rng, 4096), _random_q(m, rng, 4096)
    tp = big.jac_site(sites, qpos=dev(qt))[2].contiguous()
    rb = big.ik(sites, tp, qpos_init=dev(q0), posture=0.01, fields=big.IK_FIELDS)
    rows = np.arange(0, 4096, 64)
    for rs in ("p48", "f64"):
        small = vec_env.MyoVecEnv.from_model("myolegs", 64, row_storage=rs)
        r = small.ik(sites, tp[rows].contiguous(), qpos_init=dev(q0[rows]), posture=0.01, fields=big.IK_FIELDS)
        for k in big.IK_FIELDS:
            assert torch.equal(_bits(r[k]), _bits(rb[k][rows])), (rs, k)


@pytest.mark.gpu
def test_input_checks_without_launch():
    import torch
    from myosuite_b200 import abi
    env = _warm("elbow", n=64); m = env.mj_model; n = env.num_envs
    s = _sites(m); tp = env.jac_site(s)[2].contiguous()
    L0 = env.batch.launches
    bad = [dict(sites=[]), dict(sites=list(range(17))), dict(sites=[m.nsite]), dict(target_pos=tp.float()), dict(target_pos=tp[:, :, :2].contiguous()),
           dict(target_pos=tp.cpu()), dict(damping=0.0), dict(max_step=-1.0), dict(tol=-1.0), dict(max_iter=-1), dict(tol=float("nan")),
           dict(qpos_init=env.t["qpos"].t()), dict(dofs=np.ones(m.nv + 1, bool))]
    for kw in bad:
        args = dict(sites=s, target_pos=tp); args.update(kw)
        with pytest.raises((ValueError, KeyError)):
            env.ik(args.pop("sites"), args.pop("target_pos"), **args)
    assert env.batch.launches == L0
    # the C ABI's own checks
    out = torch.zeros((n, m.nq), dtype=torch.float64, device=env.device)
    sid = torch.as_tensor(np.array(s, np.int32), device=env.device)
    sq = torch.as_tensor(np.ascontiguousarray(m.site_quat[s]), device=env.device)
    env.batch.ik(abi.MyoIkParams(nsite=len(s), max_iter=1, tol=0.0, damping=1e-3, max_step=0.5, posture_weight=0.0, eq_weight=1.0),
                 site_id=sid, site_quat=sq, target_pos=tp, qpos=out)      # the well-formed call launches
    assert env.batch.launches == L0 + 1
    L0 += 1
    for p, bufs in ((dict(nsite=0), {}), (dict(nsite=17), {}), (dict(damping=0.0), {}), (dict(max_step=0.0), {}), (dict(tol=-1.0), {}),
                    (dict(max_iter=-1), {}), (dict(eq_weight=float("inf")), {}), ({}, dict(site_id=torch.tensor([m.nsite], dtype=torch.int32, device=env.device))),
                    ({}, dict(qpos=None)), ({}, dict(target_pos=None)), ({}, dict(site_id=None)), ({}, dict(site_quat=None))):
        prm = dict(nsite=len(s), max_iter=1, tol=0.0, damping=1e-3, max_step=0.5, posture_weight=0.0, eq_weight=1.0); prm.update(p)
        b = dict(site_id=sid, site_quat=sq, target_pos=tp, qpos=out); b.update(bufs)
        with pytest.raises(abi.MyoError):
            env.batch.ik(abi.MyoIkParams(**prm), **b)
    assert env.batch.launches == L0


@pytest.mark.gpu
def test_myoenv_single_env():
    import torch
    from myosuite_b200 import vec_env
    e1 = vec_env.MyoEnv("myoHandPoseRandom-v0", seed=SEED)
    e1.reset(seed=SEED)
    m = e1.mj_model if hasattr(e1, "mj_model") else e1.vec.mj_model
    q = e1.vec.t["qpos"][0].cpu().numpy()
    vb = vec_env.MyoVecEnv("myoHandPoseRandom-v0", 4, seed=SEED, auto_reset=False)
    vb.set_state(qpos=np.tile(q, (4, 1)))
    site = m.name2id("site", "IFtip")
    jp, jr = e1.mj_jacSite("IFtip")
    bjp, bjr, bx, _ = vb.jac_site([site])
    assert np.array_equal(jp, bjp[0, 0].cpu().numpy()) and np.array_equal(jr, bjr[0, 0].cpu().numpy())
    tp = bx[0].cpu().numpy() + 0.01
    r1 = e1.mj_ik(["IFtip"], tp, max_iter=20)
    rb = vb.ik([site], torch.as_tensor(np.tile(tp, (4, 1, 1)), device=vb.device), max_iter=20)
    assert np.array_equal(r1["qpos"], rb["qpos"][0].cpu().numpy()) and r1["niter"] == int(rb["niter"][0])
