"""The CPU oracle against (a) golden vectors produced by the reference's own Python code, and
(b) independent numpy computations / finite differences for the MuJoCo-restatement part (parity unpinned:
no MuJoCo available, see oracle/myo_oracle.c header)."""
import os

import numpy as np
import pytest

from myosuite_b200 import blob, mjcf, program
from oracle import env_oracle
from oracle.oracle_py import Oracle

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pylogic.npz"))


# ----------------------------------------------------------------------------- golden: python-side logic
def test_fatigue_known_answer():
    f = env_oracle.Fatigue(5, dt=0.002 * 5)
    for a, exp in zip(G["fatigue_kat_in"], G["fatigue_kat_out"]):
        MA, MR, MF = f.compute_act(a)
        np.testing.assert_allclose(np.stack([MA, MR, MF]), exp, rtol=1e-13, atol=1e-15)
    # SURVEY.md section 8c known answers (verified there against the reference)
    np.testing.assert_allclose(G["fatigue_kat_out"][3, 0], [0.509728576, 0.499965801, 0.6483463034, 0.5102154323, 0.7049798034], rtol=1e-9)
    np.testing.assert_allclose(G["fatigue_kat_out"][3, 2], [8.5495798416e-05, 9.1195798416e-05, 1.1398941168e-04, 8.2645798416e-05, 1.2538941168e-04], rtol=1e-9)


def test_fatigue_long_run():
    acts = np.random.default_rng(7).uniform(0, 1, (2000, 80))
    acts[500:700] = 1.0
    acts[1200:1300] = 0.0
    f = env_oracle.Fatigue(80, dt=0.001 * 10)
    for k, a in enumerate(acts):
        out = f.compute_act(a)
        if k % 50 == 0:
            np.testing.assert_allclose(np.stack(out), G["fatigue_long_out"][k // 50], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(np.stack(out), G["fatigue_long_final"], rtol=1e-12, atol=1e-14)
    assert np.allclose(f.MA + f.MR + f.MF, 1.0)


def test_action_remap_and_fatigue_chain():
    np.testing.assert_allclose(np.stack([env_oracle.action_to_ctrl(a) for a in G["step_action_none"]]), G["step_ctrl_none"], rtol=1e-15)
    f = env_oracle.Fatigue(39, dt=0.02)
    got = np.stack([f.compute_act(env_oracle.action_to_ctrl(a))[0].copy() for a in G["step_action_fatigue"]])
    np.testing.assert_allclose(got, G["step_ctrl_fatigue"], rtol=1e-13)
    # float32 actions: the reference evaluates the sigmoid in float32 -> agrees with the f64 remap to f32 round-off
    np.testing.assert_allclose(G["step_ctrl_f32in"], G["step_ctrl_none"], rtol=0, atol=2e-7)


@pytest.mark.parametrize("tag,thd", [("elbow", 0.175), ("hand", 0.7)])
def test_pose_obs_reward(tag, thd):
    q, v, a, t = (G["pose_%s_%s" % (tag, k)] for k in ("qpos", "qvel", "act", "target"))
    for i in range(len(q)):
        obs = env_oracle.pose_obs(q[i], v[i], a[i], t[i], 0.02)
        assert obs.dtype == np.float32
        np.testing.assert_array_equal(obs, G["pose_%s_obs" % tag][i])
        r = env_oracle.pose_reward(q[i], a[i], t[i], thd)
        for k in ("pose", "bonus", "penalty", "act_reg", "sparse", "dense"):
            np.testing.assert_allclose(r[k], G["pose_%s_rwd_%s" % (tag, k)][i], rtol=1e-14, atol=1e-15)
        assert bool(r["solved"]) == bool(G["pose_%s_rwd_solved" % tag][i]) and bool(r["done"]) == bool(G["pose_%s_rwd_done" % tag][i])
    assert G["pose_%s_rwd_done" % tag].sum() >= 2 and G["pose_%s_rwd_bonus" % tag].max() == 2


# ----------------------------------------------------------------------------- physics restatement: independent cross-checks
def _rand_state(m, rng, margin=0.1):
    q = m.qpos0.copy()
    for j in range(m.njnt):
        if m.jnt_type[j] != 0:
            lo, hi = m.jnt_range[j]
            q[m.jnt_qposadr[j]] = rng.uniform(lo + margin * (hi - lo), hi - margin * (hi - lo))
    return q


def _dense_M(m, qM):
    M = np.zeros((m.nv, m.nv))
    for i in range(m.nv):
        adr, j = m.dof_Madr[i], i
        while j >= 0:
            M[i, j] = M[j, i] = qM[adr]
            adr += 1
            j = m.dof_parentid[j]
    return M


@pytest.mark.parametrize("name", ["myoelbow_1dof6muscles", "myohand_pose", "myolegs"])
def test_oracle_kinematics_mass_gravity_tendon(models, name):
    m = models[name]
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(0)
    q = _rand_state(m, rng)
    o.set(qpos=q, qvel=np.zeros(m.nv), act=rng.uniform(0, 1, m.na), ctrl=rng.uniform(0, 1, m.nu))
    o.forward()
    kin = mjcf.kinematics(m, q)
    np.testing.assert_allclose(o.f("xpos").reshape(-1, 3), kin["xpos"], atol=1e-13)
    M1 = _dense_M(m, o.f("qM").copy())
    np.testing.assert_allclose(M1, mjcf.mass_matrix(m, kin), rtol=1e-10, atol=1e-14)
    o.forward()                                           # forward is idempotent (no state leaks between calls)
    np.testing.assert_array_equal(_dense_M(m, o.f("qM")), M1)
    g = np.zeros(m.nv)
    for b in range(1, m.nbody):
        if m.body_weldid[b]:
            jp, _ = mjcf.jac_point(m, kin, kin["xipos"][b], b)
            g -= m.body_mass[b] * (jp.T @ m.opt_gravity)
    np.testing.assert_allclose(o.f("qfrc_bias"), g, rtol=1e-9, atol=1e-12)
    # tendon Jacobian (incl. sphere/cylinder/inside wrapping) == finite difference of tendon length
    J = o.f("ten_J").reshape(m.ntendon, m.nv).copy()
    for d in range(m.nv):
        j = m.dof_jntid[d]
        if m.jnt_type[j] == 0:
            continue
        L = []
        for s in (+1, -1):
            qq = q.copy(); qq[m.jnt_qposadr[j]] += s * 1e-6
            o.set(qpos=qq); o.forward(); L.append(o.f("ten_length").copy())
        np.testing.assert_allclose((L[0] - L[1]) / 2e-6, J[:, d], atol=2e-8)


def test_oracle_muscle_curves():
    """MuJoCo's documented muscle curves: FL(1)=1, FL(lmin)=FL(lmax)=0, FV(0)=1, FV(-1)=0, FV(>=fvmax-1)=fvmax, passive 0 below L=1."""
    # exercised through a 1-muscle forward: elbow model, vary act/len via qpos
    from myosuite_b200 import assets
    m = assets.load("myoelbow_1dof6muscles")
    o = Oracle(*blob.pack(m))
    o.set(qpos=[1.0], act=np.zeros(6)); o.forward()
    f0 = o.f("actuator_force").copy()                      # act=0 -> passive force only (<= 0)
    assert np.all(f0 <= 0)
    o.set(act=np.ones(6)); o.forward()
    assert np.all(o.f("actuator_force") <= f0 + 1e-12)    # activation adds contractile (negative) force
    o.set(ctrl=np.ones(6), act=np.zeros(6)); o.forward()
    np.testing.assert_allclose(o.f("act_dot"), (1.0 - 0.0) / (0.01 * 0.5))        # tau_act*(0.5+1.5*0)
    o.set(ctrl=np.zeros(6), act=np.ones(6)); o.forward()
    np.testing.assert_allclose(o.f("act_dot"), (0.001 - 1.0) / (0.04 / 2.0))    # tau_deact/(0.5+1.5*1); ctrl is clamped to ctrlrange[0]=0.001 first


def test_oracle_joint_limit_and_solver(models):
    m = models["myoelbow_1dof6muscles"]
    o = Oracle(*blob.pack(m))
    o.set(qpos=[-0.05], qvel=[-1.0]); o.forward()          # below the lower limit (range 0..2.26893)
    assert o.nefc == 1 and o.f("efc_pos")[0] == pytest.approx(-0.05)
    assert o.f("efc_force")[0] > 0 and o.f("qacc")[0] > o.f("qacc_smooth")[0]
    # closed form for nv=1: a = (f + D*aref)/(M + D)
    M, D, aref, f = o.f("qM")[0], o.f("efc_D")[0], o.f("efc_aref")[0], o.f("qfrc_smooth")[0]
    assert o.f("qacc")[0] == pytest.approx((f + D * aref) / (M + D), rel=1e-12)
    o.set(qpos=[1.0], qvel=[0.0]); o.forward()
    assert o.nefc == 0 and o.f("qacc")[0] == pytest.approx(o.f("qacc_smooth")[0])


def test_oracle_hand_contacts_and_kkt(models):
    """Random hand poses produce capsule contacts; the Newton solution satisfies the optimality conditions."""
    m = models["myohand_pose"]
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(3)
    seen = seen_ell = 0
    for _ in range(20):
        q = _rand_state(m, rng, margin=-0.02)
        o.set(qpos=q, qvel=rng.normal(0, 1, m.nv), act=rng.uniform(0, 1, m.na), ctrl=rng.uniform(0, 1, m.nu)); o.forward()
        seen += o.ncon
        nefc = o.nefc
        J = o.f("efc_J").reshape(nefc, m.nv); force = o.f("efc_force")
        Mq = _dense_M(m, o.f("qM")) @ o.f("qacc")
        np.testing.assert_allclose(Mq, o.f("qfrc_smooth") + J.T @ force, rtol=1e-8, atol=1e-8 * np.abs(Mq).max())
        jar = J @ o.f("qacc") - o.f("efc_aref")
        assert np.all(force >= 0) and np.all(force[jar > 1e-9] == 0)
        g1, g2 = o.i("con_geom1"), o.i("con_geom2")
        t1, t2 = m.geom_type[g1], m.geom_type[g2]
        assert np.all(t1 <= t2) and np.all((g1 < g2) | (t1 < t2))      # MuJoCo's collider table: lower geom type first
        seen_ell += int(np.sum(t2 == 4))
    assert seen > 0 and seen_ell > 0      # capsule-capsule and capsule-ellipsoid (fingertip pad) contacts both occur


def test_oracle_rollout_stable(models):
    for name, n in (("myoelbow_1dof6muscles", 1000), ("myohand_pose", 300), ("myolegs", 100)):
        m = models[name]
        o = Oracle(*blob.pack(m))
        if m.nkey:
            o.set(qpos=m.key_qpos[0])
        rng = np.random.default_rng(1)
        for s in range(n):
            if s % 10 == 0:
                o.set(ctrl=rng.uniform(0, 1, m.nu))
            o.step()
        assert np.all(np.isfinite(o.f("qpos"))) and np.abs(o.f("qvel")).max() < 100
        assert np.all(o.f("act") >= -1e-9) and np.all(o.f("act") <= 1 + 1e-9)


# ----------------------------------------------------------------------------- golden: Walk / ObjHold task logic (reference classes run on oracle states)
T = np.load(os.path.join(os.path.dirname(__file__), "golden", "tasks.npz"))


def test_walk_obs_reward_golden(models):
    m = models["myolegs"]
    o = Oracle(*blob.pack(m))
    ids = env_oracle.walk_ids(m)
    cfg = dict(hip_period=100, min_height=0.8, max_rot=0.8, target_x_vel=0.0, target_y_vel=1.2, target_rot=m.key_qpos[0][3:7])
    for i in range(len(T["walk_qpos"])):
        o.reset(); o.set(qpos=T["walk_qpos"][i], qvel=T["walk_qvel"][i], act=T["walk_act"][i], ctrl=np.zeros(m.nu)); o.forward()
        obs, r = env_oracle.walk_obs_reward(m, o, int(T["walk_steps"][i]), 0.01, ids, cfg)
        np.testing.assert_allclose(obs, T["walk_obs"][i], rtol=1e-6, atol=1e-6)
        for k in ("vel_reward", "cyclic_hip", "ref_rot", "joint_angle_rew", "dense"):
            np.testing.assert_allclose(r[k], T["walk_" + k][i], rtol=1e-9, atol=1e-9)
        assert bool(r["done"]) == bool(T["walk_done"][i])


def test_hold_obs_reward_golden(models):
    m = models["myohand_hold"]
    o = Oracle(*blob.pack(m))
    for i in range(len(T["hold_qpos"])):
        o.reset(); o.set(qpos=T["hold_qpos"][i], qvel=T["hold_qvel"][i], act=T["hold_act"][i]); o.forward()
        obs, r = env_oracle.hold_obs_reward(m, o, 0.02, T["hold_goal"][i])
        np.testing.assert_allclose(obs, T["hold_obs"][i], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(r["dense"], T["hold_dense"][i], rtol=1e-9, atol=1e-9)
        assert bool(r["done"]) == bool(T["hold_done"][i])


def test_reach_obs_reward_golden(models):
    """ReachEnvV0 (reach_v0.py:98-160) restated in env_oracle vs vectors produced by the reference's own class, including the
    `time > 2 dt` switch of far_th that MuJoCo's per-substep time accumulation flips one control step early."""
    import json, os
    m = models["myohand_pose"]
    o = Oracle(*blob.pack(m))
    reg = json.load(open(os.path.join(os.path.dirname(blob.__file__), "assets", "registry.json")))["envs"]["myoHandReachRandom-v0"]["kwargs"]
    tips = list(reg["target_reach_range"].keys())
    assert tips == ["THtip", "IFtip", "MFtip", "RFtip", "LFtip"]           # reference registration order = obs layout order
    for i in range(len(T["reach_qpos"])):
        o.reset(); o.set(qpos=T["reach_qpos"][i], qvel=T["reach_qvel"][i], act=T["reach_act"][i]); o.forward()
        obs, r = env_oracle.reach_obs_reward(m, o, 0.02, tips, T["reach_targets"][i], float(T["reach_time"][i]), far_th=reg["far_th"])
        np.testing.assert_allclose(obs, T["reach_obs"][i], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(r["dense"], T["reach_dense"][i], rtol=1e-9, atol=1e-9)
        assert bool(r["done"]) == bool(T["reach_done"][i]) and bool(r["solved"]) == bool(T["reach_solved"][i])


def test_mujoco_goldens_if_present(models):
    """Pins the oracle to a real MuJoCo when a maintainer has produced tests/golden/mujoco_<env>.npz with tools/dump_reference.py
    (impossible in this round's containers: no mujoco).  Acceptance = north-star: qacc / actuator_force within 1e-5 relative."""
    import glob, os
    files = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "mujoco_*.npz")))
    if not files:
        pytest.skip("no MuJoCo goldens (parity unpinned, DESIGN.md section 2)")
    from myosuite_b200 import assets
    xml_of = {"Elbow": "myoelbow_1dof6muscles", "HandPose": "myohand_pose", "HandReach": "myohand_pose", "ObjHold": "myohand_hold", "Leg": "myolegs"}
    for f in files:
        G = np.load(f, allow_pickle=False)
        name = next(v for k, v in xml_of.items() if k in str(G["meta"][0]))
        m = models.get(name) or assets.load(name)
        o = Oracle(*blob.pack(m))
        for i in range(min(50, len(G["qpos"]))):
            o.reset(); o.set(qpos=G["qpos"][i], qvel=G["qvel"][i], act=G["act"][i], ctrl=G["ctrl"][i]); o.forward()
            scale = np.abs(G["qacc"][i]).max() + 1e-9
            assert np.abs(o.f("qacc") - G["qacc"][i]).max() <= 1e-5 * scale
            np.testing.assert_allclose(o.f("actuator_force"), G["actuator_force"][i], rtol=1e-5, atol=1e-5 * np.abs(G["actuator_force"][i]).max())


@pytest.mark.parametrize("name", ["myoelbow_1dof6muscles", "myohand_pose"])
def test_oracle_coriolis_from_mass_matrix_derivatives(models, name):
    """Velocity-dependent bias forces against their textbook definition from the (independently checked) mass matrix:
    c_i = sum_jk (dM_ij/dq_k - 1/2 dM_jk/dq_i) qd_j qd_k, with dM/dq by central differences.  Hinge/slide models (nq == nv)."""
    m = models[name]
    assert m.nq == m.nv
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(3)
    q = _rand_state(m, rng, margin=0.25)
    qd = rng.normal(0, 2.0, m.nv)
    z = np.zeros(m.na)

    def fwd(qq, vv):
        o.reset(); o.set(qpos=qq, qvel=vv, act=z, ctrl=np.zeros(m.nu)); o.forward()
        return o.f("qfrc_bias").copy(), _dense_M(m, o.f("qM").copy())

    b1, _ = fwd(q, qd)
    b0, _ = fwd(q, np.zeros(m.nv))
    c = b1 - b0                                            # Coriolis + centrifugal part (gravity removed)
    eps = 1e-5
    dM = np.zeros((m.nv, m.nv, m.nv))                      # dM[k] = dM/dq_k
    for k in range(m.nv):
        qa = q.copy(); qa[m.jnt_qposadr[m.dof_jntid[k]]] += eps
        qb = q.copy(); qb[m.jnt_qposadr[m.dof_jntid[k]]] -= eps
        dM[k] = (fwd(qa, np.zeros(m.nv))[1] - fwd(qb, np.zeros(m.nv))[1]) / (2 * eps)
    Mdot = np.einsum("kij,k->ij", dM, qd)
    ref = Mdot @ qd - 0.5 * np.einsum("j,ijk,k->i", qd, dM, qd)
    np.testing.assert_allclose(c, ref, rtol=2e-5, atol=2e-7 * max(1.0, np.abs(ref).max()))


# ----------------------------------------------------------------------------- contacts: independent geometry and Jacobian checks
def _point_ellipsoid_dist(y, a):
    """Distance from point y (ellipsoid frame) to the ellipsoid with semi-axes a, y outside.  Classical Lagrange-multiplier root:
    closest point x_i = a_i^2 y_i / (a_i^2 + t) with sum (a_i y_i / (a_i^2 + t))^2 = 1, t > 0 (independent of the oracle's search)."""
    from scipy.optimize import brentq
    f = lambda t: np.sum((a * y / (a * a + t)) ** 2) - 1.0
    assert f(0.0) > 0                                     # outside
    hi = 1.0
    while f(hi) > 0:
        hi *= 4
    t = brentq(f, 0.0, hi, xtol=1e-18, rtol=1e-15, maxiter=500)
    x = a * a * y / (a * a + t)
    return np.linalg.norm(y - x)


def _capsule(o, m, g):
    X = o.f("geom_xmat").reshape(-1, 9)[g].reshape(3, 3); c = o.f("geom_xpos").reshape(-1, 3)[g]
    return c, X[:, 2], m.geom_size[g, 0], m.geom_size[g, 1]


def _pair_distance(o, m, g1, g2):
    """Signed distance of a capsule-capsule or capsule-ellipsoid pair by an independent route (scipy)."""
    from scipy.optimize import minimize, minimize_scalar
    c1, a1, r1, h1 = _capsule(o, m, g1)
    if m.geom_type[g2] == 3:
        c2, a2, r2, h2 = _capsule(o, m, g2)
        f = lambda p: np.linalg.norm((c1 + a1 * p[0]) - (c2 + a2 * p[1]))
        best = min((minimize(f, [s, t], bounds=[(-h1, h1), (-h2, h2)], method="L-BFGS-B", options=dict(ftol=1e-18, gtol=1e-14)).fun
                    for s in (-h1, 0, h1) for t in (-h2, 0, h2)))
        return best - r1 - r2
    X2 = o.f("geom_xmat").reshape(-1, 9)[g2].reshape(3, 3); c2 = o.f("geom_xpos").reshape(-1, 3)[g2]; a = m.geom_size[g2].copy()
    f = lambda t: _point_ellipsoid_dist(X2.T @ (c1 + a1 * t - c2), a)
    res = minimize_scalar(f, bounds=(-h1, h1), method="bounded", options=dict(xatol=1e-13))
    return min(res.fun, f(-h1), f(h1)) - r1


def _hand_states_with_contacts(m, o, rng, want=12):
    out = []
    while len(out) < want:
        q = _rand_state(m, rng, margin=-0.02)
        o.reset(); o.set(qpos=q, qvel=np.zeros(m.nv), act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
        if o.ncon:
            out.append(q)
    return out


def test_oracle_contact_distances_independent(models):
    """Signed distances of the reported capsule-capsule and capsule-ellipsoid contacts against scipy (segment-segment minimisation;
    point-ellipsoid distance by its Lagrange root, minimised over the segment).  Ellipsoid cases are checked where the capsule axis
    stays outside the ellipsoid (the regime the colliders are specified for, DESIGN.md section 2)."""
    m = models["myohand_pose"]
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(11)
    n_cc = n_ce = 0
    for q in _hand_states_with_contacts(m, o, rng, want=10):
        o.reset(); o.set(qpos=q, qvel=np.zeros(m.nv), act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
        g1s, g2s, ds = o.i("con_geom1").copy(), o.i("con_geom2").copy(), o.f("con_dist").copy()
        for g1, g2, d in zip(g1s, g2s, ds):
            if m.geom_type[g1] != 3 or m.geom_type[g2] not in (3, 4):
                continue
            if m.geom_type[g2] == 4:
                if d < -0.5 * m.geom_size[g1, 0]:
                    continue                                # deep overlap: outside the specified regime
                n_ce += 1
            else:
                n_cc += 1
            np.testing.assert_allclose(d, _pair_distance(o, m, int(g1), int(g2)), rtol=0, atol=2e-9)
    assert n_cc >= 10 and n_ce >= 2


def test_oracle_contact_normal_jacobian_fd(models):
    """Normal row of every contact Jacobian = derivative of that pair's signed distance w.r.t. the joint angles (central differences):
    checks witness points, normals and the dof paths of the contact rows, capsule and ellipsoid colliders alike."""
    m = models["myohand_pose"]
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(12)
    checked = 0
    for q in _hand_states_with_contacts(m, o, rng, want=4):
        o.reset(); o.set(qpos=q, qvel=np.zeros(m.nv), act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
        ncon, nefc = o.ncon, o.nefc
        g1s, g2s, ds = o.i("con_geom1").copy(), o.i("con_geom2").copy(), o.f("con_dist").copy()
        J = o.f("efc_J").reshape(nefc, m.nv).copy()
        assert (nefc - 4 * ncon) >= 0                       # condim-3 pyramids: 4 rows per contact, after the limit rows
        Jc = J[nefc - 4 * ncon:].reshape(ncon, 4, m.nv)
        Jn = 0.5 * (Jc[:, 0] + Jc[:, 1])                    # (n + mu t1) and (n - mu t1) average to the normal row
        margin = 0.001
        sel = [c for c in range(ncon) if ds[c] < margin - 3e-4 and (m.geom_type[g2s[c]] != 4 or ds[c] > -0.5 * m.geom_size[g1s[c], 0])]
        fd = np.zeros((len(sel), m.nv)); eps = 1e-6
        for k in range(m.nv):
            dd = []
            for sgn in (+1, -1):
                qq = q.copy(); qq[m.jnt_qposadr[m.dof_jntid[k]]] += sgn * eps
                o.reset(); o.set(qpos=qq, qvel=np.zeros(m.nv), act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
                pairs = {(int(a), int(b)): float(x) for a, b, x in zip(o.i("con_geom1"), o.i("con_geom2"), o.f("con_dist"))}
                dd.append([pairs.get((int(g1s[c]), int(g2s[c])), np.nan) for c in sel])
            fd[:, k] = (np.array(dd[0]) - np.array(dd[1])) / (2 * eps)
        ok = ~np.isnan(fd).any(axis=1)
        assert ok.sum() >= max(1, len(sel) - 1)
        np.testing.assert_allclose(Jn[np.array(sel)[ok]], fd[ok], rtol=0, atol=5e-7)
        checked += int(ok.sum())
    assert checked >= 8


@pytest.mark.parametrize("name", ["myoelbow_1dof6muscles", "myohand_pose"])
def test_oracle_euler_step_from_forward_outputs(models, name):
    """One mj_step equals semi-implicit Euler with implicit joint damping applied to the forward pass's own outputs:
    qvel' = qvel + h (M + h diag(damping))^-1 M qacc ; qpos' = qpos + h qvel' ; act' = act + h act_dot ; time' = time + h."""
    m = models[name]
    o = Oracle(*blob.pack(m))
    rng = np.random.default_rng(21)
    q = _rand_state(m, rng, margin=0.2)
    v, a, u = rng.normal(0, 1.0, m.nv), rng.uniform(0, 1, m.na), rng.uniform(0, 1, m.nu)
    o.reset(); o.set(qpos=q, qvel=v, act=a, ctrl=u); o.forward()
    M = _dense_M(m, o.f("qM").copy()); qacc = o.f("qacc").copy(); adot = o.f("act_dot").copy(); h = m.opt_timestep
    o.reset(); o.set(qpos=q, qvel=v, act=a, ctrl=u); o.step(1)
    v1 = v + h * np.linalg.solve(M + h * np.diag(m.dof_damping), M @ qacc)
    np.testing.assert_allclose(o.f("qvel"), v1, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(o.f("qpos"), q + h * v1, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(o.f("act"), a + h * adot, rtol=1e-12, atol=1e-14)
    assert o.f("time")[0] == pytest.approx(h)


def test_tendon_length_ranges_vs_reference_xml(models):
    """Weak anchor to MuJoCo-derived numbers inside the reference's own files (SURVEY 8c): the muscles' `lengthrange` attributes in
    the leg / hand XMLs were produced by MuJoCo-based tooling.  Sampling the joint-range box, the oracle's actuator lengths must span
    the same intervals.  Legs: 90 % of the 80 muscles agree at both ends within 10 % of their span (outliers: the vasti/patella
    group, whose joints are tied by equalities the sampling ignores).  Hand: several XML values are stale w.r.t. the XML's own
    geometry (e.g. FDS4: the straight polyline through its sites is 0.409 m, below the listed minimum 0.422 m), so only a majority test."""
    for name, base, frac10, frac20 in (("myolegs", "key", 0.85, 0.92), ("myohand_pose", "qpos0", 0.42, 0.60)):
        m = models[name]
        o = Oracle(*blob.pack(m))
        rng = np.random.default_rng(0)
        lo, hi = np.full(m.nu, np.inf), np.full(m.nu, -np.inf)
        for it in range(600):
            q = (m.key_qpos[0] if base == "key" else m.qpos0).copy()
            for j in range(m.njnt):
                if m.jnt_type[j] != 0 and m.jnt_limited[j]:
                    a, b = m.jnt_range[j]
                    q[m.jnt_qposadr[j]] = rng.choice([a, b]) if it % 3 == 0 else rng.uniform(a, b)
            o.reset(); o.set(qpos=q, qvel=np.zeros(m.nv), act=np.zeros(m.na), ctrl=np.zeros(m.nu)); o.forward()
            L = o.f("actuator_length"); lo, hi = np.minimum(lo, L), np.maximum(hi, L)
        lr = m.actuator_lengthrange; span = lr[:, 1] - lr[:, 0]
        dlo, dhi = np.abs(lo - lr[:, 0]) / span, np.abs(hi - lr[:, 1]) / span
        assert np.mean((dlo < 0.1) & (dhi < 0.1)) >= frac10, (name, np.mean((dlo < 0.1) & (dhi < 0.1)))
        assert np.mean((dlo < 0.2) & (dhi < 0.2)) >= frac20, (name, np.mean((dlo < 0.2) & (dhi < 0.2)))
        assert 0.9 < np.median((hi - lo) / span) < 1.1


def test_statistical_drop_in_vs_reference_npg_logs():
    """End-to-end statistical anchor to numbers the REFERENCE STACK produced (MuJoCo + reference env code + mjrl sampler): iteration 0
    of the committed NPG baselines (myosuite/agents/baslines_NPG/<env>/*/*/logs/log.csv; 96 trajectories of a freshly initialised
    Gaussian policy: mean ~ 0, log_std -0.25, job_config.yaml) logged for myoHandPoseRandom-v0 mean return -336.1, std 28.1,
    max -265.8, min -408.6, success 0 %, and for myoElbowPose1D6MRandom-v0 mean 61-65, std 189-191, success 54-55 %.
    The same protocol on this repo's oracle + env logic (tests/devtools/npg_iter0_check.py; full-size run: hand -335.8 / 29.8 / -266.5 /
    -403.7 / 0 %, elbow 62.9 / 187 / 58 %) must land inside sampling error of those."""
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "devtools"))
    import npg_iter0_check as chk
    h = chk.run("myoHandPoseRandom-v0", 48, seed=1)
    assert abs(h["mean"] + 336.1) < 15 and 18 < h["std"] < 42 and h["success_pct"] == 0 and h["max"] < -200 and h["min"] > -470, h
    e = chk.run("myoElbowPose1D6MRandom-v0", 480, seed=1)
    assert abs(e["mean"] - 63.0) < 45 and abs(e["std"] - 190) < 25 and abs(e["success_pct"] - 54.5) < 15, e

