"""Inverse dynamics (myo_batch_inverse, MyoVecEnv.inverse, MyoEnv.mj_inverse) against the CPU oracle's mj_inverse and against the
forward dynamics it inverts.

CPU: the myo_inverse_buffers field order against abi.py; the oracle's recursive Newton-Euler with the acceleration against its own mass
matrix and bias on every shipped model and the sweep models; its round trips (forward -> inverse gives qfrc_actuator back, with
constraints and through one Euler step with implicit damping); efc_force of the inverse at the forward's qacc.

GPU, on both row storages: every registered base task at its benchmarked launch shape after a reset and random-action steps against the
oracle (tests/inverse_oracle.c); the round trips through the device's own forward pass and integrator; invariance under act, ctrl and
the warm start; no side effects; slot independence at trajectory scale; input checks."""
import ctypes
import os

import numpy as np
import pytest

from inverse_oracle import INV_DISCRETE, INV_NOCONSTRAINT, InvOracle
from parity_helpers import _in_regime, _states
from test_mj_data import BOUND, CASES, ROWS, SEED, WARM, _contact_force_ref, _header_struct, _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FREE_REL = 1e-12           # constraints off: relative to the env's largest term (M qacc, bias - passive, qfrc_inverse)
MOMENT_REL = 5e-12         # actuator_moment against gear x ten_J, relative to the env's largest moment: the readout's length bound
                           # (test_mj_data.py); the reach task's hand measures 1.4e-12 on an H100
CON_MID, CON_MAX, CON_SHARE = 1e-6, 1e-5, 0.99       # with constraints: the readout's qacc bounds (test_mj_data.py)
ROUNDOFF_REL = 1e-9        # round trips: what exceeds the solver's stop rule, relative to the env's largest term
REPORT = {}
SHIPPED = ["myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso"]


def qM_dense(m, qM):
    M = np.zeros((m.nv, m.nv))
    for i in range(m.nv):
        adr, j = m.dof_Madr[i], i
        while j >= 0:
            M[i, j] = M[j, i] = qM[adr]; adr += 1; j = m.dof_parentid[j]
    return M


# ----------------------------------------------------------------------------- CPU
def test_inverse_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_inverse_buffers")
    assert len(fields) == decls and abi.INVERSE_FIELDS == fields
    assert [n for n, _ in abi.MyoInverseBuffers._fields_] == fields and ctypes.sizeof(abi.MyoInverseBuffers) == 8 * len(fields)
    assert set(abi.INVERSE_SHAPES) == set(fields) - {"qacc"}
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert src.index("} myo_data_buffers;") < src.index("} myo_inverse_buffers;") < src.index("int myo_batch_inverse(")
    assert "#define MYO_INV_NOCONSTRAINT %d " % abi.INV_NOCONSTRAINT in src and "#define MYO_INV_DISCRETE %d " % abi.INV_DISCRETE in src
    assert "myo_batch_inverse" in abi.EXPORTS


def _sweeps(tmp):
    import test_actuation_zoo as AZ
    return {k: v["m"] for k, v in AZ.build_zoo(tmp, names=["SWEEP_%d" % nv for nv in AZ.SWEEP_NV]).items()}


def test_oracle_rne_with_acceleration(models, tmp_path):
    """Constraints off: RNE with the acceleration (+ armature qacc - passive) equals qM qacc + qfrc_bias - qfrc_passive of the oracle's own
    forward pass at random states and random accelerations: an independent check of the mass matrix and the bias."""
    from myosuite_b200 import blob
    ms = {k: models[k] for k in SHIPPED}
    ms.update(_sweeps(tmp_path))
    rng = np.random.default_rng(SEED)
    worst = {}
    for name, m in ms.items():
        o = InvOracle(*blob.pack(m))
        qpos, qvel, act, _ = _states(m, 6, rng)
        for e in range(len(qpos)):
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e]); o.forward()
            M, bias, passive = qM_dense(m, o.f("qM")), o.f("qfrc_bias").copy(), o.f("qfrc_passive").copy()
            qacc = rng.normal(0, 10, m.nv)
            got = o.inverse(qacc, INV_NOCONSTRAINT)
            ref = M @ qacc + bias - passive
            scale = max(np.abs(M @ qacc).max(), np.abs(bias).max(), np.abs(passive).max(), np.abs(ref).max())
            err = float(np.abs(got - ref).max() / scale)
            worst[name] = max(worst.get(name, 0.0), err)
            assert err <= FREE_REL, (name, e, err)
            assert not np.any(o.f("qfrc_constraint"))
    print("\nRNE with acceleration vs qM qacc + bias - passive, worst relative: %s" % {k: "%.1e" % v for k, v in worst.items()})


def _roundtrip_states(models, tmp_path):
    """(name, model, [(qpos, qvel, act)]) at states the oracle reaches by stepping (shipped models), and the zoo configurations"""
    import test_actuation_zoo as AZ
    import test_contact_zoo as CZ
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    rng = np.random.default_rng(SEED)
    out = []
    for name in SHIPPED:
        m = models[name]
        o = Oracle(*blob.pack(m))
        qpos, qvel, act, ctrl = _states(m, 3, rng, overshoot=0.0, vel=0.3)
        sts = []
        for e in range(len(qpos)):
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.step(20)
            sts.append((o.f("qpos").copy(), o.f("qvel").copy(), o.f("act").copy()))
        out.append((name, m, sts))
    (tmp_path / "c").mkdir(); (tmp_path / "a").mkdir()
    cz = CZ.build_zoo(tmp_path / "c")
    for key in ("CAP_CAP", "PLANE_CAP", "CAP_ELL", "COMBO"):
        m = cz[key][0]
        cfgs = CZ._configs({key: cz[key]}, key) if key != "COMBO" else CZ._configs(cz, key)
        qpos = np.stack([q for _, q in cfgs]); qvel, act, _ = CZ._state(m, qpos, 5, [lb != "generic" for lb, _ in cfgs])
        out.append(("contact/" + key, m, list(zip(qpos, qvel, act))))
    for key, z in AZ.build_zoo(tmp_path / "a", names=["WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS", "SWEEP_16", "SWEEP_40"]).items():
        out.append(("actuation/" + key, z["m"], list(zip(z["qpos"], z["qvel"], z["act"]))))
    return out


def test_oracle_round_trips(models, tmp_path):
    """Forward, then the inverse of its qacc gives qfrc_actuator back (the residual is the Newton gradient the oracle's solve stopped at),
    and efc_force of the inverse equals the forward's.  Discrete: one oracle_step from s, then the inverse of (qvel' - qvel) / h with
    INV_DISCRETE at s gives qfrc_actuator(s) back, at states without an active constraint row."""
    from myosuite_b200 import blob
    worst, worst_d, nd = {}, {}, 0
    for name, m, sts in _roundtrip_states(models, tmp_path):
        o = InvOracle(*blob.pack(m))
        h = m.opt_timestep
        for qpos, qvel, act in sts:
            o.reset(); o.set(qpos=qpos, qvel=qvel, act=act); o.forward()
            qacc, act_f, nefc = o.f("qacc").copy(), o.f("qfrc_actuator").copy(), o.nefc
            f_fwd, c_fwd = o.f("efc_force").copy(), o.f("qfrc_constraint").copy()
            scale = max(np.abs(act_f).max(), np.abs(c_fwd).max(), np.abs(o.f("qfrc_bias")).max(), 1e-300)
            got = o.inverse(qacc)
            assert o.nefc == nefc
            err = float(np.abs(got - act_f).max() / scale)
            ferr = float(np.abs(o.f("efc_force") - f_fwd).max() / max(np.abs(f_fwd).max(), 1e-300)) if nefc else 0.0
            worst[name] = max(worst.get(name, 0.0), err, ferr)
            assert err <= ROUNDOFF_REL and ferr <= ROUNDOFF_REL, (name, err, ferr)
            if np.any(o.f("efc_force") != 0):
                continue
            o.reset(); o.set(qpos=qpos, qvel=qvel, act=act); o.step(1)
            qacc_d = (o.f("qvel") - qvel) / h
            o.reset(); o.set(qpos=qpos, qvel=qvel, act=act)
            got = o.inverse(qacc_d, INV_DISCRETE)
            err = float(np.abs(got - act_f).max() / scale)
            worst_d[name] = max(worst_d.get(name, 0.0), err); nd += 1
            assert err <= ROUNDOFF_REL, (name, "discrete", err)
    print("\nforward -> inverse, worst relative residual (qfrc_actuator, efc_force): %s" % {k: "%.1e" % v for k, v in worst.items()})
    print("step -> discrete inverse over %d constraint-free states: %s" % (nd, {k: "%.1e" % v for k, v in worst_d.items()}))
    assert "myoelbow_1dof6muscles" in worst_d and nd >= 10


# ----------------------------------------------------------------------------- GPU helpers
def _inv_oracles(env):
    from test_product_parity import Oracles
    oracles = Oracles(env)
    oracles.Oracle, oracles.base = InvOracle, InvOracle(env.I, env.D)
    return oracles


def _set(o, S, e, m):
    o.reset()
    o.set(qpos=S["qpos"][e], qvel=S["qvel"][e], act=S["act"][e, :m.na], ctrl=np.zeros(m.nu))


def _host(D):
    return {k: v.cpu().numpy().copy() for k, v in D.items()}


ALL = ("qfrc_inverse", "qfrc_constraint", "contact_force", "actuator_moment")


def _run_variants(env, Q, R):
    """the four inverses the oracle comparison checks: (random, readout qacc) x (constraints on, off)"""
    out = {}
    for qn, q in (("rand", R), ("readout", Q)):
        out[qn, True] = _host(env.inverse(q, fields=ALL))
        out[qn, False] = _host(env.inverse(q, constraints=False, fields=("qfrc_inverse", "qfrc_constraint")))
    out["discrete", True] = _host(env.inverse(R, discrete=True, fields=ALL))
    return out


def compare_env(env, V, QH, RH, S, e, o, worst):
    """Every inverse output of env e against the oracle set to its rows; False (skipped) outside the contact regime."""
    m = env.mj_model
    msg = "%s env %d" % (env.env_id or "model", e)
    for qn, q in (("rand", RH[e]), ("readout", QH[e]), ("discrete", RH[e])):
        for con in ((True,) if qn == "discrete" else (True, False)):
            _set(o, S, e, m)
            ref = o.inverse(q, (0 if con else INV_NOCONSTRAINT) | (INV_DISCRETE if qn == "discrete" else 0))
            if qn == "discrete":       # the oracle's M qacc_c: qacc_c = M^-1 (M + h B) q
                q = np.linalg.solve(qM_dense(m, o.f("qM")), qM_dense(m, o.f("qM")) @ q + m.opt_timestep * m.dof_damping * q)
            if qn == "rand" and con and not _in_regime(o, m):
                return False
            Mq = qM_dense(m, o.f("qM")) @ q
            rc = o.f("qfrc_constraint").copy()
            scale = max(np.abs(ref).max(), np.abs(Mq).max(), np.abs(ref - Mq + rc).max(), np.abs(rc).max())
            D = V[qn, con]
            err = float(max(np.abs(D["qfrc_inverse"][e] - ref).max(), np.abs(D["qfrc_constraint"][e] - rc).max()) / scale)
            key = "%s_%s" % (qn, "con" if con else "free")
            worst[key] = max(worst.get(key, 0.0), err)
            if not con:
                assert err <= FREE_REL and not np.any(D["qfrc_constraint"][e]), (msg, key, err)
                continue
            worst[key + "_over_mid"] = worst.get(key + "_over_mid", 0) + int(err >= CON_MID)
            assert err < CON_MAX, (msg, key, err)
            nc = o.ncon
            ref_f = _contact_force_ref(o, m)
            if nc:
                fs = max(np.abs(ref_f[:, 0]).max(), 1e-300)
                ferr = float(np.abs(D["contact_force"][e, :nc] - ref_f).max() / fs)
                worst[key + "_contact_force"] = max(worst.get(key + "_contact_force", 0.0), ferr)
                assert ferr < CON_MAX, (msg, key, "contact_force", ferr)
            assert not np.any(D["contact_force"][e, nc:]), msg
            if qn == "rand":
                J = o.f("ten_J").reshape(-1, m.nv)[m.actuator_trnid[:, 0]] * m.actuator_gear[:, 0, None]
                merr = float(np.abs(D["actuator_moment"][e] - J).max() / max(np.abs(J).max(), 1e-300))
                worst["actuator_moment"] = max(worst.get("actuator_moment", 0.0), merr)
                assert merr <= MOMENT_REL, (msg, merr)
    return True


def _warm_env(case, rows, **kw):
    import torch
    from myosuite_b200 import vec_env
    eid, n = CASES[case]
    env = vec_env.MyoVecEnv(eid, n, seed=SEED, row_storage=rows, **kw)
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(WARM):
        env.step((torch.rand(n, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
    return env


def _random_qacc(env, Q, seed=SEED):
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    mag = Q.abs().amax(1, keepdim=True).clamp_min(1.0)
    return (torch.randn(Q.shape, generator=g, dtype=torch.float64).to(env.device) * mag).contiguous()


def _report(key, worst, extra=""):
    REPORT[key] = extra + ", ".join("%s %.1e" % (k, v) if isinstance(v, float) else "%s %d" % (k, v) for k, v in sorted(worst.items()))
    print("\n%s %s" % (key, REPORT[key]))


# ----------------------------------------------------------------------------- GPU: registered tasks against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_inverse_vs_oracle(case, rows):
    """qfrc_inverse and qfrc_constraint with random accelerations and with the readout's qacc, with and without constraints, and of
    the random accelerations read as discrete ones; contact_force; actuator_moment.  Every env (p48), every 4th and the 64 most contact-heavy (f64)."""
    import torch
    env = _warm_env(case, rows)
    n = env.num_envs
    D = env.data("qacc", "ncon")
    Q = D["qacc"].clone(); R = _random_qacc(env, Q)
    V = _run_variants(env, Q, R)
    ncon = D["ncon"].cpu().numpy()
    torch.cuda.synchronize()
    S = env.get_env_state()
    QH, RH = Q.cpu().numpy(), R.cpu().numpy()
    envs = range(n) if rows == "p48" else sorted(set(range(0, n, 4)) | set(int(e) for e in np.argsort(ncon, kind="stable")[::-1][:64]))
    oracles = _inv_oracles(env)
    worst, checked, skipped = {}, 0, 0
    for e in envs:
        o = oracles.get(S["env_prm"][e] if "env_prm" in S else None)
        if compare_env(env, V, QH, RH, S, e, o, worst):
            checked += 1
        else:
            skipped += 1
    _report("%s[%s]" % (case, rows), worst, "checked %d, skipped (contact regime) %d; worst " % (checked, skipped))
    assert skipped <= 0.25 * len(envs) and checked > 0
    for k in ("rand_con", "readout_con", "discrete_con"):
        assert worst.get(k + "_over_mid", 0) <= (1 - CON_SHARE) * checked, k


# ----------------------------------------------------------------------------- GPU: round trips through the device's forward pass
def _tol(env):
    return float(env.cfg.solver_tolerance) or 1e-10


def _round_trip(env, worst, discrete_envs=None):
    """readout qacc -> inverse against the readout's qfrc_actuator.  Returns (ratio to the stop rule, round-off excess) per env."""
    m = env.mj_model
    D = _host(env.data("qacc", "qfrc_actuator"))
    q = env.torch.as_tensor(D["qacc"], device=env.device)
    I = _host(env.inverse(q, fields=("qfrc_inverse", "qfrc_constraint")))
    r = I["qfrc_inverse"] - D["qfrc_actuator"]
    stop = _tol(env) * m.stat_meaninertia * max(1, m.nv)
    big = np.maximum.reduce([np.abs(D["qfrc_actuator"]).max(1), np.abs(I["qfrc_constraint"]).max(1), np.abs(I["qfrc_inverse"]).max(1), np.full(len(r), 1e-300)])
    gn = np.linalg.norm(r, axis=1)
    excess = np.maximum(gn - stop, 0) / big
    worst["stop_ratio"] = max(worst.get("stop_ratio", 0.0), float((gn / stop).max()))
    worst["roundoff"] = max(worst.get("roundoff", 0.0), float(excess.max()))
    assert excess.max() <= ROUNDOFF_REL, (env.env_id, float(excess.max()))
    return D, I, big, stop


def _discrete_round_trip(env, D, I, big, stop, worst):
    """one substep through the kernel's own integrator, restore, invert (qvel' - qvel) / h: qfrc_actuator(s) back, on the envs without an
    active constraint row"""
    torch = env.torch
    m = env.mj_model
    free = np.nonzero(~np.any(I["qfrc_constraint"] != 0, axis=1))[0]
    keep = {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart", "time")}
    env.forward_debug(np.zeros((env.num_envs, m.nu)), 1)
    qd = ((env.t["qvel"] - keep["qvel"]) / m.opt_timestep).contiguous()
    for k, v in keep.items():
        env.t[k].copy_(v)
    Id = _host(env.inverse(qd, discrete=True))
    r = (Id["qfrc_inverse"] - D["qfrc_actuator"])[free]
    excess = np.maximum(np.linalg.norm(r, axis=1) - stop, 0) / big[free]
    worst["discrete_roundoff"] = max(worst.get("discrete_roundoff", 0.0), float(excess.max()) if len(free) else 0.0)
    worst["discrete_envs"] = worst.get("discrete_envs", 0) + len(free)
    assert len(free) == 0 or excess.max() <= ROUNDOFF_REL, float(excess.max())
    return len(free)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_device_round_trip(case, rows):
    """readout qacc -> inverse = readout qfrc_actuator up to phase_solve's stop rule (tol meaninertia max(1, nv) on the gradient norm)
    plus round-off; on the elbow also the discrete round trip through one substep of the kernel's integrator."""
    env = _warm_env(case, rows)
    worst = {}
    D, I, big, stop = _round_trip(env, worst)
    if case == "elbow":
        assert _discrete_round_trip(env, D, I, big, stop, worst) >= env.num_envs // 8
    _report("round trip %s[%s]" % (case, rows), worst)


@pytest.fixture(scope="module")
def zoos(tmp_path_factory):
    import test_actuation_zoo as AZ
    import test_contact_zoo as CZ
    tmp = tmp_path_factory.mktemp("inverse_zoo")
    (tmp / "c").mkdir(); (tmp / "a").mkdir()
    return CZ.build_zoo(tmp / "c"), AZ.build_zoo(tmp / "a", names=["WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS", "SWEEP_16", "SWEEP_40"])


ZOO_CASES = ["contact/" + k for k in ("CAP_CAP", "PLANE_CAP", "CAP_ELL", "ELL_ELL", "COMBO")] + \
            ["actuation/" + k for k in ("WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS", "SWEEP_16", "SWEEP_40")]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", ZOO_CASES)
def test_zoo_round_trip(zoos, name, rows):
    """The round trip on the contact and actuation zoo models (MyoVecEnv.from_model); on the actuation zoo also the discrete one at the
    configurations without an active constraint row."""
    import test_contact_zoo as CZ
    from myosuite_b200 import vec_env
    kind, key = name.split("/")
    if kind == "contact":
        m = zoos[0][key][0]
        cfgs = CZ._configs({key: zoos[0][key]}, key) if key != "COMBO" else CZ._configs(zoos[0], key)
        qpos = np.stack([q for _, q in cfgs]); qvel, act, _ = CZ._state(m, qpos, 5, [lb != "generic" for lb, _ in cfgs])
    else:
        z = zoos[1][key]; m, qpos, qvel, act = z["m"], z["qpos"], z["qvel"], z["act"]
    env = vec_env.MyoVecEnv(None, len(qpos), model=m, row_storage=rows)
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    worst = {}
    D, I, big, stop = _round_trip(env, worst)
    if kind == "actuation":
        _discrete_round_trip(env, D, I, big, stop, worst)
    _report("zoo round trip %s[%s]" % (name, rows), worst)


# ----------------------------------------------------------------------------- GPU: invariance and no side effects
def _bits(D):
    return {k: v.clone() for k, v in D.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("eid,n", [("myoHandPoseRandom-v0", 999), ("myoHandObjHoldRandom-v0", 517), ("myoFatiLegWalk-v0", 333)])
def test_invariance_and_no_side_effects(eid, n):
    """qfrc_inverse and every other output are bit-identical after act, ctrl and the warm start change; an inverse leaves every bound
    tensor bit-identical; twin batches with and without inverses between their 50 steps stay bit-identical."""
    import torch
    from myosuite_b200 import vec_env
    a_env, b_env = (vec_env.MyoVecEnv(eid, n, seed=SEED) for _ in range(2))
    m = a_env.mj_model
    for env in (a_env, b_env):
        env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for step in range(50):
        act = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(a_env.device)
        R = _random_qacc(a_env, a_env.data("qacc")["qacc"], seed=step)
        before = {k: a_env.t[k].clone() for k in BOUND if k in a_env.t}
        for con, disc in ((True, False), (False, True), (True, True)):
            a_env.inverse(R, constraints=con, discrete=disc, fields=ALL)
        torch.cuda.synchronize()
        for k, v in before.items():
            assert _same(v, a_env.t[k]), (step, k)
        if step % 10 == 3:
            # act, ctrl (through a forward pass without substeps) and the warm start do not enter
            ref = _bits(a_env.inverse(R, fields=ALL))
            a_env.t["act"].copy_(torch.rand_like(a_env.t["act"]))
            a_env.forward_debug(np.random.default_rng(step).uniform(0, 1, (n, m.nu)), 0)
            a_env.t["qacc_warmstart"].copy_(torch.randn_like(a_env.t["qacc_warmstart"]))
            got = a_env.inverse(R, fields=ALL)
            for k in ALL:
                assert _same(ref[k], got[k]), (step, k)
            for k, v in before.items():          # the state back for the twin comparison (an env step overwrites ctrl before it reads it)
                a_env.t[k].copy_(v)
        a_env.step(act); b_env.step(act.clone())
        torch.cuda.synchronize()
        for k in BOUND:
            if k in a_env.t:
                assert _same(a_env.t[k], b_env.t[k]), (step, k)
    print("\n%s n %d: 50 twin steps bit-identical with inverses between them" % (eid, n))


@pytest.mark.gpu
def test_unrequested_outputs_untouched():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv("myoHandObjHoldRandom-v0", 100, seed=SEED)
    env.reset(seed=SEED)
    R = _random_qacc(env, env.data("qacc")["qacc"])
    full = _bits(env.inverse(R, fields=ALL))
    torch.cuda.synchronize()
    sent = {k: torch.full_like(v, float("nan")) for k, v in full.items()}
    for ask in (("qfrc_inverse",), ("qfrc_inverse", "contact_force"), ("qfrc_inverse", "actuator_moment", "qfrc_constraint")):
        for v in sent.values():
            v.fill_(float("nan"))
        n0 = env.batch.launches
        env.batch.inverse(stream=env._stream(), qacc=R, **{k: sent[k] for k in ask})
        torch.cuda.synchronize()
        assert env.batch.launches == n0 + 1
        for k, v in sent.items():
            assert torch.equal(v, full[k]) if k in ask else v.isnan().all(), (ask, k)


# ----------------------------------------------------------------------------- GPU: trajectory shape
@pytest.mark.gpu
def test_trajectory_batch_matches_small_batch():
    """10 240 hand states in one physics-only batch (a recorded trajectory as envs) give the same outputs, bit for bit, as the same
    states at other slots of a 64-env batch: results do not depend on the slot."""
    import torch
    from myosuite_b200 import vec_env
    from myosuite_b200 import assets
    m = assets.load("myohand_pose")
    T = 10240
    rng = np.random.default_rng(SEED)
    qpos, qvel, _, _ = _states(m, T, rng, overshoot=0.0, vel=0.5)
    big = vec_env.MyoVecEnv.from_model("myohand_pose", T)
    big.set_state(qpos=qpos, qvel=qvel)
    qacc = torch.as_tensor(rng.normal(0, 50, (T, m.nv)), device=big.device)
    n0 = big.batch.launches
    out = _bits(big.inverse(qacc, fields=ALL))
    assert big.batch.launches == n0 + 1
    small = vec_env.MyoVecEnv.from_model("myohand_pose", 64)
    idx = rng.choice(T, 64, replace=False)
    small.set_state(qpos=qpos[idx], qvel=qvel[idx])
    got = small.inverse(qacc[torch.as_tensor(idx, device=big.device)].contiguous(), fields=ALL)
    torch.cuda.synchronize()
    for k in ALL:
        assert _same(got[k], out[k][torch.as_tensor(idx, device=big.device)]), k
    assert torch.isfinite(out["qfrc_inverse"]).all()


# ----------------------------------------------------------------------------- GPU: input checks and the single-env facade
@pytest.mark.gpu
def test_input_checks_without_launch():
    import torch
    from myosuite_b200 import abi, vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 8, seed=SEED)
    nv = env.mj_model.nv
    good = torch.zeros(8, nv, dtype=torch.float64, device=env.device)
    n0 = env.batch.launches
    for bad in (torch.zeros(8, nv + 1, dtype=torch.float64, device=env.device), torch.zeros(7, nv, dtype=torch.float64, device=env.device),
                good.float(), good.cpu(), good.cpu().numpy()):
        with pytest.raises(ValueError):
            env.inverse(bad)
    out = torch.zeros_like(good)
    with pytest.raises(abi.MyoError, match="unknown flag"):
        env.batch.inverse(flags=4, qacc=good, qfrc_inverse=out)
    with pytest.raises(abi.MyoError, match="required"):
        env.batch.inverse(qacc=good)
    with pytest.raises(abi.MyoError, match="required"):
        env.batch.inverse(qfrc_inverse=out)
    with pytest.raises(KeyError):
        env.inverse(good, fields=("qacc",))
    unbound = abi.Batch(env.dev_model, env.device_index, 8, env.cfg)
    with pytest.raises(abi.MyoError, match="bound"):
        unbound.inverse(qacc=good, qfrc_inverse=out)
    assert env.batch.launches == n0 and unbound.launches == 0
    sv = env.state_version
    env.inverse(good)
    assert env.batch.launches == n0 + 1 and env.state_version == sv


@pytest.mark.gpu
def test_myoenv_mj_inverse():
    from myosuite_b200 import vec_env
    env = vec_env.MyoEnv("myoHandObjHoldRandom-v0", seed=3)
    m = env.mj_model
    env.step(env.action_space.sample())
    L = env.vec.batch
    qacc = np.random.default_rng(0).normal(0, 10, m.nv)
    n0 = L.launches
    r = env.mj_inverse(qacc)
    assert L.launches == n0 + 1
    assert r["qfrc_inverse"].shape == (m.nv,) and r["actuator_moment"].shape == (m.nu, m.nv) and r["contact_force"].shape == (env.vec.dims.maxcon, 6)
    v = env.vec.inverse(env.vec.torch.as_tensor(qacc[None], device=env.vec.device), fields=env.vec.INVERSE_FIELDS)
    for k, x in v.items():
        assert np.array_equal(r[k], x[0].cpu().numpy()), k
    r2 = env.mj_inverse(qacc, constraints=False, discrete=True)
    assert not np.any(r2["qfrc_constraint"]) and not np.array_equal(r2["qfrc_inverse"], r["qfrc_inverse"])


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\ninverse dynamics:")
        for k in sorted(REPORT):
            print("  %-36s %s" % (k, REPORT[k]))
