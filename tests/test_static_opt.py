"""Muscle static optimisation (myo_batch_static_opt, MyoVecEnv.static_opt, MyoEnv.static_opt) against a CPU reference that shares nothing
with the solver (tests/static_opt_ref.py: the problem from the oracle, solved by bounded least squares), and against the forward dynamics
and activation dynamics that the solution is meant to drive.

CPU: the header matches abi.py; the numpy restatement of the dual Newton agrees with lsq_linear on every shipped and zoo model at random
states; the excitation formula takes act to a* through the oracle's own step, including the zoo's tausmooth > 0 muscles.
GPU, on both row storages: every registered base task at its benchmarked shape after random-action steps (act against the CPU reference
with constraints off, muscle gain and bias against the oracle, and a solver-independent KKT certificate on every env); the round trip
through the forward pass and the activation dynamics; the zoo's MUSCLE model and the 40-dof sweep model (the dense solver's n > 36 path);
bit-for-bit independence of batch size, slot and scratch layout; warm starts; no side effects; input checks; the single env; and
computed muscle control of a recorded hand trajectory on the device."""
import ctypes
import os

import numpy as np
import pytest

import static_opt_ref as R
from inverse_oracle import INV_DISCRETE, INV_NOCONSTRAINT, InvOracle
from parity_helpers import _states
from test_mj_data import BOUND, CASES, ROWS, SEED, WARM, _header_struct, _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIPPED = ["myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso"]
ZOO = ["MUSCLE", "WRAP", "SWEEP_40"]
RESERVE = 1.0              # reserve strength rho of the tests (every dof) on the elbow, the hands and the zoo models ...
RESERVE_OF = {"myolegs": 100.0, "myotorso": 100.0}    # ... and on the legs and the torso, whose joint torques are larger by about that
CASE_RESERVE = {"walk_fatigue": 100.0, "stand": 100.0, "torso": 100.0}   # much (DESIGN.md section 2: Newton steps against the scale)
NEWTON_VS_LSQ = 1e-10      # |a_newton - a_lsq|_inf (CPU): 1.9e-14 measured (legs); bvls stops at its own optimality tolerance
ACT_REF = 1e-7             # device act against the oracle-built CPU reference, constraints off: t and G agree to ~1e-12 relative
                           # (test_inverse.py FREE_REL, test_mj_data.py LEN_REL / FRC_REL), amplified by the problem's conditioning and
                           # by bvls's own stopping tolerance; the worst measured is printed
GAIN_REL = 1e-10           # muscle_gain / muscle_bias against the oracle: test_mj_data.py's FRC_REL for actuator_force
KKT_REL = 1e-12            # a == clip(G' lambda / w, 0, 1), with G' lambda recomputed from the dense moments (rounding of the product)
EXCITE_TOL = 1e-12         # act after one step with ctrl against a* where ctrl is not clipped
QFRC_REL = 1e-10           # qfrc_inverse of the static optimisation against myo_batch_inverse's, relative to the env's largest entry
ROUNDOFF_REL = 1e-9        # test_inverse.py's round-trip bound: what exceeds the forward solver's stop rule, relative to the largest term
REPORT = {}


# ----------------------------------------------------------------------------- CPU
def test_static_opt_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_static_opt_buffers")
    assert len(fields) == decls and abi.STATIC_OPT_FIELDS == fields
    assert [n for n, _ in abi.MyoStaticOptBuffers._fields_] == fields and ctypes.sizeof(abi.MyoStaticOptBuffers) == 8 * len(fields)
    assert set(abi.STATIC_OPT_SHAPES) == set(fields) - {"qacc", "weight", "reserve", "lambda0"}
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    p = src[src.index("} myo_static_opt_buffers;"):]
    assert "typedef struct { int32_t max_iter; double tol; } myo_static_opt_params;" in p
    assert [n for n, _ in abi.MyoStaticOptParams._fields_] == ["max_iter", "tol"]
    assert "myo_batch_static_opt" in abi.EXPORTS and "int myo_batch_static_opt(" in src


def _zoo(tmp):
    import test_actuation_zoo as AZ
    return AZ.build_zoo(tmp, names=ZOO)


def _cases(models, tmp, n_shipped=4):
    """(name, model, qpos, qvel, act) at random states (shipped models) and at the zoo's configurations"""
    rng = np.random.default_rng(SEED)
    out = []
    for name in SHIPPED:
        m = models[name]
        qpos, qvel, act, _ = _states(m, n_shipped, rng, overshoot=0.0, vel=0.3)
        out.append((name, m, qpos, qvel, act))
    for name, z in _zoo(tmp).items():
        out.append(("zoo/" + name, z["m"], z["qpos"][:6], z["qvel"][:6], z["act"][:6]))
    return out


def test_dual_newton_matches_lsq(models, tmp_path):
    """The dual Newton (numpy restatement) against bounded least squares on the eliminated problem, with random weights and reserves and
    accelerations around the passive one, with and without constraints: same a, r = t - G a, the stop rule met, and r = t on dofs no
    muscle crosses."""
    from myosuite_b200 import blob
    rng = np.random.default_rng(SEED)
    worst, iters = {}, {}
    for name, m, qpos, qvel, act in _cases(models, tmp_path):
        o = InvOracle(*blob.pack(m))
        for e in range(len(qpos)):
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=np.zeros(m.nu)); o.forward()
            qacc = o.f("qacc").copy() + rng.normal(0, 1, m.nv)
            flags = 0 if e % 2 == 0 else INV_NOCONSTRAINT
            t, G, AM, g, b, _ = R.problem(o, m, qpos[e], qvel[e], act[e], qacc, flags)
            assert np.all(g <= 0)
            w = rng.uniform(0.5, 2.0, m.nu)
            rho = RESERVE_OF.get(name, RESERVE) * rng.uniform(0.5, 2.0, m.nv)
            a, r, lam, it, conv, fn = R.solve_dual_newton(t, G, w, rho)
            assert conv, (name, e, it, fn)
            al, rl = R.solve_lsq(t, G, w, rho)
            err = float(np.abs(a - al).max())
            worst[name] = max(worst.get(name, 0.0), err)
            iters[name] = max(iters.get(name, 0), it)
            assert err <= NEWTON_VS_LSQ, (name, e, err)
            assert np.all((a >= 0) & (a <= 1))
            free = ~np.any(AM != 0, axis=0)
            assert np.all(np.abs(r[free] - t[free]) <= 1e-12 * max(1.0, np.abs(t).max()))        # no muscle crosses: r = t
    print("\ndual Newton vs lsq_linear(bvls), worst |da|: %s; most Newton steps: %s" % ({k: "%.1e" % v for k, v in worst.items()}, iters))


def test_excitation_reaches_target(models, tmp_path):
    """ctrl from the excitation formula, then one oracle_step: act' = a* where ctrl is inside the range, and at a range end act stops short of
    a* on that side; on the hand and on the zoo's MUSCLE model (tausmooth > 0, gear != 1, ctrllimited false, a ctrlrange inside [0, 1])."""
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    rng = np.random.default_rng(SEED)
    z = _zoo(tmp_path)
    worst, clipped, smooth = 0.0, 0, 0
    for m, qpos, qvel, act in ((models["myohand_pose"],) + tuple(_states(models["myohand_pose"], 4, rng, overshoot=0.0, vel=0.3)[:3]),
                               (z["MUSCLE"]["m"], z["MUSCLE"]["qpos"], z["MUSCLE"]["qvel"], z["MUSCLE"]["act"])):
        o = Oracle(*blob.pack(m))
        for e in range(len(qpos)):
            a0 = np.clip(act[e], 0, 1)
            target = np.clip(a0 + rng.normal(0, 0.05, m.nu), 0, 1)
            target[::5] = rng.uniform(0, 1, len(target[::5]))       # some targets out of reach in one step
            ctrl = np.array([R.excitation(m, i, a0[i], target[i]) for i in range(m.nu)])
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=a0, ctrl=ctrl); o.step(1)
            got = o.f("act")
            for i in range(m.nu):
                lo, hi = R.ctrl_range(m, i)
                smooth += int(m.actuator_dynprm[i, 2] > 0)
                if lo < ctrl[i] < hi:
                    worst = max(worst, abs(got[i] - target[i]))
                    assert abs(got[i] - target[i]) <= EXCITE_TOL, (i, got[i], target[i])
                else:
                    clipped += 1
                    # at a range end: act goes as far toward a* as the range allows (a* is out of reach on that side)
                    assert (ctrl[i] == hi and got[i] <= target[i] + EXCITE_TOL) or (ctrl[i] == lo and got[i] >= target[i] - EXCITE_TOL), (i, ctrl[i], got[i], target[i])
    assert clipped > 0 and smooth > 0
    print("\nexcitation: worst |act' - a*| %.1e where not clipped; %d clipped" % (worst, clipped))


# ----------------------------------------------------------------------------- GPU helpers
def _host(D):
    return {k: v.cpu().numpy().copy() for k, v in D.items()}


ALL = ("act", "reserve_force", "ctrl", "actuator_force", "muscle_gain", "muscle_bias", "qfrc_inverse", "lambda", "niter", "converged",
       "residual")


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


def kkt(env, S, qacc, rho, w, con=True, disc=False, rows=None):
    """The solver-independent certificate on every env (or on the envs `rows` selects): 0 <= a <= 1 exactly, a = clip(G' lambda / w, 0, 1)
    with G' lambda from the dense moments and the returned gain, reserve_force = rho^2 lambda exactly, and the primal residual within the
    stop rule."""
    m = env.mj_model
    M = _host(env.inverse(qacc, constraints=con, discrete=disc, fields=("qfrc_inverse", "actuator_moment")))
    if rows is not None:
        M, S = {k: v[rows] for k, v in M.items()}, {k: v[rows] for k, v in S.items()}
    a, lam, g, b, r = S["act"], S["lambda"], S["muscle_gain"], S["muscle_bias"], S["reserve_force"]
    assert np.all((a >= 0) & (a <= 1))
    assert np.array_equal(r, (rho ** 2)[None, :] * lam)
    # the inverse pass is the inverse's; the two kernels contract multiply-adds differently
    qs = np.maximum(np.abs(M["qfrc_inverse"]).max(1, keepdims=True), 1e-6)      # (1e-6: passive states where it is round-off alone)
    assert np.all(np.abs(S["qfrc_inverse"] - M["qfrc_inverse"]) <= QFRC_REL * qs), float((np.abs(S["qfrc_inverse"] - M["qfrc_inverse"]) / qs).max())
    AM = M["actuator_moment"]
    s = np.einsum("nmi,ni->nm", AM, lam) * g
    scale = np.maximum(np.abs(np.einsum("nmi,ni->nm", np.abs(AM), np.abs(lam)) * g), 1e-300)
    ref = np.clip(s / w[None, :], 0, 1)
    kerr = float(np.max(np.abs(a - ref) / np.maximum(scale / w[None, :], 1.0)))
    assert kerr <= KKT_REL, kerr
    t = S["qfrc_inverse"] - np.einsum("nmi,nm->ni", AM, b)
    F = np.einsum("nmi,nm->ni", AM, g * a) + r - t
    terms = np.einsum("nmi,nm->ni", np.abs(AM), np.abs(g * a)) + np.abs(r) + np.abs(t) + np.abs(np.einsum("nmi,nm->ni", AM, b))
    thr = 1e-12 * np.maximum(1.0, np.abs(t).max(1))
    assert np.all(S["converged"] == 1) and np.all(S["residual"] <= thr * (1 + 1e-9)), int(np.sum(S["converged"] != 1))
    slack = 64 * np.finfo(float).eps * terms.max(1)          # the host's recomputation of F rounds differently from the device's
    assert np.all(np.abs(F).max(1) <= thr + slack), float((np.abs(F).max(1) / (thr + slack)).max())
    return kerr, float((np.abs(F).max(1) / thr).max())


def _report(key, worst, extra=""):
    REPORT[key] = extra + ", ".join("%s %.1e" % (k, v) if isinstance(v, float) else "%s %s" % (k, v) for k, v in sorted(worst.items()))
    print("\n%s %s" % (key, REPORT[key]))


# ----------------------------------------------------------------------------- GPU: registered tasks
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_static_opt_vs_reference(case, rows):
    """At the benchmarked shape after random-action steps, with the readout's qacc: the KKT certificate on every env (constraints on and
    off); act against the oracle-built lsq reference and muscle_gain / muscle_bias against the oracle on 24 envs (constraints off)."""
    import torch
    from test_inverse import _inv_oracles
    env = _warm_env(case, rows)
    m, n = env.mj_model, env.num_envs
    Q = env.data("qacc")["qacc"].clone()
    rho0 = CASE_RESERVE.get(case, RESERVE)
    rho = np.full(m.nv, rho0); w = np.ones(m.nu)
    worst = {}
    for con in (True, False):
        S = _host(env.static_opt(Q, rho0, constraints=con, fields=ALL))
        k, f = kkt(env, S, Q, rho, w, con=con)
        worst["kkt_%s" % con] = k; worst["F/stop_%s" % con] = f
        worst["niter_max_%s" % con] = int(S["niter"].max()); worst["niter_mean_%s" % con] = float(S["niter"].mean())
    torch.cuda.synchronize()
    st = env.get_env_state()
    QH = Q.cpu().numpy()
    oracles = _inv_oracles(env)
    wa = wg = 0.0
    for e in np.random.default_rng(SEED).choice(n, min(n, 24), replace=False):
        o = oracles.get(st["env_prm"][e] if "env_prm" in st else None)
        t, G, AM, g, b, _ = R.problem(o, m, st["qpos"][e], st["qvel"][e], st["act"][e, :m.na], QH[e], INV_NOCONSTRAINT)
        al, _ = R.solve_lsq(t, G, w, rho)
        wa = max(wa, float(np.abs(S["act"][e] - al).max()))
        gs = max(np.abs(g).max(), np.abs(b).max(), 1e-300)
        wg = max(wg, float(max(np.abs(S["muscle_gain"][e] - g).max(), np.abs(S["muscle_bias"][e] - b).max()) / gs))
    worst["act_vs_lsq"] = wa; worst["gain_bias"] = wg
    _report("%s[%s]" % (case, rows), worst)
    assert wa <= ACT_REF and wg <= GAIN_REL


# ----------------------------------------------------------------------------- GPU: round trips
def _round_trip(env, Q, worst, rho0, con=True, disc=False):
    """act := a*, qfrc_applied := r, one mj_step; the inverse of that step's qacc (with the same flags) gives G a* + AM' b + r back.  The
    step always runs its constraints, so without constraints (and for the discrete inverse, as in test_inverse.py) only the envs whose step
    has no active constraint row are compared."""
    m, n = env.mj_model, env.num_envs
    S = env.static_opt(Q, rho0, constraints=con, discrete=disc, fields=ALL)
    st = {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart", "time")}
    r = env.rollout(S["ctrl"][:, None].contiguous(), qfrc_applied=S["reserve_force"][:, None].contiguous(),
                    initial_state=dict(st, act=S["act"].contiguous()), fields=("qvel", "qacc", "act"))
    qacc = ((r["qvel"][:, 0] - st["qvel"]) / m.opt_timestep).contiguous() if disc else r["qacc"][:, 0].contiguous()
    I = _host(env.inverse(qacc, constraints=con, discrete=disc, fields=("qfrc_inverse", "qfrc_constraint", "actuator_moment")))
    fc = _host(env.inverse(r["qacc"][:, 0].contiguous(), fields=("qfrc_constraint",)))["qfrc_constraint"]
    keep = np.arange(n) if (con and not disc) else np.nonzero(~np.any(fc != 0, axis=1))[0]
    H = _host(S)
    act_f = np.einsum("nmi,nm->ni", I["actuator_moment"], H["actuator_force"])
    err = (I["qfrc_inverse"] - act_f - H["reserve_force"])[keep]
    tol = float(env.cfg.solver_tolerance) or 1e-10
    stop = tol * m.stat_meaninertia * max(1, m.nv)
    big = np.maximum.reduce([np.abs(act_f).max(1), np.abs(H["reserve_force"]).max(1), np.abs(I["qfrc_constraint"]).max(1),
                             np.abs(I["qfrc_inverse"]).max(1), np.full(n, 1e-300)])[keep]
    excess = np.maximum(np.linalg.norm(err, axis=1) - stop, 0) / big
    key = "roundtrip_%s%s" % ("con" if con else "free", "_disc" if disc else "")
    worst[key] = max(worst.get(key, 0.0), float(excess.max()) if len(keep) else 0.0)
    worst[key + "_envs"] = worst.get(key + "_envs", 0) + len(keep)
    assert len(keep) == 0 or excess.max() <= ROUNDOFF_REL, (key, float(excess.max()))
    # the excitation: one step with ctrl from the current act
    r2 = env.rollout(S["ctrl"][:, None].contiguous(), initial_state=st, fields=("act",))
    got, ctrl, tgt = r2["act"][:, 0].cpu().numpy(), H["ctrl"], H["act"]
    lo = np.array([R.ctrl_range(m, i)[0] for i in range(m.nu)]); hi = np.array([R.ctrl_range(m, i)[1] for i in range(m.nu)])
    inside = (ctrl > lo) & (ctrl < hi)
    e1 = float(np.abs(got - tgt)[inside].max()) if inside.any() else 0.0
    worst["excitation"] = max(worst.get("excitation", 0.0), e1)
    assert e1 <= EXCITE_TOL, e1
    at_lo, at_hi = ctrl == lo[None, :], ctrl == hi[None, :]
    at_end = ~inside
    assert np.all(at_lo | at_hi | inside)                                   # clipped ctrl sits at a range end ...
    assert np.all(got[at_hi] <= tgt[at_hi] + EXCITE_TOL) and np.all(got[at_lo & ~at_hi] >= tgt[at_lo & ~at_hi] - EXCITE_TOL)   # ... a* out of reach there
    worst["ctrl_clipped_share"] = float(at_end.mean())
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", ["elbow", "hand_pose", "hold", "walk_fatigue", "torso"])
def test_round_trip_through_forward(case, rows):
    """The solution drives the requested acceleration: with constraints, without, and with discrete=True (constraints off)."""
    env = _warm_env(case, rows)
    Q = env.data("qacc")["qacc"].clone()
    worst = {}
    for con, disc in ((True, False), (False, False), (False, True)):
        _round_trip(env, Q, worst, CASE_RESERVE.get(case, RESERVE), con=con, disc=disc)
    _report("round trip %s[%s]" % (case, rows), worst)


@pytest.fixture(scope="module")
def zoo(tmp_path_factory):
    return _zoo(tmp_path_factory.mktemp("static_opt_zoo"))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", ZOO)
def test_zoo(zoo, name, rows):
    """The MUSCLE model (gear != 1, tausmooth > 0, ctrllimited false) and SWEEP_40 (nv = 40 > 36: the dense solver's row fallback):
    KKT certificate, act against the lsq reference, the round trips."""
    from myosuite_b200 import blob, vec_env
    z = zoo[name]; m = z["m"]
    assert m.nu > 0
    env = vec_env.MyoVecEnv(None, len(z["qpos"]), model=m, row_storage=rows)
    env.set_state(qpos=z["qpos"], qvel=z["qvel"], act=np.clip(z["act"], 0, 1))
    Q = env.data("qacc")["qacc"].clone()
    worst = {}
    S = _host(env.static_opt(Q, RESERVE, fields=ALL))
    worst["kkt"], worst["F/stop"] = kkt(env, S, Q, np.full(m.nv, RESERVE), np.ones(m.nu))
    worst["niter_max"] = int(S["niter"].max())
    S0 = _host(env.static_opt(Q, RESERVE, constraints=False, fields=ALL))
    o = InvOracle(*blob.pack(m))
    st = env.get_env_state(); QH = Q.cpu().numpy(); wa = 0.0
    for e in range(min(16, env.num_envs)):
        t, G, _, g, b, _ = R.problem(o, m, st["qpos"][e], st["qvel"][e], st["act"][e], QH[e], INV_NOCONSTRAINT)
        al, _ = R.solve_lsq(t, G, np.ones(m.nu), np.full(m.nv, RESERVE))
        wa = max(wa, float(np.abs(S0["act"][e] - al).max()))
    worst["act_vs_lsq"] = wa
    assert wa <= ACT_REF
    for con, disc in ((True, False), (False, False), (False, True)):
        _round_trip(env, Q, worst, RESERVE, con=con, disc=disc)
    _report("zoo %s[%s]" % (name, rows), worst)


# ----------------------------------------------------------------------------- GPU: bit for bit
@pytest.mark.gpu
def test_batch_slot_and_layout_independence():
    """4096 hand envs against the same states at other slots of a 64-env batch, and against a batch at another contact capacity (another
    scratch layout): every output bit-identical.  A warm start from the returned lambda converges in at most one step."""
    import torch
    from myosuite_b200 import assets, vec_env
    m = assets.load("myohand_pose")
    T = 4096
    rng = np.random.default_rng(SEED)
    qpos, qvel, act, _ = _states(m, T, rng, overshoot=0.0, vel=0.5)
    big = vec_env.MyoVecEnv.from_model("myohand_pose", T)
    big.set_state(qpos=qpos, qvel=qvel, act=act)
    qacc = torch.as_tensor(rng.normal(0, 20, (T, m.nv)), device=big.device)
    w = torch.as_tensor(rng.uniform(0.5, 2, m.nu), device=big.device)
    n0 = big.batch.launches
    out = big.static_opt(qacc, RESERVE, weight=w, fields=ALL)
    assert big.batch.launches == n0 + 1
    idx = rng.choice(T, 64, replace=False); it = torch.as_tensor(idx, device=big.device)
    for maxcon in (None, 24):
        small = vec_env.MyoVecEnv.from_model("myohand_pose", 64, **({} if maxcon is None else dict(maxcon=maxcon)))
        small.set_state(qpos=qpos[idx], qvel=qvel[idx], act=act[idx])
        got = small.static_opt(qacc[it].contiguous(), RESERVE, weight=w, fields=ALL)
        torch.cuda.synchronize()
        for k in ALL:
            assert _same(got[k], out[k][it]), (maxcon, k)
    assert torch.all(out["converged"] == 1) and torch.isfinite(out["act"]).all()
    warm = big.static_opt(qacc, RESERVE, weight=w, warmstart=out["lambda"].contiguous(), fields=ALL)
    assert int(warm["niter"].max()) <= 1 and torch.all(warm["converged"] == 1)
    print("\nhand 4096: Newton steps mean %.2f max %d; from the returned lambda max %d"
          % (out["niter"].double().mean().item(), out["niter"].max().item(), warm["niter"].max().item()))


@pytest.mark.gpu
def test_no_side_effects_and_unrequested_outputs():
    """Twin batches with and without static_opt calls between their 50 steps stay bit-identical, every bound tensor is untouched by a call,
    and outputs that are not requested are not written."""
    import torch
    from myosuite_b200 import vec_env
    eid, n = "myoHandObjHoldRandom-v0", 517
    a_env, b_env = (vec_env.MyoVecEnv(eid, n, seed=SEED) for _ in range(2))
    m = a_env.mj_model
    for env in (a_env, b_env):
        env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for step in range(50):
        act = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(a_env.device)
        Q = a_env.data("qacc")["qacc"].clone()
        before = {k: a_env.t[k].clone() for k in BOUND if k in a_env.t}
        a_env.static_opt(Q, RESERVE, fields=ALL)
        a_env.static_opt(Q, RESERVE, constraints=False, discrete=True)
        torch.cuda.synchronize()
        for k, v in before.items():
            assert _same(v, a_env.t[k]), (step, k)
        a_env.step(act); b_env.step(act.clone())
        torch.cuda.synchronize()
        for k in BOUND:
            if k in a_env.t:
                assert _same(a_env.t[k], b_env.t[k]), (step, k)
    from myosuite_b200 import abi
    Q = a_env.data("qacc")["qacc"].clone()
    full = {k: v.clone() for k, v in a_env.static_opt(Q, RESERVE, fields=ALL).items()}
    reserve = torch.full((m.nv,), RESERVE, dtype=torch.float64, device=a_env.device)
    params = abi.MyoStaticOptParams(max_iter=50, tol=1e-12)
    for ask in (("act",), ("act", "ctrl", "lambda"), ("act", "muscle_gain", "niter", "residual")):
        sent = {k: torch.full_like(v, -7 if v.dtype == torch.int32 else float("nan")) for k, v in full.items()}
        n0 = a_env.batch.launches
        a_env.batch.static_opt(params, stream=a_env._stream(), qacc=Q, reserve=reserve, **{k: sent[k] for k in ask})
        torch.cuda.synchronize()
        assert a_env.batch.launches == n0 + 1
        for k, v in sent.items():
            untouched = (v == -7).all() if v.dtype == torch.int32 else v.isnan().all()
            assert torch.equal(v, full[k]) if k in ask else untouched, (ask, k)


@pytest.mark.gpu
def test_input_checks_without_launch():
    import torch
    from myosuite_b200 import abi, vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 8, seed=SEED)
    nv, nu = env.mj_model.nv, env.mj_model.nu
    good = torch.zeros(8, nv, dtype=torch.float64, device=env.device)
    n0 = env.batch.launches
    for bad in (torch.zeros(8, nv + 1, dtype=torch.float64, device=env.device), good.float(), good.cpu()):
        with pytest.raises(ValueError):
            env.static_opt(bad, 1.0)
    for kw in (dict(reserve=0.0), dict(reserve=-1.0), dict(reserve=float("nan")), dict(reserve=np.ones(nv + 1)),
               dict(reserve=1.0, weight=np.zeros(nu)), dict(reserve=1.0, weight=torch.ones(nu, device=env.device) * -1),
               dict(reserve=1.0, max_iter=-1), dict(reserve=1.0, tol=-1.0), dict(reserve=1.0, tol=float("inf")),
               dict(reserve=1.0, warmstart=torch.zeros(8, nv + 1, dtype=torch.float64, device=env.device))):
        with pytest.raises(ValueError):
            env.static_opt(good, **kw)
    with pytest.raises(KeyError):
        env.static_opt(good, 1.0, fields=("qacc",))
    out = torch.zeros(8, nu, dtype=torch.float64, device=env.device)
    rho = torch.ones(nv, dtype=torch.float64, device=env.device)
    P = abi.MyoStaticOptParams(max_iter=50, tol=1e-12)
    for params, flags, bufs, msg in ((P, 4, dict(qacc=good, reserve=rho, act=out), "unknown flag"),
                                     (P, 0, dict(reserve=rho, act=out), "required"), (P, 0, dict(qacc=good, act=out), "required"),
                                     (P, 0, dict(qacc=good, reserve=rho), "required"),
                                     (abi.MyoStaticOptParams(max_iter=-1, tol=0.0), 0, dict(qacc=good, reserve=rho, act=out), "max_iter"),
                                     (abi.MyoStaticOptParams(max_iter=5, tol=-1.0), 0, dict(qacc=good, reserve=rho, act=out), "tol"),
                                     (abi.MyoStaticOptParams(max_iter=5, tol=float("nan")), 0, dict(qacc=good, reserve=rho, act=out), "finite")):
        with pytest.raises(abi.MyoError, match=msg):
            env.batch.static_opt(params, flags=flags, **bufs)
    unbound = abi.Batch(env.dev_model, env.device_index, 8, env.cfg)
    with pytest.raises(abi.MyoError, match="bound"):
        unbound.static_opt(P, qacc=good, reserve=rho, act=out)
    assert env.batch.launches == n0 and unbound.launches == 0
    sv = env.state_version
    env.static_opt(good, 1.0)
    assert env.batch.launches == n0 + 1 and env.state_version == sv


@pytest.mark.gpu
def test_myoenv_static_opt():
    from myosuite_b200 import vec_env
    env = vec_env.MyoEnv("myoHandPoseRandom-v0", seed=3)
    m = env.mj_model
    env.step(env.action_space.sample())
    qacc = np.random.default_rng(0).normal(0, 10, m.nv)
    L = env.vec.batch
    n0 = L.launches
    r = env.static_opt(qacc, RESERVE, fields=ALL)
    assert L.launches == n0 + 1
    assert r["act"].shape == (m.nu,) and r["reserve_force"].shape == (m.nv,) and isinstance(r["niter"], int) and r["converged"] == 1
    v = env.vec.static_opt(env.vec.torch.as_tensor(qacc[None], device=env.vec.device), RESERVE, fields=ALL)
    for k, x in v.items():
        assert np.array_equal(np.asarray(r[k]), x[0].cpu().numpy()), k


# ----------------------------------------------------------------------------- GPU: computed muscle control on the device
CMC_ENVS, CMC_STEPS, KP, KV = 256, 200, 100.0, 20.0
CMC_RESERVE = 10.0         # reserves ten times stronger than on the hand's other tests; the reserve share of the generalized force is reported


def _reference(h):
    """position, velocity and acceleration of the hand trajectory fixture at timestep h (tests/golden/make_hand_trajectory.py: every 5th
    frame of MyoSuite's tutorial 6 trajectory), from a cubic spline through its frames"""
    from scipy.interpolate import CubicSpline
    z = np.load(os.path.join(ROOT, "tests", "golden", "hand_trajectory.npz"))
    q, dt = z["qpos"].astype(np.float64), float(z["dt"])
    sp = CubicSpline(np.arange(len(q)) * dt, q, axis=0)
    tt = np.arange(0, (len(q) - 1) * dt, h)
    return sp(tt), sp(tt, 1), sp(tt, 2)


@pytest.mark.gpu
def test_cmc_tracks_hand_trajectory():
    """256 hand envs start at different frames of the trajectory; each step computes qacc_d = acc_ref + 20 (vel_ref - qvel) + 100 (pos_ref -
    qpos), solves the static optimisation, rolls one mj_step out with ctrl and reserve_force and adopts the state.  The RMS tracking error
    over all joints and 200 steps is at least 10x below that of the same starts with zero ctrl and no reserves, and at least 8x below on
    every joint the reference moves by more than 0.1 rad over the window (10.0x to 15.3x measured on an H100).  (On the joints it holds nearly still the passive hand stays within about 1e-3
    rad, while the muscles' one-step activation lag costs CMC about as much: the per-joint ratios are reported.)"""
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv.from_model("myohand_pose", CMC_ENVS)
    m = env.mj_model
    pos, vel, acc = _reference(m.opt_timestep)
    starts = np.random.default_rng(SEED).integers(0, len(pos) - CMC_STEPS - 1, CMC_ENVS)
    dev = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=env.device)
    P, V, A, st0 = dev(pos), dev(vel), dev(acc), torch.as_tensor(starts, device=env.device)
    errs, shares, iters, unconv = {}, [], [], []
    for mode in ("cmc", "passive"):
        env.set_state(qpos=pos[starts], qvel=vel[starts], act=np.zeros((CMC_ENVS, m.na)))
        sq = torch.zeros(m.nq, dtype=torch.float64, device=env.device)
        for k in range(CMC_STEPS):
            i0 = st0 + k
            q, v = env.t["qpos"], env.t["qvel"]
            if mode == "cmc":
                qd = (A[i0] + KV * (V[i0] - v) + KP * (P[i0] - q)).contiguous()
                S = env.static_opt(qd, CMC_RESERVE, fields=("ctrl", "reserve_force", "converged", "niter", "actuator_force"))
                unconv.append(float((S["converged"] != 1).double().mean().item()))
                ctrl, qf = S["ctrl"], S["reserve_force"]
                musc = torch.einsum("nmi,nm->ni", env.inverse(qd, fields=("actuator_moment",))["actuator_moment"], S["actuator_force"])
                shares.append((qf.abs().sum(1) / (qf.abs().sum(1) + musc.abs().sum(1)).clamp_min(1e-300)).mean().item())
                iters.append(S["niter"].double().mean().item())
            else:
                ctrl, qf = torch.zeros(CMC_ENVS, m.nu, dtype=torch.float64, device=env.device), None
            r = env.rollout(ctrl[:, None].contiguous(), qfrc_applied=None if qf is None else qf[:, None].contiguous())
            for key in ("qpos", "qvel", "act", "time"):
                env.t[key].copy_(r[key][:, 0])
            env.t["qacc_warmstart"].copy_(r["qacc"][:, 0])
            sq += ((env.t["qpos"] - P[i0 + 1]) ** 2).sum(0)
        errs[mode] = torch.sqrt(sq / (CMC_STEPS * CMC_ENVS)).cpu().numpy()
    ratio = errs["passive"] / np.maximum(errs["cmc"], 1e-300)
    moving = np.array([np.ptp(pos[s:s + CMC_STEPS + 1, j]) for s in starts for j in range(m.nq)]).reshape(CMC_ENVS, m.nq).mean(0) > 0.1
    pooled = float(np.sqrt(np.mean(errs["passive"] ** 2)) / np.sqrt(np.mean(errs["cmc"] ** 2)))
    REPORT["cmc"] = ("per-joint RMS error: CMC max %.2e mean %.2e rad, passive max %.2e mean %.2e, pooled ratio %.1f, worst ratio on the %d "
                     "moving joints %.1f, per joint %s; reserve share of "
                     "|generalized force| %.3f; Newton steps per solve %.2f; solves stopped unconverged at max_iter %.4f"
                     % (errs["cmc"].max(), errs["cmc"].mean(), errs["passive"].max(), errs["passive"].mean(), pooled, int(moving.sum()),
                        ratio[moving].min(), np.round(ratio, 1).tolist(), float(np.mean(shares)),
                        float(np.mean(iters)), float(np.mean(unconv))))
    print("\n" + REPORT["cmc"])
    assert pooled >= 10 and moving.sum() >= 8 and np.all(ratio[moving] >= 8), (pooled, ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nmuscle static optimisation:")
        for k in sorted(REPORT):
            print("  %-36s %s" % (k, REPORT[k]))
