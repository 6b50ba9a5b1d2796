"""mj_step rollouts (myo_batch_rollout, MyoVecEnv.rollout, MyoEnv.mj_rollout) against the env step, the CPU oracle and the inverse
dynamics.

CPU: the myo_rollout_buffers field order against abi.py; the oracle with qfrc_applied (tests/rollout_oracle.c) on every shipped model and
the sweep models (the force enters qfrc_smooth exactly, it moves qacc by M^-1 f where no constraint row exists, and at its default zero
the forward pass and the step are bit-identical to the oracle's own).

GPU, on both row storages where physics is compared: bit-equality with env steps of the same ctrl; every registered base task and the
contact and sweep zoo models against the oracle with random ctrl and applied forces; the round trip with the discrete inverse; no side
effects; start state, resumption and slot independence; input checks and the single-env facade."""
import ctypes
import os

import numpy as np
import pytest

from parity_helpers import _in_regime, _states, relerr
from rollout_oracle import AppliedOracle
from test_inverse import ROUNDOFF_REL, SHIPPED, _sweeps, _tol, qM_dense
from test_mj_data import BOUND, CASES, ROWS, SEED, WARM, _header_struct, _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
APPLIED_REL = 1e-12        # qacc(f) - qacc(0) against M^-1 f, relative to the largest of the three
QPOS_ATOL, QVEL_REL, QACC_REL = 2e-7, 1e-5, 1e-6        # the mid-episode bounds of test_product_parity.py
MAX_SKIP = 0.25            # largest share of the checked envs outside the contact regime or with dropped contacts
N_ORACLE = 48              # envs replayed on the oracle per case and shape
REPORT = {}
# the base tasks at their benchmarked shapes; the walk without fatigue (a rollout runs no fatigue, and the env step has to match it)
ROLL_CASES = {("walk" if k == "walk_fatigue" else k): (("myoLegWalk-v0", n) if k == "walk_fatigue" else (eid, n)) for k, (eid, n) in CASES.items()}


# ----------------------------------------------------------------------------- CPU
def test_rollout_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_rollout_buffers")
    assert len(fields) == decls and abi.ROLLOUT_FIELDS == fields
    assert [n for n, _ in abi.MyoRolloutBuffers._fields_] == fields and ctypes.sizeof(abi.MyoRolloutBuffers) == 8 * len(fields)
    assert set(abi.ROLLOUT_SHAPES) | {"overflow"} | {"ctrl", "qfrc_applied"} | set(abi.ROLLOUT_STATE.values()) == set(fields)
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert src.index("} myo_inverse_buffers;") < src.index("} myo_rollout_buffers;") < src.index("int myo_batch_rollout(")
    assert "myo_batch_rollout" in abi.EXPORTS


def _oracle_models(models, tmp_path):
    ms = {k: models[k] for k in SHIPPED}
    ms.update(_sweeps(tmp_path))
    return ms


def test_oracle_applied_force(models, tmp_path):
    """qfrc_smooth(f) - qfrc_smooth(0) = f to round-off at any state; qacc(f) - qacc(0) = M^-1 f (numpy solve with the oracle's qM) at the
    states without a constraint row; the field is zero after oracle_reset."""
    from myosuite_b200 import blob
    rng = np.random.default_rng(SEED)
    worst, free = {}, 0
    for name, m in _oracle_models(models, tmp_path).items():
        o = AppliedOracle(*blob.pack(m))
        assert not np.any(o.f("qfrc_applied"))
        qpos, qvel, act, ctrl = _states(m, 32, rng, overshoot=0.0, vel=0.3)
        for e in range(len(qpos)):
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
            s0, a0, nefc = o.f("qfrc_smooth").copy(), o.f("qacc").copy(), o.nefc
            f = rng.normal(0, 1, m.nv) * max(np.abs(s0).max(), 1e-3)
            o.set(qfrc_applied=f); o.forward()
            s1, a1 = o.f("qfrc_smooth").copy(), o.f("qacc").copy()
            assert o.nefc == nefc
            scale = max(np.abs(s0).max(), np.abs(f).max())
            serr = float(np.abs((s1 - s0) - f).max() / scale)
            w = worst.setdefault(name, [0.0, 0.0])
            w[0] = max(w[0], serr)
            assert serr <= 4 * np.finfo(float).eps, (name, e, serr)
            if nefc == 0:
                ref = np.linalg.solve(qM_dense(m, o.f("qM")), f)
                err = float(np.abs((a1 - a0) - ref).max() / max(np.abs(a0).max(), np.abs(a1).max(), np.abs(ref).max()))
                w[1] = max(w[1], err); free += 1
                assert err <= APPLIED_REL, (name, e, err)
            o.reset()
            assert not np.any(o.f("qfrc_applied"))
    print("\napplied force, worst relative (qfrc_smooth, qacc over %d constraint-free states): %s" % (free, {k: "%.1e %.1e" % tuple(v) for k, v in worst.items()}))
    assert free >= 10


def test_oracle_default_zero_bit_identical(models, tmp_path):
    """With qfrc_applied at its default zero, the forward pass and 20 steps of the oracle with the applied force are bit-identical to
    oracle_forward / oracle_step: the same state, qacc, qfrc_smooth and qfrc_constraint."""
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    rng = np.random.default_rng(SEED)
    for name, m in _oracle_models(models, tmp_path).items():
        I, D = blob.pack(m)
        a, b = Oracle(I, D), AppliedOracle(I, D)
        qpos, qvel, act, ctrl = _states(m, 3, rng)
        for e in range(len(qpos)):
            for o in (a, b):
                o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e])
            assert not np.any(b.f("qfrc_applied"))
            for run in ("forward", "step"):
                for o in (a, b):
                    o.forward() if run == "forward" else o.step(20)
                for k in ("qpos", "qvel", "act", "qacc", "qacc_warmstart", "qacc_smooth", "qfrc_smooth", "qfrc_constraint", "time"):
                    assert np.array_equal(a.f(k).view(np.int64), b.f(k).view(np.int64)), (name, e, run, k)


# ----------------------------------------------------------------------------- GPU helpers
def _warm(eid, n, rows, **kw):
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv(eid, n, seed=SEED, row_storage=rows, **kw)
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(WARM):
        env.step((torch.rand(n, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
    return env, g


def _report(key, text):
    REPORT[key] = text
    print("\n%s %s" % (key, text))


def _bits(D):
    return {k: v.clone() for k, v in D.items()}


# ----------------------------------------------------------------------------- GPU: the env step, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(ROLL_CASES))
def test_rollout_equals_env_steps(case, rows):
    """8 intervals of frame_skip substeps with the next 8 actions as ctrl (normalize_act off, auto-reset off) against 8 env steps of the
    same batch from the same state: qpos, qvel, act, qacc (the stored warm start) and time bit-equal at every interval, overflow equal."""
    import torch
    eid, n = ROLL_CASES[case]
    env, g = _warm(eid, n, rows, normalize_act=False, auto_reset=False)
    m = env.mj_model
    acts = [(torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device) for _ in range(8)]
    ctrl = torch.stack(acts, 1).double().contiguous()
    out = env.rollout(ctrl, substeps=env.frame_skip, fields=env.ROLLOUT_FIELDS)
    env.t["overflow"].zero_()
    diff = {}
    for t in range(8):
        env.step(acts[t])
        for k, s in (("qpos", "qpos"), ("qvel", "qvel"), ("act", "act"), ("qacc", "qacc_warmstart"), ("time", "time")):
            ref = env.t[s][:, :m.na] if k == "act" else env.t[s]
            if not _same(out[k][:, t], ref):
                diff.setdefault(k, []).append(t)
    torch.cuda.synchronize()
    assert not diff, diff
    assert torch.equal(out["overflow"] != 0, env.t["overflow"] != 0)
    _report("step %s[%s]" % (case, rows), "n %d: 8 intervals of %d substeps bit-equal, %d envs with dropped contacts" % (n, env.frame_skip, int((out["overflow"] != 0).sum())))


# ----------------------------------------------------------------------------- GPU: the oracle, with applied forces
@pytest.fixture(scope="module")
def zoos(tmp_path_factory):
    import test_actuation_zoo as AZ
    import test_contact_zoo as CZ
    tmp = tmp_path_factory.mktemp("rollout_zoo")
    (tmp / "c").mkdir(); (tmp / "a").mkdir()
    return CZ.build_zoo(tmp / "c", names=None), AZ.build_zoo(tmp / "a", names=["SWEEP_16", "SWEEP_40"])


ORACLE_CASES = list(ROLL_CASES) + ["contact/COMBO", "actuation/SWEEP_16", "actuation/SWEEP_40"]


def _oracle_env(name, rows, zoos):
    import test_contact_zoo as CZ
    from myosuite_b200 import vec_env
    if name in ROLL_CASES:
        return _warm(*ROLL_CASES[name], rows)[0], None
    kind, key = name.split("/")
    if kind == "contact":
        m = zoos[0][key][0]
        cfgs = CZ._configs(zoos[0], key)
        qpos = np.stack([q for _, q in cfgs]); qvel, act, _ = CZ._state(m, qpos, 5, [lb != "generic" for lb, _ in cfgs])
    else:
        z = zoos[1][key]; m, qpos, qvel, act = z["m"], z["qpos"], z["qvel"], z["act"]
    env = vec_env.MyoVecEnv(None, len(qpos), model=m, row_storage=rows)
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    return env, 5


def _load(o, env, S, e):
    m = env.mj_model
    o.reset()
    o.set(qpos=S["qpos"][e], qvel=S["qvel"][e], act=S["act"][e, :m.na], qacc_warmstart=S["qacc_warmstart"][e])
    o.f("time")[:] = S["time"][e]
    o.f("wrap_warm")[:] = 1


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", ORACLE_CASES)
def test_rollout_vs_oracle(zoos, name, rows):
    """Random ctrl (a fifth of it outside [0, 1]) and qfrc_applied scaled to each env's largest qfrc_actuator, in two shapes: frame_skip
    intervals of one substep, and one interval of frame_skip substeps.  The oracle replays each checked env with the kernel's wrap rule
    (roots cold at the start of every interval) and is held to the mid-episode bounds at every interval."""
    import torch
    from test_product_parity import Oracles
    env, fs = _oracle_env(name, rows, zoos)
    fs = fs or env.frame_skip
    m, n = env.mj_model, env.num_envs
    S = env.get_env_state()
    fa = env.data("qfrc_actuator")["qfrc_actuator"].abs().amax(1).clamp_min(1e-3).cpu().numpy()
    rng = np.random.default_rng(SEED)
    envs = np.sort(rng.choice(n, min(N_ORACLE, n), replace=False))
    oracles = None
    if name in ROLL_CASES:          # (the hold task's per-env object sizes are patched into copies of the model, as for the env step)
        oracles = Oracles(env)
        oracles.Oracle, oracles.base = AppliedOracle, AppliedOracle(env.I, env.D)
    worst, cnt = dict(qpos=0.0, qvel=0.0, qacc=0.0), dict(checked=0, skipped=0)
    for substeps, nstep in ((1, fs), (fs, 1)):
        ctrl = rng.uniform(-0.25, 1.25, (n, nstep, m.nu))
        f = rng.normal(0, 0.5, (n, nstep, m.nv)) * fa[:, None, None]
        out = env.rollout(torch.as_tensor(ctrl, device=env.device), qfrc_applied=torch.as_tensor(f, device=env.device), substeps=substeps,
                          fields=env.ROLLOUT_FIELDS)
        O = {k: v.cpu().numpy() for k, v in out.items()}
        for e in envs:
            if O["overflow"][e]:
                cnt["skipped"] += 1
                continue
            o = oracles.get(S["env_prm"][e] if "env_prm" in S else None) if oracles else AppliedOracle(env.I, env.D)
            _load(o, env, S, e)
            ok, rec = True, []
            for t in range(nstep):
                o.f("wrap_z")[:] = -1          # the kernel cold-starts the inverse-wrap roots at every launch
                o.set(ctrl=ctrl[e, t], qfrc_applied=f[e, t])
                for _ in range(substeps):
                    o.step(1); ok = ok and _in_regime(o, m)
                rec.append(tuple(o.f(k).copy() for k in ("qpos", "qvel", "act", "qacc", "time")))
            if not ok:
                cnt["skipped"] += 1
                continue
            cnt["checked"] += 1
            msg = "%s[%s] env %d, %d x %d" % (name, rows, e, nstep, substeps)
            for t, (qp, qv, ac, qa, tm) in enumerate(rec):
                worst["qpos"] = max(worst["qpos"], float(np.abs(O["qpos"][e, t] - qp).max()))
                worst["qvel"] = max(worst["qvel"], relerr(O["qvel"][e, t], qv))
                worst["qacc"] = max(worst["qacc"], relerr(O["qacc"][e, t], qa))
                np.testing.assert_allclose(O["qpos"][e, t], qp, rtol=0, atol=QPOS_ATOL, err_msg=msg)
                assert relerr(O["qvel"][e, t], qv) < QVEL_REL, (msg, t)
                assert relerr(O["qacc"][e, t], qa) < QACC_REL, (msg, t)
                np.testing.assert_allclose(O["act"][e, t], ac, rtol=0, atol=1e-12, err_msg=msg)
                assert O["time"][e, t] == tm[0], (msg, t)
    _report("oracle %s[%s]" % (name, rows), "checked %d, skipped %d; worst qpos %.1e qvel %.1e qacc %.1e" % (
        cnt["checked"], cnt["skipped"], worst["qpos"], worst["qvel"], worst["qacc"]))
    assert cnt["skipped"] <= MAX_SKIP * (cnt["checked"] + cnt["skipped"]) and cnt["checked"] > 0


# ----------------------------------------------------------------------------- GPU: the round trip with the inverse
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(ROLL_CASES))
def test_inverse_round_trip(case, rows):
    """qfrc_applied = inverse(qacc_target, discrete) - qfrc_actuator, then one substep: (qvel1 - qvel0) / h returns qacc_target to round-off
    on the envs without an active constraint row; every env lies within the Newton stop rule plus round-off, measured in force as
    test_inverse.py's _round_trip does (the discrete inverse of the reached acceleration against qfrc_actuator + qfrc_applied)."""
    import torch
    from test_inverse import _random_qacc
    eid, n = ROLL_CASES[case]
    env, _ = _warm(eid, n, rows)
    m = env.mj_model
    h = m.opt_timestep
    D = env.data("qacc", "qfrc_actuator")
    fact = D["qfrc_actuator"].clone()
    target = _random_qacc(env, D["qacc"].clone())
    I0 = {k: v.clone() for k, v in env.inverse(target, discrete=True, fields=("qfrc_inverse", "qfrc_constraint")).items()}
    applied = (I0["qfrc_inverse"] - fact).contiguous()
    out = env.rollout(torch.zeros(n, 1, m.nu, dtype=torch.float64, device=env.device), qfrc_applied=applied[:, None].contiguous(), substeps=1)
    reached = ((out["qvel"][:, 0] - env.t["qvel"]) / h).contiguous()
    I1 = env.inverse(reached, discrete=True, fields=("qfrc_inverse", "qfrc_constraint"))
    fact, applied, target, reached = (x.cpu().numpy() for x in (fact, applied, target, reached))
    inv0, con0, inv1 = (x.cpu().numpy() for x in (I0["qfrc_inverse"], I0["qfrc_constraint"], I1["qfrc_inverse"]))
    stop = _tol(env) * m.stat_meaninertia * max(1, m.nv)
    big = np.maximum.reduce([np.abs(fact).max(1), np.abs(con0).max(1), np.abs(inv0).max(1), np.full(n, 1e-300)])
    gn = np.linalg.norm(inv1 - (fact + applied), axis=1)
    excess = np.maximum(gn - stop, 0) / big
    free = ~np.any(con0 != 0, axis=1)
    ratio = np.abs(reached - target).max(1) / np.maximum(np.abs(target).max(1), 1e-300)
    _report("round trip %s[%s]" % (case, rows), "stop ratio %.2e, round-off %.1e; %d envs without a constraint row: qacc ratio %.1e" % (
        float((gn / stop).max()), float(excess.max()), int(free.sum()), float(ratio[free].max()) if free.any() else 0.0))
    assert excess.max() <= ROUNDOFF_REL
    assert not free.any() or ratio[free].max() <= ROUNDOFF_REL
    if case == "elbow":
        assert free.sum() >= n // 8


# ----------------------------------------------------------------------------- GPU: no side effects
@pytest.mark.gpu
@pytest.mark.parametrize("eid,n", [("myoHandPoseRandom-v0", 999), ("myoHandObjHoldRandom-v0", 517), ("myoFatiLegWalk-v0", 333)])
def test_no_side_effects(eid, n):
    """Twin batches, one with rollouts (from the bound state and from other states) between its 50 steps: every bound tensor stays
    bit-identical across each rollout and between the twins, and so does a full readout at the end."""
    import torch
    from myosuite_b200 import vec_env
    a_env, b_env = (vec_env.MyoVecEnv(eid, n, seed=SEED) for _ in range(2))
    m = a_env.mj_model
    for env in (a_env, b_env):
        env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for step in range(50):
        act = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(a_env.device)
        before = {k: a_env.t[k].clone() for k in BOUND if k in a_env.t}
        sv = a_env.state_version
        ctrl = torch.rand(n, 2, m.nu, generator=g, dtype=torch.float64).to(a_env.device)
        f = torch.randn(n, 2, m.nv, generator=g, dtype=torch.float64).to(a_env.device)
        a_env.rollout(ctrl, qfrc_applied=f, substeps=3, fields=a_env.ROLLOUT_FIELDS)
        if step % 10 == 5:
            st = {"qvel": torch.randn(n, m.nv, generator=g, dtype=torch.float64).to(a_env.device), "time": torch.zeros(n, dtype=torch.float64, device=a_env.device)}
            a_env.rollout(ctrl, substeps=2, initial_state=st, fields=("qpos",))
        torch.cuda.synchronize()
        assert a_env.state_version == sv
        for k, v in before.items():
            assert _same(v, a_env.t[k]), (step, k)
        a_env.step(act); b_env.step(act.clone())
        torch.cuda.synchronize()
        for k in BOUND:
            if k in a_env.t:
                assert _same(a_env.t[k], b_env.t[k]), (step, k)
    da, db = a_env.data(), b_env.data()
    torch.cuda.synchronize()
    for k in da:
        assert _same(da[k], db[k]), k
    print("\n%s n %d: 50 twin steps and the readout bit-identical with rollouts between them" % (eid, n))


@pytest.mark.gpu
def test_unrequested_outputs_untouched():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv("myoHandObjHoldRandom-v0", 100, seed=SEED)
    env.reset(seed=SEED)
    m = env.mj_model
    ctrl = torch.rand(100, 3, m.nu, dtype=torch.float64, device=env.device)
    full = _bits(env.rollout(ctrl, substeps=2, fields=env.ROLLOUT_FIELDS))
    torch.cuda.synchronize()
    sent = {k: torch.full_like(v, -7) for k, v in full.items()}
    for ask in (("qpos",), ("qvel", "time"), ("act", "qacc", "overflow")):
        for v in sent.values():
            v.fill_(-7)
        n0 = env.batch.launches
        env.batch.rollout(3, 2, stream=env._stream(), ctrl=ctrl, **{k: sent[k] for k in ask})
        torch.cuda.synchronize()
        assert env.batch.launches - n0 in (3, 6)          # one launch per interval (and a regroup before each where the batch regroups)
        for k, v in sent.items():
            assert _same(v, full[k]) if k in ask else bool((v == -7).all()), (ask, k)


# ----------------------------------------------------------------------------- GPU: start state, resumption, slot independence
@pytest.mark.gpu
def test_start_state_resumption_and_slots():
    """An explicit initial_state equal to the bound state changes nothing; rollout(T=8) equals rollout(T=3) then rollout(T=5) from row 2
    with its qacc as the warm start; 4096 hand envs equal the same envs at other slots of a 64-env batch: all bit for bit."""
    import torch
    from myosuite_b200 import assets, vec_env
    m = assets.load("myohand_pose")
    N = 4096
    rng = np.random.default_rng(SEED)
    qpos, qvel, act, _ = _states(m, N, rng, overshoot=0.0, vel=0.5)
    big = vec_env.MyoVecEnv.from_model("myohand_pose", N)
    big.set_state(qpos=qpos, qvel=qvel, act=act)
    big.t["time"].copy_(torch.as_tensor(rng.uniform(0, 1, N), device=big.device))
    dev = big.device
    ctrl = torch.as_tensor(rng.uniform(-0.2, 1.2, (N, 8, m.nu)), device=dev)
    f = torch.as_tensor(rng.normal(0, 5, (N, 8, m.nv)), device=dev)
    F = big.ROLLOUT_FIELDS
    ref = _bits(big.rollout(ctrl, qfrc_applied=f, substeps=4, fields=F))
    st = {k: big.t[k][:, :m.na].contiguous() if k == "act" else big.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart", "time")}
    got = big.rollout(ctrl, qfrc_applied=f, substeps=4, initial_state=st, fields=F)
    for k in F:
        assert _same(got[k], ref[k]), ("explicit start", k)
    a = _bits(big.rollout(ctrl[:, :3].contiguous(), qfrc_applied=f[:, :3].contiguous(), substeps=4, fields=F))
    st2 = {"qpos": a["qpos"][:, 2].contiguous(), "qvel": a["qvel"][:, 2].contiguous(), "act": a["act"][:, 2].contiguous(),
           "qacc_warmstart": a["qacc"][:, 2].contiguous(), "time": a["time"][:, 2].contiguous()}
    b = big.rollout(ctrl[:, 3:].contiguous(), qfrc_applied=f[:, 3:].contiguous(), substeps=4, initial_state=st2, fields=F)
    for k in ("qpos", "qvel", "act", "qacc", "time"):
        assert _same(torch.cat([a[k], b[k]], 1), ref[k]), ("resumed", k)
    assert _same((a["overflow"] != 0) | (b["overflow"] != 0), ref["overflow"] != 0)
    small = vec_env.MyoVecEnv.from_model("myohand_pose", 64)
    idx = rng.choice(N, 64, replace=False)
    ti = torch.as_tensor(idx, device=dev)
    small.set_state(qpos=qpos[idx], qvel=qvel[idx], act=act[idx])
    small.t["time"].copy_(big.t["time"][ti])
    s = small.rollout(ctrl[ti].contiguous(), qfrc_applied=f[ti].contiguous(), substeps=4, fields=F)
    torch.cuda.synchronize()
    for k in F:
        assert _same(s[k], ref[k][ti]), ("slots", k)
    assert torch.isfinite(ref["qvel"]).all()
    print("\nhand %d envs: explicit start, resumption 3 + 5 and the 64-env batch bit-identical (launch info %s)" % (N, big.batch.launch_info()))


# ----------------------------------------------------------------------------- GPU: input checks and the single-env facade
@pytest.mark.gpu
def test_input_checks_without_launch():
    import torch
    from myosuite_b200 import abi, vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 8, seed=SEED)
    m = env.mj_model
    dev = env.device
    good = torch.zeros(8, 4, m.nu, dtype=torch.float64, device=dev)
    n0 = env.batch.launches
    for bad in (torch.zeros(8, 4, m.nu + 1, dtype=torch.float64, device=dev), torch.zeros(7, 4, m.nu, dtype=torch.float64, device=dev),
                torch.zeros(8, 0, m.nu, dtype=torch.float64, device=dev), torch.zeros(8, m.nu, dtype=torch.float64, device=dev),
                good.float(), good.cpu(), good.cpu().numpy(), torch.zeros(8, m.nu, 4, dtype=torch.float64, device=dev).transpose(1, 2)):
        with pytest.raises(ValueError):
            env.rollout(bad)
    for kw in (dict(qfrc_applied=torch.zeros(8, 3, m.nv, dtype=torch.float64, device=dev)), dict(qfrc_applied=torch.zeros(8, 4, m.nv, device=dev)),
               dict(initial_state={"qpos": torch.zeros(8, m.nq + 1, dtype=torch.float64, device=dev)}),
               dict(initial_state={"time": torch.zeros(8, 1, dtype=torch.float64, device=dev)}), dict(substeps=0)):
        with pytest.raises(ValueError):
            env.rollout(good, **kw)
    with pytest.raises(KeyError):
        env.rollout(good, initial_state={"target": torch.zeros(8, m.nq, dtype=torch.float64, device=dev)})
    with pytest.raises(KeyError):
        env.rollout(good, fields=("ctrl",))
    out = torch.zeros(8, 4, m.nq, dtype=torch.float64, device=dev)
    with pytest.raises(abi.MyoError, match="ctrl is required"):
        env.batch.rollout(4, 1, qpos=out)
    for nstep, sub in ((0, 1), (4, 0), (-1, 2)):
        with pytest.raises(abi.MyoError, match=">= 1"):
            env.batch.rollout(nstep, sub, ctrl=good, qpos=out)
    unbound = abi.Batch(env.dev_model, env.device_index, 8, env.cfg)
    with pytest.raises(abi.MyoError, match="bound"):
        unbound.rollout(4, 1, ctrl=good, qpos=out)
    assert env.batch.launches == n0 and unbound.launches == 0
    sv = env.state_version
    env.rollout(good)
    assert env.batch.launches > n0 and env.state_version == sv


@pytest.mark.gpu
def test_myoenv_mj_rollout():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoEnv("myoHandObjHoldRandom-v0", seed=3)
    m = env.mj_model
    env.step(env.action_space.sample())
    v = env.vec
    rng = np.random.default_rng(0)
    ctrl, f = rng.uniform(0, 1, (5, m.nu)), rng.normal(0, 1, (5, m.nv))
    before = env.get_env_state()
    r = env.mj_rollout(ctrl, qfrc_applied=f, substeps=2)
    assert r["qpos"].shape == (5, m.nq) and r["qacc"].shape == (5, m.nv) and r["time"].shape == (5,) and isinstance(r["overflow"], int)
    b = v.rollout(torch.as_tensor(ctrl[None], device=v.device), qfrc_applied=torch.as_tensor(f[None], device=v.device), substeps=2, fields=v.ROLLOUT_FIELDS)
    for k in ("qpos", "qvel", "act", "qacc", "time"):
        assert np.array_equal(r[k], b[k][0].cpu().numpy()), k
    after = env.get_env_state()
    for k, x in before.items():
        assert np.array_equal(x, after[k]), k
    r2 = env.mj_rollout(ctrl[:2], initial_state={"qpos": r["qpos"][1], "qvel": r["qvel"][1], "act": r["act"][1], "qacc_warmstart": r["qacc"][1],
                                                 "time": r["time"][1]}, substeps=2)
    assert abs(r2["time"][0] - r["time"][1] - 2 * m.opt_timestep) < 1e-12


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nrollouts:")
        for k in sorted(REPORT):
            print("  %-36s %s" % (k, REPORT[k]))
