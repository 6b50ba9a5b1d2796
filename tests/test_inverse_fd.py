"""Finite-difference Jacobians of the inverse dynamics (myo_batch_inverse_fd, MyoVecEnv.inverse_fd, MyoEnv.mjd_inverseFD) against the CPU
reference (tests/inverse_fd_ref.py), closed forms and the call's own nominal.

CPU: the myo_inverse_fd_buffers / myo_inverse_fd_params field order against abi.py; on every shipped model and the SWEEP / MUSCLE zoo
models the reference's DfDa is the oracle's dense mass matrix (constraints off) and M + h diag(damping) (discrete), its DfDv at qvel = 0 is
diag(damping), and its DfDa does not depend on actuation.

GPU, every base task on both row storages: against the CPU reference at eps 1e-6 and 1e-4; each qpos (hinge / slide), qvel and qacc row
equals the difference of a second call's nominal from a host-built perturbed state, bit for bit; the actuation blocks against the
reference's difference of qfrc_actuator; batch-size and single-env independence; no side effects; the overflow flag; input checks before
any launch."""
import ctypes
import os

import numpy as np
import pytest

import inverse_fd_ref as R
from fd_oracle import FdOracle
from inverse_oracle import INV_DISCRETE, INV_NOCONSTRAINT, InvOracle
from parity_helpers import _states
from test_inverse import FREE_REL, SHIPPED, qM_dense
from test_mj_data import BOUND, CASES, ROWS, SEED, WARM, _header_struct, _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-6
ROUND = 64 * np.finfo(float).eps      # closed forms: |J - ref| <= ROUND * scale / eps, scale = the largest |f| of the passes (f is formed
                                      # by sums of O(nv) terms, each rounded once; the difference of two such sums keeps their error)
CHANGED_SHARE = 0.01                  # columns whose perturbation changes the contact list or the active rows: counted, under 1 %
REPORT = {}


def _report(key, text):
    REPORT[key] = text
    print("\n%s %s" % (key, text))


# ----------------------------------------------------------------------------- CPU
def test_inverse_fd_structs_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_inverse_fd_buffers")
    assert len(fields) == decls and abi.INVERSE_FD_FIELDS == fields
    assert [n for n, _ in abi.MyoInverseFdBuffers._fields_] == fields and ctypes.sizeof(abi.MyoInverseFdBuffers) == 8 * len(fields)
    assert set(abi.INVERSE_FD_SHAPES) == set(fields) - {"qacc", "qpos0", "qvel0", "act0", "overflow"}
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert "typedef struct { double eps; int32_t actuation; } myo_inverse_fd_params;" in src
    assert [n for n, _ in abi.MyoInverseFdParams._fields_] == ["eps", "actuation"] and ctypes.sizeof(abi.MyoInverseFdParams) == 16
    assert src.index("} myo_cmc_params;") < src.index("} myo_inverse_fd_buffers;") < src.index("int myo_batch_inverse_fd(")
    assert "myo_batch_inverse_fd" in abi.EXPORTS


def _cpu_models(models, tmp_path):
    import test_actuation_zoo as AZ
    ms = {k: models[k] for k in SHIPPED}
    ms.update({k: v["m"] for k, v in AZ.build_zoo(tmp_path, names=["MUSCLE"] + ["SWEEP_%d" % nv for nv in AZ.SWEEP_NV]).items()})
    return ms


def _scale(P):
    return max(max(np.abs(fi).max(), np.abs(fa).max()) for _, _, fi, fa, _ in P)


def test_reference_closed_forms(models, tmp_path):
    """Constraints off: DfDa = M (the oracle's dense mass matrix of its forward pass) and, with discrete, M + h diag(damping), within
    ROUND scale / eps; at qvel = 0 with actuation off, DfDv = diag(damping) within that bound plus 2 eps max_i |bias(e_i) - bias(0)| (the
    bias is quadratic in qvel, so its forward difference at 0 is eps times that coefficient); DfDa with and without actuation agree within
    the round-off bound (qfrc_actuator does not depend on qacc)."""
    from myosuite_b200 import blob
    rng = np.random.default_rng(SEED)
    worst = {}
    for name, m in _cpu_models(models, tmp_path).items():
        I, D = blob.pack(m)
        o, fo = InvOracle(I, D), FdOracle(I, D)
        qpos, qvel, act, _ = _states(m, 2, rng, overshoot=0.0, vel=0.3)
        h, damp = m.opt_timestep, m.dof_damping
        for e in range(len(qpos)):
            qacc = rng.normal(0, 10, m.nv)
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e]); o.forward()
            M = qM_dense(m, o.f("qM"))
            for flags, ref in ((INV_NOCONSTRAINT, M), (INV_NOCONSTRAINT | INV_DISCRETE, M + h * np.diag(damp))):
                P = R.passes(o, fo, qpos[e], qvel[e], act[e], qacc, EPS, flags)
                bound = ROUND * _scale(P) / EPS
                J0, _, _ = R.jacobians(P, EPS, False)
                J1, _, _ = R.jacobians(P, EPS, True)
                key = "DfDa" + (" discrete" if flags & INV_DISCRETE else "")
                err = np.abs(J0["DfDa"] - ref).max() / bound
                worst[key] = max(worst.get(key, 0.0), err)
                assert err <= 1, (name, e, key, err)
                err = np.abs(J1["DfDa"] - J0["DfDa"]).max() / bound
                worst["DfDa actuation"] = max(worst.get("DfDa actuation", 0.0), err)
                assert err <= 1, (name, e, "actuation", err)
            # DfDv at rest
            v0 = np.zeros(m.nv)
            P = R.passes(o, fo, qpos[e], v0, act[e], qacc, EPS, INV_NOCONSTRAINT)
            J0, _, _ = R.jacobians(P, EPS, False)
            o.reset(); o.set(qpos=qpos[e], qvel=v0, act=act[e]); o.forward(); b0 = o.f("qfrc_bias").copy()
            quad = 0.0
            for i in range(m.nv):
                v = v0.copy(); v[i] = 1.0
                o.reset(); o.set(qpos=qpos[e], qvel=v, act=act[e]); o.forward()
                quad = max(quad, np.abs(o.f("qfrc_bias") - b0).max())
            bound = ROUND * _scale(P) / EPS + 2 * EPS * quad
            err = np.abs(J0["DfDv"] - np.diag(damp)).max() / bound
            worst["DfDv rest"] = max(worst.get("DfDv rest", 0.0), err)
            assert err <= 1, (name, e, "DfDv", err)
    print("\nreference closed forms, worst share of the bound: %s" % {k: "%.2f" % v for k, v in worst.items()})


# ----------------------------------------------------------------------------- GPU helpers
COMBOS = [(0, "rand", 1e-6), (0, "readout", 1e-4), (INV_NOCONSTRAINT, "rand", 1e-4), (INV_NOCONSTRAINT, "readout", 1e-6),
          (INV_DISCRETE, "rand", 1e-6), (INV_DISCRETE, "readout", 1e-4)]      # (flags, qacc, eps); each runs with actuation 0 and 1
ALL = ("DfDq", "DfDv", "DfDa", "qfrc_inverse")


def _warm(eid, n, rows="p48", **kw):
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv(eid, n, seed=SEED, row_storage=rows, **kw)
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(WARM):
        env.step((torch.rand(n, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
    return env


def _qaccs(env):
    """the readout's qacc at the bound state and a random one of the same magnitude per env"""
    import torch
    Q = env.data("qacc")["qacc"].clone()
    g = torch.Generator(device="cpu").manual_seed(SEED)
    mag = Q.abs().amax(1, keepdim=True).clamp_min(1.0)
    return {"readout": Q, "rand": (torch.randn(Q.shape, generator=g, dtype=torch.float64).to(env.device) * mag).contiguous()}


def _call(env, q, flags, actuation, eps, fields=ALL, **kw):
    return env.inverse_fd(q, eps=eps, actuation=actuation, constraints=not flags & INV_NOCONSTRAINT, discrete=bool(flags & INV_DISCRETE),
                          fields=fields, **kw)


def _host(D):
    return {k: v.cpu().numpy() for k, v in D.items()}


# ----------------------------------------------------------------------------- GPU: the CPU reference
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_against_reference(case, rows):
    """Every combination of COMBOS with actuation 0 and 1 against the CPU reference at the same eps, at the benchmarked batch size, on 4
    envs spread over the batch.  Per entry |J - J_ref| <= 2 FREE_REL scale / eps, scale as tests/test_inverse.py has it (the largest of
    |qfrc_inverse|, |M qacc|, |qfrc_bias| and, here, |qfrc_actuator| over the passes), except: columns whose perturbation changes the
    contact list or the active row set on the CPU are counted, not compared (asserted under 1 % and printed); and with constraints on the
    p48 rows, which store the contact Jacobian rows with 36 mantissa bits, so that each pass's rounding of them reaches f divided by eps
    (up to 150x the bound on hold at eps 1e-4 on an H100) -- those are reported.  The actuation blocks: DfDq(0) - DfDq(1) and DfDv(0) - DfDv(1) against the reference's difference of
    qfrc_actuator, within the readout's qfrc_actuator bound (FRC_REL of the largest |qfrc_actuator|) over eps."""
    from test_inverse import _inv_oracles
    from test_mj_data import FRC_REL
    eid, n = CASES[case]
    env = _warm(eid, n, rows)
    m = env.mj_model
    qs = _qaccs(env)
    S = env.get_env_state()
    envs = [0, n // 3, (2 * n) // 3, n - 1]
    oracles = _inv_oracles(env)
    fo = FdOracle(env.I, env.D)
    worst, counted, cols, reported, bad = {}, 0, 0, {}, []
    for flags, qk, eps in COMBOS:
        dev = {a: _host(_call(env, qs[qk], flags, a, eps)) for a in (0, 1)}
        QH = qs[qk].cpu().numpy()
        for e in envs:
            o = oracles.get(S["env_prm"][e] if "env_prm" in S else None)
            P = R.passes(o, fo, S["qpos"][e], S["qvel"][e], S["act"][e, :m.na], QH[e], eps, flags)
            o.reset(); o.set(qpos=S["qpos"][e], qvel=S["qvel"][e], act=S["act"][e, :m.na]); o.forward()
            scale = max(_scale(P), np.abs(qM_dense(m, o.f("qM")) @ QH[e]).max(), np.abs(o.f("qfrc_bias")).max(), 1e-300)
            bound = 2 * FREE_REL * scale / eps
            amax = max(max(np.abs(fa).max() for _, _, _, fa, _ in P), 1e-300)
            for a in (0, 1):
                J, f0, changed = R.jacobians(P, eps, a)
                if flags & INV_NOCONSTRAINT:      # the nominal: test_inverse.py's bound, plus the readout's qfrc_actuator bound with actuation
                    err = float(np.abs(dev[a]["qfrc_inverse"][e] - f0).max() / (FREE_REL * scale + a * FRC_REL * amax))
                    worst["nominal act %d" % a] = max(worst.get("nominal act %d" % a, 0.0), err)
                    if err > 1:
                        bad.append((e, flags, a, "nominal", err))
                for b in R.BLOCKS:
                    keep = ~changed[b]
                    if a == 0:
                        counted += int(changed[b].sum()); cols += len(keep)
                    err = float(np.abs(dev[a][b][e][keep] - J[b][keep]).max() / bound) if keep.any() else 0.0
                    key = "%s flags %d act %d eps %.0e" % (b, flags, a, eps)
                    if rows == "p48" and not flags & INV_NOCONSTRAINT:
                        reported[key] = max(reported.get(key, 0.0), err)
                        continue
                    worst[key] = max(worst.get(key, 0.0), err)
                    if err > 1:
                        bad.append((e, key, err))
            # the actuation blocks: the reference's difference of qfrc_actuator
            r = 1.0 / eps
            fa0 = P[0][3]
            for b in ("DfDq", "DfDv"):
                ref = np.stack([(fa - fa0) * r for blk, _, _, fa, _ in P[1:] if blk == b])
                err = float(np.abs((dev[0][b][e] - dev[1][b][e]) - ref).max() / (FRC_REL * amax / eps))
                worst["actuation " + b] = max(worst.get("actuation " + b, 0.0), err)
                if err > 1:
                    bad.append((e, "actuation " + b, flags, eps, err))
    _report("reference %s %s" % (case, rows), "changed columns %d/%d; worst share of the bound %s%s" % (
        counted, cols, {k: "%.2g" % v for k, v in sorted(worst.items())},
        ("; f32 rows with constraints (reported): %s" % {k: "%.2g" % v for k, v in sorted(reported.items())}) if reported else ""))
    assert not bad, bad[:10]
    assert counted <= CHANGED_SHARE * cols, (counted, cols)


# ----------------------------------------------------------------------------- GPU: the call's own nominal, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_rows_equal_nominal_differences(case, rows):
    """On every hinge and slide qpos column and every qvel and qacc column, row i equals (qfrc_inverse of a second call started at the
    host-built perturbed state - the nominal) * (1 / eps), bit for bit, for flags 0, NOCONSTRAINT and DISCRETE with actuation 0 and 1
    (readout qacc with flags 0, random qacc otherwise).  Free-joint quaternions start at (1, 0, 0, 0), where mj_integratePos renormalises
    them exactly, so that the host-built qpos is the device's."""
    import torch
    eid, _ = CASES[case]
    n = 64
    env = _warm(eid, n, rows)
    m = env.mj_model
    for j in np.nonzero(m.jnt_type == 0)[0]:
        a = m.jnt_qposadr[j] + 3
        env.t["qpos"][:, a:a + 4] = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64, device=env.device)
    qs = _qaccs(env)
    S = {k: env.t[k].clone() for k in ("qpos", "qvel", "act")}
    r = 1.0 / EPS
    hinge = [(int(m.jnt_dofadr[j]), int(m.jnt_qposadr[j])) for j in range(m.njnt) if m.jnt_type[j] in (2, 3)]
    ncol = 0
    for flags in (0, INV_NOCONSTRAINT, INV_DISCRETE):
        q = qs["readout" if flags == 0 else "rand"]
        for a in (0, 1):
            out = _call(env, q, flags, a, EPS)
            f0 = out["qfrc_inverse"]

            def nominal(**st):
                return _call(env, q, flags, a, EPS, fields=("DfDa", "qfrc_inverse"), initial_state=dict(S, **st))["qfrc_inverse"]
            for d, qa in hinge:
                x = S["qpos"].clone(); x[:, qa] += EPS
                assert torch.equal(out["DfDq"][:, d], (nominal(qpos=x) - f0) * r), (case, rows, flags, a, "q", d)
            for i in range(m.nv):
                x = S["qvel"].clone(); x[:, i] += EPS
                assert torch.equal(out["DfDv"][:, i], (nominal(qvel=x) - f0) * r), (case, rows, flags, a, "v", i)
                x = q.clone(); x[:, i] += EPS
                f = _call(env, x, flags, a, EPS, fields=("DfDa", "qfrc_inverse"), initial_state=S)["qfrc_inverse"]
                assert torch.equal(out["DfDa"][:, i], (f - f0) * r), (case, rows, flags, a, "a", i)
            ncol += len(hinge) + 2 * m.nv
    _report("self-consistency %s %s" % (case, rows), "%d columns x %d envs bit-identical" % (ncol, n))


# ----------------------------------------------------------------------------- GPU: independence, side effects, overflow, checks
@pytest.mark.gpu
@pytest.mark.parametrize("maxcon", [None, 8])
def test_batch_and_single_env_independence(maxcon):
    """A 4096-env hand batch equals 64-env batches of every 64th env bit for bit, at two contact capacities; MyoEnv.mjd_inverseFD equals
    env 0 of a batch."""
    import torch
    from myosuite_b200 import vec_env
    kw = {} if maxcon is None else {"maxcon": maxcon}
    big = _warm("myoHandPoseRandom-v0", 4096, **kw)
    q = _qaccs(big)["rand"]
    S = {k: big.t[k].clone() for k in ("qpos", "qvel", "act")}
    fields = ALL + ("overflow",)
    for a in (0, 1):
        ob = _call(big, q, 0, a, EPS, fields=fields)
        for k0 in (0, 17):
            sel = torch.arange(k0, 4096, 64, device=big.device)
            small = vec_env.MyoVecEnv("myoHandPoseRandom-v0", 64, seed=SEED, **kw)
            os_ = _call(small, q[sel].contiguous(), 0, a, EPS, fields=fields, initial_state={k: v[sel].contiguous() for k, v in S.items()})
            for k in fields:
                assert _same(ob[k][sel], os_[k]), (maxcon, a, k)
    env1 = vec_env.MyoEnv("myoHandPoseRandom-v0", seed=SEED, **kw)
    st = {k: S[k][0].cpu().numpy() for k in S}
    got = env1.mjd_inverseFD(q[0].cpu().numpy(), flg_actuation=True, initial_state=st)
    ob = _call(big, q, 0, 1, EPS)
    for g_, k in zip(got, ("DfDq", "DfDv", "DfDa")):
        assert np.array_equal(g_, ob[k][0].cpu().numpy()), k


@pytest.mark.gpu
def test_no_side_effects():
    """Bound tensors unchanged and 50 twin env steps bit-identical after calls; outputs not requested are untouched; a twin batch created
    and used between two calls leaves the results unchanged; two launches per call."""
    import torch
    from myosuite_b200 import abi, vec_env
    a, b = (_warm("myoHandObjHoldRandom-v0", 256) for _ in range(2))
    m = a.mj_model
    q = _qaccs(a)["rand"]
    before = {k: a.t[k].clone() for k in BOUND if k in a.t}
    l0 = a.batch.launches
    first = _call(a, q, 0, 1, EPS, fields=ALL + ("overflow",))
    assert a.batch.launches - l0 == 2
    for k, v in before.items():
        assert _same(v, a.t[k]), k
    twin = _warm("myoHandObjHoldRandom-v0", 256)      # the coexistence pattern: another batch set up and used between two calls
    _call(twin, _qaccs(twin)["readout"], INV_DISCRETE, 0, 1e-4)
    twin.step(torch.zeros(256, m.nu, device=twin.device))
    again = _call(a, q, 0, 1, EPS, fields=ALL + ("overflow",))
    for k in first:
        assert _same(first[k], again[k]), k
    g = torch.Generator(device="cpu").manual_seed(5)
    for _ in range(50):
        act = (torch.rand(256, m.nu, generator=g) * 2 - 1).to(a.device)
        a.step(act); b.step(act)
    for k in before:
        assert _same(a.t[k], b.t[k]), k
    nv = m.nv
    for only in ("DfDq", "DfDv", "DfDa"):
        T = {k: torch.full((256, nv, nv), 7.0, dtype=torch.float64, device=a.device) for k in ("DfDq", "DfDv", "DfDa")}
        a.batch.inverse_fd(abi.MyoInverseFdParams(eps=EPS, actuation=0), stream=a._stream(), qacc=q, **{only: T[only]})
        torch.cuda.synchronize()
        assert not bool((T[only] == 7).all())
        assert all(bool((T[k] == 7).all()) for k in T if k != only), only


@pytest.mark.gpu
def test_overflow_flag(tmp_path):
    """The COMBO contact zoo model at maxcon 1 sets overflow; the same states at full capacity leave it clear."""
    import test_contact_zoo as CZ
    from myosuite_b200 import vec_env
    zoo = CZ.build_zoo(tmp_path)
    m = zoo["COMBO"][0]
    cfgs = CZ._configs(zoo, "COMBO")
    qpos = np.stack([q for _, q in cfgs])
    qvel, act, _ = CZ._state(m, qpos, 5, [lb != "generic" for lb, _ in cfgs])
    n = len(qpos)
    res = {}
    for maxcon in (1, 64):
        env = vec_env.MyoVecEnv(None, n, model=m, maxcon=maxcon)
        env.set_state(qpos=qpos, qvel=qvel, act=act)
        q = env.torch.zeros((n, m.nv), dtype=env.torch.float64, device=env.device)
        res[maxcon] = env.inverse_fd(q, fields=("DfDq", "overflow"))["overflow"].cpu().numpy()
    assert res[1].any() and not res[64].any(), res


@pytest.mark.gpu
def test_input_checks_without_launch():
    """Every listed failure raises before any launch: myo_batch_launch_count is unchanged.  (The n_env x columns > int32 check needs a
    batch of over 2^31 / (3 nv) envs and is not exercised here.)"""
    import torch
    from myosuite_b200 import abi
    env = _warm("myoElbowPose1D6MRandom-v0", 8)
    m, n = env.mj_model, 8
    q = torch.zeros(n, m.nv, dtype=torch.float64, device=env.device)
    J = torch.zeros(n, m.nv, m.nv, dtype=torch.float64, device=env.device)
    L, P = env.batch.L, abi.MyoInverseFdParams
    base = env.batch.launches
    bad = [(P(eps=EPS, actuation=0), 0, dict(DfDq=J)),                 # no qacc
           (P(eps=EPS, actuation=0), 0, dict(qacc=q)),                 # no Jacobian
           (P(eps=EPS, actuation=0), 4, dict(qacc=q, DfDq=J)),         # unknown flag bit
           (P(eps=0.0, actuation=0), 0, dict(qacc=q, DfDq=J)),
           (P(eps=-1e-6, actuation=0), 0, dict(qacc=q, DfDq=J)),
           (P(eps=float("nan"), actuation=0), 0, dict(qacc=q, DfDq=J)),
           (P(eps=float("inf"), actuation=0), 0, dict(qacc=q, DfDq=J)),
           (P(eps=EPS, actuation=2), 0, dict(qacc=q, DfDq=J)),
           (P(eps=EPS, actuation=-1), 0, dict(qacc=q, DfDq=J))]
    for p, flags, t in bad:
        with pytest.raises(abi.MyoError):
            env.batch.inverse_fd(p, flags=flags, **t)
    d = abi.MyoInverseFdBuffers(); d.qacc = q.data_ptr(); d.DfDq = J.data_ptr()
    assert L.myo_batch_inverse_fd(None, ctypes.byref(d), ctypes.byref(P(eps=EPS, actuation=0)), 0, None) != 0
    assert L.myo_batch_inverse_fd(env.batch.handle, None, ctypes.byref(P(eps=EPS, actuation=0)), 0, None) != 0
    assert L.myo_batch_inverse_fd(env.batch.handle, ctypes.byref(d), None, 0, None) != 0
    unbound = abi.Batch(env.dev_model, env.device_index, n, env.cfg)
    with pytest.raises(abi.MyoError):
        unbound.inverse_fd(P(eps=EPS, actuation=0), qacc=q, DfDq=J)
    assert unbound.launches == 0
    for kw in (dict(eps=0), dict(eps=float("nan")), dict(actuation=2), dict(fields=("overflow",)), dict(fields=("C",)),
               dict(initial_state={"qacc_warmstart": q}), dict(initial_state={"time": q[:, 0].contiguous()})):
        with pytest.raises((ValueError, KeyError)):
            env.inverse_fd(q, **kw)
    for bad_q in (q.float(), q.cpu(), q[:4], torch.zeros(2 * n, m.nv, dtype=torch.float64, device=env.device)[::2]):
        with pytest.raises(ValueError):
            env.inverse_fd(bad_q)
    assert env.batch.launches == base
    env.inverse_fd(q)
    assert env.batch.launches == base + 2


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\n---- inverse-dynamics FD (tests/test_inverse_fd.py)")
        for k in sorted(REPORT):
            print("%-40s %s" % (k, REPORT[k]))
