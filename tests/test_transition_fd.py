"""Finite-difference transition Jacobians (myo_batch_transition_fd, MyoVecEnv.transition_fd, MyoEnv.mjd_transitionFD) against rollouts,
the CPU reference and closed forms.

CPU: the myo_fd_buffers / myo_fd_params field order against abi.py; integratePos / differentiatePos of tests/fd_oracle.c round-trip on
every shipped model and the sweep models; oracle_transition_fd on constraint-free states against independent closed forms (the act
block of B from MuJoCo's activation dynamics, the qvel rows of the act columns from M, the damping, the moment arms and the numpy muscle
gain); the ctrl clamp rule at and near both ends of ctrlrange.

GPU, on both row storages where physics is compared: every column sampled from every block equals the stated difference of rollouts
from host-built perturbed starts, bit for bit; A and B against oracle_transition_fd; the structural zeros and identities; batch-size and
single-env independence; no side effects; the overflow flag; input checks before any launch."""
import ctypes
import os

import numpy as np
import pytest

from fd_oracle import FdOracle
from parity_helpers import _states
from test_actuation_zoo import muscle_dynamics, muscle_gain
from test_inverse import SHIPPED, _sweeps, qM_dense
from test_mj_data import BOUND, CASES, ROWS, SEED, WARM, _header_struct, _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-6
ORACLE_REL = 1e-6          # free-of-constraint envs: |A - A_oracle| per block, relative to the env's largest entry of that block (at least
                           # 1e-6 of the matrix's largest entry, for blocks that are zero up to the CPU reference's round-off)
# the base tasks at their benchmarked shapes; the walk without fatigue (the FD intervals run no fatigue)
FD_CASES = {("walk" if k == "walk_fatigue" else k): (("myoLegWalk-v0", n) if k == "walk_fatigue" else (eid, n)) for k, (eid, n) in CASES.items()}
REPORT = {}


def _report(key, text):
    REPORT[key] = text
    print("\n%s %s" % (key, text))


# ----------------------------------------------------------------------------- CPU
def test_fd_structs_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_fd_buffers")
    assert len(fields) == decls and abi.FD_FIELDS == fields
    assert [n for n, _ in abi.MyoFdBuffers._fields_] == fields and ctypes.sizeof(abi.MyoFdBuffers) == 8 * len(fields)
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert "typedef struct { double eps; int32_t centered, substeps; } myo_fd_params;" in src
    assert [n for n, _ in abi.MyoFdParams._fields_] == ["eps", "centered", "substeps"] and ctypes.sizeof(abi.MyoFdParams) == 16
    assert src.index("} myo_ik_params;") < src.index("} myo_fd_buffers;") < src.index("int myo_batch_transition_fd(")
    assert "myo_batch_transition_fd" in abi.EXPORTS


def _models(models, tmp_path):
    ms = {k: models[k] for k in SHIPPED}
    ms.update(_sweeps(tmp_path))
    return ms


def test_oracle_integrate_differentiate(models, tmp_path):
    """differentiatePos(q, integratePos(q, v, dt), dt) = v to 1e-12 relative plus the cancellation of q + v dt - q (4 ulp(max|q|) / dt),
    free joints included (random unit quaternions)."""
    from myosuite_b200 import blob
    rng = np.random.default_rng(SEED)
    for name, m in _models(models, tmp_path).items():
        o = FdOracle(*blob.pack(m))
        qpos, _, _, _ = _states(m, 8, rng)
        for e in range(len(qpos)):
            q = qpos[e].copy()
            for j in np.nonzero(m.jnt_type == 0)[0]:
                a = m.jnt_qposadr[j] + 3
                u = rng.normal(size=4); q[a:a + 4] = u / np.linalg.norm(u)
            v = rng.normal(0, 1, m.nv)
            for dt in (1.0, 1e-3, 1e-6):
                q2 = o.integrate_pos(q, v, dt)
                got = o.differentiate_pos(q, q2, dt)
                tol = 1e-12 * max(1.0, np.abs(v).max()) + 4 * np.spacing(max(1.0, np.abs(q).max())) / dt
                assert np.abs(got - v).max() <= tol, (name, e, dt, np.abs(got - v).max(), tol)


def _free_states(o, m, rng, n, vel=0.05):
    """States of m with no contact, limit or equality row active: interior joints, small velocities, checked on the oracle after one step
    of each perturbation's size (eps moves nothing across a margin at these distances)."""
    out = []
    for _ in range(200 * n):
        qpos, qvel, act, ctrl = _states(m, 1, rng, overshoot=-0.2, vel=vel)
        o.reset(); o.set(qpos=qpos[0], qvel=qvel[0], act=act[0], ctrl=ctrl[0]); o.forward()
        if o.nefc == 0:
            o.step(1)
            if o.nefc == 0:
                out.append((qpos[0], qvel[0], act[0], ctrl[0]))
        if len(out) == n:
            break
    return out


def test_oracle_closed_forms(models):
    """At substeps = 1 on constraint-free states of the elbow and the hand: B's act block is diagonal with h d act_dot / d ctrl (numpy
    activation dynamics: h / tau for tausmooth 0), B's qpos / qvel rows are exactly 0; the qvel rows of the act columns are
    h (M + h diag(damping))^-1 (moment_i gain_i); forward and centred agree to O(eps)."""
    from myosuite_b200 import blob
    rng = np.random.default_rng(SEED)
    worst = {}
    for name in ("myoelbow_1dof6muscles", "myohand_pose"):
        m = models[name]
        o = FdOracle(*blob.pack(m))
        h, nv, na = m.opt_timestep, m.nv, m.na
        states = _free_states(o, m, rng, 6)
        assert len(states) >= 3, name
        for qpos, qvel, act, ctrl in states:
            o.reset(); o.set(qpos=qpos, qvel=qvel, act=act)
            Af, Bf = o.transition_fd(ctrl, eps=EPS)
            Ac, Bc = o.transition_fd(ctrl, eps=EPS, centered=True)
            assert np.array_equal(o.f("qpos"), qpos) and np.array_equal(o.f("qvel"), qvel)      # the state is restored
            assert not np.any(Bf[:2 * nv]) and not np.any(Bc[:2 * nv])
            Bact = Bc[2 * nv:]
            assert not np.any(Bact - np.diag(np.diag(Bact)))
            d = 1e-7
            ref = np.array([h * (muscle_dynamics(ctrl[i] + d, act[i], m.actuator_dynprm[i]) - muscle_dynamics(ctrl[i] - d, act[i], m.actuator_dynprm[i])) / (2 * d)
                            for i in range(m.nu)])
            worst[name + " B act"] = max(worst.get(name + " B act", 0), np.abs(np.diag(Bact) - ref).max() / np.abs(ref).max())
            # act columns: forward pass at the start for the moment arms and the gain
            o.set(ctrl=ctrl); o.forward()
            M = qM_dense(m, o.f("qM"))
            L, V, J = o.f("actuator_length"), o.f("actuator_velocity"), o.f("ten_J").reshape(m.ntendon, nv)
            G = np.stack([m.actuator_gear[i, 0] * J[m.actuator_trnid[i, 0]] * muscle_gain(L[i], V[i], m.actuator_lengthrange[i], m.actuator_gainprm[i])[0]
                          for i in range(m.nu)], axis=1)
            ref = h * np.linalg.solve(M + h * np.diag(m.dof_damping), G)
            got = Ac[nv:2 * nv, 2 * nv:]
            worst[name + " A qvel/act"] = max(worst.get(name + " A qvel/act", 0), np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))
            worst[name + " fwd-ctr"] = max(worst.get(name + " fwd-ctr", 0), np.abs(Af - Ac).max() / np.abs(Ac).max(), np.abs(Bf - Bc).max() / np.abs(Bc).max())
            o.reset()
    print(worst)
    for k, v in worst.items():
        assert v < (1e-4 if "fwd-ctr" in k else 1e-5), (k, v)


def test_oracle_ctrl_clamp_rule(models):
    """ctrl at the low end, at the high end, interior and within eps of each end of ctrlrange: a column that can only go one way equals
    that one-sided expression, also when centred; an interior column is the two-sided one (forward only when not centred)."""
    from myosuite_b200 import blob
    m = models["myoelbow_1dof6muscles"]
    assert np.all(m.actuator_ctrllimited) and m.nq == m.nv
    o = FdOracle(*blob.pack(m))
    rng = np.random.default_rng(SEED)
    qpos, qvel, act, _ = _states(m, 1, rng, overshoot=-0.2, vel=0.05)
    lo, hi = m.actuator_ctrlrange[:, 0], m.actuator_ctrlrange[:, 1]
    ctrl = np.array([lo[0], hi[1], 0.5 * (lo[2] + hi[2]), lo[3] + 0.3 * EPS, hi[4] - 0.3 * EPS, 0.25])

    def interval(c):        # x' of one interval from the start with ctrl c (the reference's cold wrap roots, warm-start rule)
        o.reset(); o.set(qpos=qpos[0], qvel=qvel[0], act=act[0], ctrl=c)
        o.f("wrap_z")[:] = -1; o.f("wrap_warm")[:] = 1
        o.step(1)
        return np.concatenate([o.f("qpos").copy(), o.f("qvel").copy(), o.f("act").copy()])
    x0 = interval(ctrl)
    sides = set()
    for centered in (False, True):
        o.reset(); o.set(qpos=qpos[0], qvel=qvel[0], act=act[0])
        _, B = o.transition_fd(ctrl, eps=EPS, centered=centered, A=False)
        for i in range(m.nu):
            cp, cm = ctrl.copy(), ctrl.copy(); cp[i] += EPS; cm[i] -= EPS
            fwd = lo[i] <= ctrl[i] and ctrl[i] + EPS <= hi[i]
            back = (centered or not fwd) and lo[i] <= ctrl[i] - EPS and ctrl[i] <= hi[i]
            sides.add((fwd, back))
            if fwd and back:
                ref = (interval(cp) - interval(cm)) * (1 / (2 * EPS))
            elif fwd:
                ref = (interval(cp) - x0) * (1 / EPS)
            else:
                ref = (x0 - interval(cm)) * (1 / EPS)
            assert np.array_equal(B[:, i], ref), (centered, i, ctrl[i])
    assert sides == {(True, False), (False, True), (True, True)}


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


def _ctrl_mix(env, g):
    """ctrl rows mixing values at 0, at 1, within eps of the ends and interior across envs and actuators (uniform pass counts per round)"""
    import torch
    n, nu = env.num_envs, env.mj_model.nu
    c = torch.rand(n, nu, generator=g, dtype=torch.float64)
    k = torch.randint(0, 5, (n, nu), generator=g)
    c = torch.where(k == 0, torch.zeros_like(c), torch.where(k == 1, torch.ones_like(c), c))
    c = torch.where(k == 2, torch.full_like(c, 0.3 * EPS), c)
    return c.to(env.device).contiguous()


def _start(env):
    return {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart")}


def _x(env, R):
    return R["qpos"][:, 0], R["qvel"][:, 0], R["act"][:, 0]


def _hinge_cols(m):
    return [int(m.jnt_dofadr[j]) for j in range(m.njnt) if m.jnt_type[j] in (2, 3)]


def _sample(cols, k, rng):
    cols = list(cols)
    return cols if len(cols) <= k else sorted(rng.choice(cols, k, replace=False).tolist())


# ----------------------------------------------------------------------------- GPU: rollouts, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(FD_CASES))
def test_columns_equal_rollout_differences(case, rows):
    """Columns sampled from every block (every column on the elbow; free-joint rotation columns excluded) against the stated difference
    of rollout(substeps=...) from host-built perturbed starts and from the start, in torch f64, bit for bit: forward and centred,
    substeps 1 and frame_skip, ctrl rows mixing 0, 1, near-end and interior values.  Rows of free-joint rotations (differentiatePos of a
    quaternion, through atan2) are compared to 1e-8 of the column's largest entry plus 64 ulp(1) / eps, the others exactly.  Free-joint quaternions start at (1, 0, 0, 0)."""
    import torch
    eid, n = FD_CASES[case]
    env, g = _warm(eid, n, rows, normalize_act=False, auto_reset=False)
    m = env.mj_model
    nv, na, nu, nq, nx = m.nv, m.na, m.nu, m.nq, 2 * m.nv + m.na
    rng = np.random.default_rng(SEED)
    ctrl = _ctrl_mix(env, g)
    S = _start(env)
    for j in np.nonzero(m.jnt_type == 0)[0]:
        # free-joint quaternions at (1, 0, 0, 0): integratePos renormalises every quaternion of a perturbed qpos column, which is exact
        # there, so the host-built starts match the device's bit for bit (the legs then face another way about z; the hold object is at
        # its qpos0 orientation)
        a = m.jnt_qposadr[j] + 3
        S["qpos"][:, a:a + 4] = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64, device=env.device)
    lim, lo, hi = (torch.as_tensor(x, device=env.device) for x in (m.actuator_ctrllimited.astype(bool), m.actuator_ctrlrange[:, 0], m.actuator_ctrlrange[:, 1]))
    rot = np.zeros(nv, bool)
    for j in np.nonzero(m.jnt_type == 0)[0]:
        rot[m.jnt_dofadr[j] + 3:m.jnt_dofadr[j] + 6] = True
    exact_rows = torch.as_tensor(np.concatenate([~rot, np.ones(nv + na, bool)]), device=env.device)
    k = 100 if case == "elbow" else 4
    qcols = _sample(_hinge_cols(m) + [int(d) for d in np.nonzero(~rot)[0] if d not in _hinge_cols(m)], k, rng)
    acols = [nv + c for c in _sample(range(nv), k, rng)] + [2 * nv + c for c in _sample(range(na), k, rng)]
    ucols = _sample(range(nu), k, rng)
    for substeps in (1, env.n_frames):
        def roll(**st):
            R = env.rollout(ctrl[:, None].contiguous(), substeps=substeps, initial_state=dict(S, **st), fields=("qpos", "qvel", "act"))
            return R
        def roll_u(c):
            return env.rollout(c[:, None].contiguous(), substeps=substeps, initial_state=S, fields=("qpos", "qvel", "act"))
        R0 = roll()
        for centered in (False, True):
            out = env.transition_fd(ctrl, eps=EPS, centered=centered, substeps=substeps, initial_state=S)
            A, B = out["A"], out["B"]

            def diff(Rp, Rm, r):       # (x+ (-) x-) * r on the exact rows (hinge / slide and free translations subtract)
                qp, vp, ap = _x(env, Rp); qm, vm, am = _x(env, Rm)
                dq = torch.zeros(n, nv, dtype=torch.float64, device=env.device)
                for j in range(m.njnt):
                    qa, da = m.jnt_qposadr[j], m.jnt_dofadr[j]
                    w = 3 if m.jnt_type[j] == 0 else 1
                    dq[:, da:da + w] = qp[:, qa:qa + w] - qm[:, qa:qa + w]
                    if m.jnt_type[j] == 0:      # mju_subQuat (compared to round-off only)
                        a, b_ = qm[:, qa + 3:qa + 7], qp[:, qa + 3:qa + 7]
                        w0 = a[:, 0] * b_[:, 0] + (a[:, 1:] * b_[:, 1:]).sum(1)
                        ax = a[:, :1] * b_[:, 1:] - b_[:, :1] * a[:, 1:] - torch.cross(a[:, 1:], b_[:, 1:], dim=1)
                        sn = ax.norm(dim=1)
                        ang = 2 * torch.atan2(sn, w0)
                        ang = torch.where(ang > np.pi, ang - 2 * np.pi, ang)
                        dq[:, da + 3:da + 6] = ax / sn.clamp_min(1e-300)[:, None] * ang[:, None]
                return torch.cat([dq, vp - vm, ap - am], 1) * r

            def check(got, ref, label):
                e = exact_rows
                assert torch.equal(got[:, e], ref[:, e]), (case, rows, substeps, centered, label, (got[:, e] - ref[:, e]).abs().max().item())
                if not e.all():
                    scale = got.abs().max(1, keepdim=True).values.clamp_min(1e-300)
                    assert ((got[:, ~e] - ref[:, ~e]).abs() - 1e-8 * scale).max() <= 64 * np.finfo(float).eps / EPS, label

            r1, r2 = 1.0 / EPS, 1.0 / (2.0 * EPS)
            for c in qcols + acols:
                def pert(h):
                    if c < nv:
                        j = int(np.nonzero(m.jnt_dofadr == c)[0][0]) if c in m.jnt_dofadr else None
                        q = S["qpos"].clone()
                        if j is not None and m.jnt_type[j] in (2, 3):
                            q[:, m.jnt_qposadr[j]] += h
                        else:     # free-joint translation: the dof's position coordinate
                            jf = int(np.nonzero((m.jnt_dofadr <= c) & (m.jnt_type == 0))[0][-1])
                            q[:, m.jnt_qposadr[jf] + c - m.jnt_dofadr[jf]] += h
                        return roll(qpos=q)
                    if c < 2 * nv:
                        v = S["qvel"].clone(); v[:, c - nv] += h; return roll(qvel=v)
                    a = S["act"].clone(); a[:, c - 2 * nv] += h; return roll(act=a)
                Rp = pert(EPS)
                ref = diff(Rp, pert(-EPS), r2) if centered else diff(Rp, R0, r1)
                check(A[:, :, c], ref, "A col %d" % c)
            for i in ucols:
                x = ctrl[:, i]
                inr = lambda a_, b_: (~lim[i]) | ((a_ >= lo[i]) & (a_ <= hi[i]) & (b_ >= lo[i]) & (b_ <= hi[i]))
                fwd = inr(x, x + EPS)
                back = (torch.full_like(fwd, centered) | ~fwd) & inr(x - EPS, x)
                cp, cm = ctrl.clone(), ctrl.clone(); cp[:, i] += EPS; cm[:, i] -= EPS
                Rp, Rm = roll_u(cp), roll_u(cm)
                both, only_f, only_b = (fwd & back)[:, None], (fwd & ~back)[:, None], (~fwd & back)[:, None]
                ref = torch.where(both, diff(Rp, Rm, r2), torch.where(only_f, diff(Rp, R0, r1), torch.where(only_b, diff(R0, Rm, r1), torch.zeros(1, dtype=torch.float64, device=env.device))))
                check(B[:, :, i], ref, "B col %d" % i)
            assert bool(((ctrl == 0) | (ctrl == 1)).any())
    _report("bit-identity %s %s" % (case, rows), "A cols %s, B cols %s" % (qcols + acols, ucols))


# ----------------------------------------------------------------------------- GPU: the CPU reference
ORACLE_CASES = {"elbow": ("myoElbowPose1D6MRandom-v0", 64), "hand_pose": ("myoHandPoseRandom-v0", 64), "reach": ("myoHandReachRandom-v0", 64),
                "hold": ("myoHandObjHoldRandom-v0", 32), "stand": ("myoLegStandRandom-v0", 16)}


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_against_oracle(case, rows):
    """A and B (forward, substeps 1) against oracle_transition_fd.  Envs with no constraint row in the nominal or any perturbed step
    (checked on the oracle's start and end of the nominal) are held to ORACLE_REL of the env's largest entry per block; hold and stand
    states are lifted into free flight so that their free-joint columns are exercised.  On contact-rich envs the worst deviation and the
    share of columns within 1e-3 are reported."""
    import torch
    from myosuite_b200 import vec_env
    eid, n = ORACLE_CASES[case]
    env = vec_env.MyoVecEnv(eid, n, seed=SEED, row_storage=rows, auto_reset=False, normalize_act=False)
    env.reset(seed=SEED)
    m = env.mj_model
    rng = np.random.default_rng(SEED)
    qpos = env.t["qpos"].cpu().numpy().copy()
    qvel = rng.normal(0, 0.05, (n, m.nv)); act = rng.uniform(0, 1, (n, m.na)); ctrl = rng.uniform(0.05, 0.95, (n, m.nu))
    for j in np.nonzero(m.jnt_type == 0)[0]:        # free flight: lift the free body well clear of everything
        qpos[:, m.jnt_qposadr[j] + 2] += 5.0
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    out = env.transition_fd(torch.as_tensor(ctrl, device=env.device), eps=EPS)
    A, B = out["A"].cpu().numpy(), out["B"].cpu().numpy()
    qws = env.t["qacc_warmstart"].cpu().numpy()
    o = FdOracle(env.I, env.D)
    nv, nx = m.nv, 2 * m.nv + m.na
    blocks = {"q": slice(0, nv), "v": slice(nv, 2 * nv), "a": slice(2 * nv, nx)}
    worst_free, worst_c, within, cols, nfree, where = 0.0, 0.0, 0, 0, 0, None
    for e in range(n):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        free = o.nefc == 0
        o.step(1); free = free and o.nefc == 0
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], qacc_warmstart=qws[e])
        Ao, Bo = o.transition_fd(ctrl[e], eps=EPS)
        if free:
            nfree += 1
            for mk, M_, Mo in (("A", A[e], Ao), ("B", B[e], Bo)):
                for bk, sl in blocks.items():
                    ref = max(np.abs(Mo[sl]).max(), 1e-6 * np.abs(Mo).max())      # (blocks that are exactly 0 in exact arithmetic)
                    d = np.abs(M_[sl] - Mo[sl]) / ref
                    if d.max() > worst_free:
                        worst_free, where = d.max(), (e, mk, bk, np.unravel_index(d.argmax(), d.shape), ref)
        else:
            for M_, Mo in ((A[e], Ao), (B[e], Bo)):
                d = np.abs(M_ - Mo).max(0) / np.maximum(np.abs(Mo).max(0), 1e-12)
                worst_c = max(worst_c, d.max()); within += int((d <= 1e-3).sum()); cols += d.size
    _report("oracle %s %s" % (case, rows), "constraint-free envs %d/%d worst %.2e (at %s); contact envs worst %.2e, columns within 1e-3: %s"
            % (nfree, n, worst_free, where, worst_c, "%.3f" % (within / cols) if cols else "-"))
    assert nfree > 0 or case == "stand"          # (the legs' equality rows are always active)
    assert worst_free <= ORACLE_REL, worst_free


# ----------------------------------------------------------------------------- GPU: structure
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(FD_CASES))
def test_structure(case):
    """substeps = 1 on reached states: act rows are zero in the qpos and qvel columns; the act/act and act/ctrl blocks are diagonal; B's
    qpos / qvel rows are zero; hinge / slide qpos rows equal [I 0 0] + h (qvel rows) to 8 ulp(max|qpos|) / eps."""
    import torch
    eid, n = FD_CASES[case]
    env, g = _warm(eid, min(n, 512), "p48", normalize_act=False, auto_reset=False)
    m = env.mj_model
    nv, na, nx = m.nv, m.na, 2 * m.nv + m.na
    ctrl = _ctrl_mix(env, g)
    out = env.transition_fd(ctrl, eps=EPS, centered=True)
    A, B = out["A"], out["B"]
    off = ~torch.eye(na, dtype=torch.bool, device=env.device)
    assert not A[:, 2 * nv:, :2 * nv].any()
    assert not A[:, 2 * nv:, 2 * nv:][:, off].any() and not B[:, 2 * nv:][:, off].any()
    assert not B[:, :2 * nv].any()
    h = m.opt_timestep
    hinge = [int(m.jnt_dofadr[j]) for j in range(m.njnt) if m.jnt_type[j] in (2, 3)]
    I = torch.zeros(nv, nx, dtype=torch.float64, device=env.device); I[:, :nv] = torch.eye(nv)
    ref = I[hinge] + h * A[:, nv:2 * nv][:, hinge]
    qmax = env.t["qpos"].abs().max().item()
    bound = 8 * np.spacing(max(qmax, 1.0)) / EPS
    d = (A[:, hinge] - ref).abs().max().item()
    _report("structure %s" % case, "qpos-row identity worst %.2e (bound %.2e)" % (d, bound))
    assert d <= bound, (d, bound)


# ----------------------------------------------------------------------------- GPU: independence, side effects, overflow, checks
@pytest.mark.gpu
def test_batch_and_single_env_independence():
    """A 4096-env hand batch equals a 64-env batch of the same states bit for bit; MyoEnv.mjd_transitionFD equals env 0 of a batch."""
    import torch
    from myosuite_b200 import vec_env
    big, g = _warm("myoHandPoseRandom-v0", 4096, "p48", normalize_act=False, auto_reset=False)
    ctrl = _ctrl_mix(big, g)
    S = _start(big)
    for centered in (False, True):
        ob = big.transition_fd(ctrl, centered=centered, substeps=2, fields=("A", "B", "overflow"))
        small = vec_env.MyoVecEnv("myoHandPoseRandom-v0", 64, seed=SEED, normalize_act=False, auto_reset=False)
        sel = torch.arange(0, 4096, 64, device=big.device)
        os_ = small.transition_fd(ctrl[sel].contiguous(), centered=centered, substeps=2, initial_state={k: v[sel].contiguous() for k, v in S.items()},
                                  fields=("A", "B", "overflow"))
        for k in ("A", "B", "overflow"):
            assert _same(ob[k][sel], os_[k]), k
    env1 = vec_env.MyoEnv("myoHandPoseRandom-v0", seed=SEED, normalize_act=False)
    st = {k: S[k][0].cpu().numpy() for k in S}
    A1, B1 = env1.mjd_transitionFD(ctrl[0].cpu().numpy(), initial_state=st)
    ob = big.transition_fd(ctrl, fields=("A", "B"))
    assert np.array_equal(A1, ob["A"][0].cpu().numpy()) and np.array_equal(B1, ob["B"][0].cpu().numpy())


@pytest.mark.gpu
def test_no_side_effects():
    """Bound tensors unchanged; 50 twin env steps match bit for bit; with only A requested B's buffer is untouched, and the other way."""
    import torch
    from myosuite_b200 import abi
    envs = [_warm("myoHandObjHoldRandom-v0", 256, "p48")[0] for _ in range(2)]
    a, b = envs
    before = {k: a.t[k].clone() for k in BOUND if k in a.t}
    ctrl = torch.full((256, a.mj_model.nu), 0.5, dtype=torch.float64, device=a.device)
    a.transition_fd(ctrl, centered=True, substeps=3)
    for k, v in before.items():
        assert _same(v, a.t[k]), k
    g = torch.Generator(device="cpu").manual_seed(5)
    for _ in range(50):
        act = (torch.rand(256, a.mj_model.nu, generator=g) * 2 - 1).to(a.device)
        a.step(act); b.step(act)
    for k in before:
        assert _same(a.t[k], b.t[k]), k
    m = a.mj_model
    nx = 2 * m.nv + m.na
    for only in ("A", "B"):
        A = torch.full((256, nx, nx), 7.0, dtype=torch.float64, device=a.device)
        B = torch.full((256, nx, m.nu), 7.0, dtype=torch.float64, device=a.device)
        a.batch.transition_fd(abi.MyoFdParams(eps=EPS, centered=0, substeps=1), stream=a._stream(), ctrl=ctrl, **({"A": A} if only == "A" else {"B": B}))
        torch.cuda.synchronize()
        assert bool((B == 7).all()) if only == "A" else bool((A == 7).all())
        assert not bool(((A if only == "A" else B) == 7).all())


@pytest.mark.gpu
def test_overflow_flag(tmp_path):
    """A contact zoo model at a capacity that drops contacts sets overflow; the same states at full capacity leave it clear."""
    import torch
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
        env2 = vec_env.MyoVecEnv(None, n, model=m, maxcon=maxcon)
        env2.set_state(qpos=qpos, qvel=qvel, act=act)
        ctrl = torch.full((n, m.nu), 0.5, dtype=torch.float64, device=env.device)
        res[maxcon] = env.transition_fd(ctrl, fields=("A", "overflow"))["overflow"].cpu().numpy()
        R = env2.rollout(ctrl[:, None].contiguous(), fields=("overflow",))["overflow"].cpu().numpy()
        if maxcon == 64:
            assert not R.any()
    assert res[1].any() and not res[64].any(), res


@pytest.mark.gpu
def test_input_checks_without_launch():
    """Every listed failure raises before any launch: myo_batch_launch_count is unchanged."""
    import torch
    from myosuite_b200 import abi
    env, _ = _warm("myoElbowPose1D6MRandom-v0", 8, "p48")
    m, n = env.mj_model, 8
    nx = 2 * m.nv + m.na
    ctrl = torch.full((n, m.nu), 0.5, dtype=torch.float64, device=env.device)
    A = torch.zeros(n, nx, nx, dtype=torch.float64, device=env.device)
    L, P = env.batch.L, abi.MyoFdParams
    base = env.batch.launches
    bad = [dict(params=P(eps=EPS, centered=0, substeps=1), tensors=dict(A=A)),                          # no ctrl
           dict(params=P(eps=EPS, centered=0, substeps=1), tensors=dict(ctrl=ctrl)),                     # neither A nor B
           dict(params=P(eps=0.0, centered=0, substeps=1), tensors=dict(ctrl=ctrl, A=A)),
           dict(params=P(eps=-1e-6, centered=0, substeps=1), tensors=dict(ctrl=ctrl, A=A)),
           dict(params=P(eps=float("nan"), centered=0, substeps=1), tensors=dict(ctrl=ctrl, A=A)),
           dict(params=P(eps=float("inf"), centered=0, substeps=1), tensors=dict(ctrl=ctrl, A=A)),
           dict(params=P(eps=EPS, centered=0, substeps=0), tensors=dict(ctrl=ctrl, A=A)),
           dict(params=P(eps=EPS, centered=2, substeps=1), tensors=dict(ctrl=ctrl, A=A))]
    for b in bad:
        with pytest.raises(abi.MyoError):
            env.batch.transition_fd(b["params"], **b["tensors"])
    d = abi.MyoFdBuffers(); d.ctrl = ctrl.data_ptr(); d.A = A.data_ptr()
    assert L.myo_batch_transition_fd(None, ctypes.byref(d), ctypes.byref(P(eps=EPS, centered=0, substeps=1)), None) != 0
    assert L.myo_batch_transition_fd(env.batch.handle, None, ctypes.byref(P(eps=EPS, centered=0, substeps=1)), None) != 0
    assert L.myo_batch_transition_fd(env.batch.handle, ctypes.byref(d), None, None) != 0
    unbound = abi.Batch(env.dev_model, env.device_index, n, env.cfg)
    with pytest.raises(abi.MyoError):
        unbound.transition_fd(P(eps=EPS, centered=0, substeps=1), ctrl=ctrl, A=A)
    assert unbound.launches == 0
    for kw in (dict(eps=0), dict(eps=float("nan")), dict(substeps=0), dict(centered=2), dict(fields=("overflow",)), dict(fields=("C",))):
        with pytest.raises((ValueError, KeyError)):
            env.transition_fd(ctrl, **kw)
    for bad_ctrl in (ctrl.float(), ctrl.cpu(), ctrl[:, :1], ctrl.t()):
        with pytest.raises(ValueError):
            env.transition_fd(bad_ctrl)
    assert env.batch.launches == base
    env.transition_fd(ctrl)
    assert env.batch.launches > base


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\n---- transition FD (tests/test_transition_fd.py)")
        for k in sorted(REPORT):
            print("%-40s %s" % (k, REPORT[k]))
