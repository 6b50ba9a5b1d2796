"""CPU reference of mjd_inverseFD (myo_batch_inverse_fd), float64, with no device code: f = qfrc_inverse from InvOracle.inverse
(tests/inverse_oracle.c), qfrc_actuator from the oracle's own forward pass at the same state, and the qpos perturbation through
FdOracle.integrate_pos (mj_integratePos).  Forward differences, row i of a block = (f(x + eps e_i) - f(x)) * (1 / eps), in MuJoCo's layout
(DfDq[i, j] = d f_j / d q_i).  Every pass starts from a reset oracle: cold inverse-wrap roots, as every device pass."""
import numpy as np

BLOCKS = ("DfDq", "DfDv", "DfDa")


def passes(o, fo, qpos, qvel, act, qacc, eps, flags=0):
    """The nominal pass and the 3 nv perturbed ones: [(block or None, i, qfrc_inverse, qfrc_actuator, signature)], where signature is the
    contact count, the constraint row count and the set of rows with a non-zero force (the contact list and the active row set)."""
    nv = len(qvel)
    act = np.asarray(act, dtype=np.float64)

    def one(q, v, a):
        o.reset(); o.set(qpos=q, qvel=v, act=act, ctrl=np.zeros(len(o.f("ctrl"))))
        f = o.inverse(a, flags)
        sig = (o.ncon, o.nefc, tuple(np.nonzero(o.f("efc_force")[:o.nefc])[0].tolist()))
        o.reset(); o.set(qpos=q, qvel=v, act=act, ctrl=np.zeros(len(o.f("ctrl"))))
        o.forward()
        return f, o.f("qfrc_actuator").copy(), sig

    out = [(None, -1) + one(qpos, qvel, qacc)]
    for i in range(nv):
        e = np.zeros(nv); e[i] = 1.0
        out.append(("DfDq", i) + one(fo.integrate_pos(qpos, e, eps), qvel, qacc))
    for i in range(nv):
        v = np.array(qvel, dtype=np.float64); v[i] += eps
        out.append(("DfDv", i) + one(qpos, v, qacc))
    for i in range(nv):
        a = np.array(qacc, dtype=np.float64); a[i] += eps
        out.append(("DfDa", i) + one(qpos, qvel, a))
    return out


def jacobians(P, eps, actuation):
    """{DfDq, DfDv, DfDa: [nv, nv]}, the nominal f and {block: [nv] bool, the column changes the contact list or the active rows} from
    passes(); f = qfrc_inverse - qfrc_actuator when `actuation`."""
    r = 1.0 / eps
    _, _, f0i, f0a, sig0 = P[0]
    f0 = f0i - f0a if actuation else f0i
    nv = len(f0)
    J = {b: np.zeros((nv, nv)) for b in BLOCKS}
    changed = {b: np.zeros(nv, bool) for b in BLOCKS}
    for blk, i, fi, fa, sig in P[1:]:
        J[blk][i] = ((fi - fa if actuation else fi) - f0) * r
        changed[blk][i] = sig != sig0
    return J, f0, changed


def inverse_fd(o, fo, qpos, qvel, act, qacc, eps, flags=0, actuation=False):
    """(Jacobians, nominal f, changed columns) at one state: the reference of one env of myo_batch_inverse_fd"""
    return jacobians(passes(o, fo, qpos, qvel, act, qacc, eps, flags), eps, actuation)
