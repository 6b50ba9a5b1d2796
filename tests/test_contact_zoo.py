"""Every contact collider class and contact-parameter branch of the step kernel against the CPU oracle, on synthetic models.

The shipped models reach only part of the contact code: no sphere pair, friction 1 / 1, gap 0, solimp power 2 and one solref
everywhere, and the parallel-axis and two-contact branches only by chance.  The zoo here is one small model per collider class
(CT_CAP_CAP .. CT_ELL_ELL, one or two free bodies, nv <= 12) plus one combined model with five free bodies whose analytic and
ellipsoid pairs interleave in model pair order.  Each is written as MJCF, compiled by `mjcf.compile_mjcf` and run as a physics-only
batch.  Every geom has contype = conaffinity = 0: only the explicit <pair>s collide.  One muscle on a tendon between two sites of the
same body gives every model an actuator (the batch needs an action row) without exerting any net force.

Pair parameters: friction (0.7, 1.3) and (1.3, 0.7) (the tangent rows and the pyramid regulariser see both), condim 1 and 3, gap > 0
with margin > gap (contacts detected but inactive), solimp power 1, 2 and 2.5 with a width of 1 cm, so that active contacts fall on
both sides of solimp[3], and four different solrefs.  The configurations put every pair at five signed distances (beyond the margin,
inside (margin - gap, margin], just inside margin - gap, touching, 3 mm deep) at seeded random orientations, plus the degenerate
poses of each collider: exactly and nearly parallel capsules, a sphere beyond a capsule's end cap, a capsule lying on and standing
upright on the plane, a capsule axis through an ellipsoid's centre and along its principal axis, a three-equal-radii ellipsoid
against a spheroid, and tilted ellipsoids on the plane."""
import os

import numpy as np
import pytest

from parity_helpers import _in_regime, relerr

ROWS = ["p48", "f64"]
# one forward pass: test_gpu_parity.py holds the hand to 1e-7.  Here one generic SPH_CAP config measures 1.0e-7 on an H100, bit for bit the
# same in both row storages and at solver tolerances 1e-10 and 1e-12: round-off of the light (0.07 kg) stiff bodies, not storage or
# convergence.  Every other class stays below 7.3e-8; the four arithmetic mutations this module is meant to catch move qacc by >= 1e-3.
FWD_QACC = 2e-7
DIST_RTOL, DIST_ATOL = 1e-7, 1e-11    # contact distances (test_gpu_parity.py)
ROLL_QPOS, ROLL_QVEL = 1e-7, 1e-5     # 10 chained substeps
MID = dict(qpos=2e-7, qvel=1e-5, qacc=1e-6)     # product kernels: the mid-episode bounds of test_product_parity.py
NGEN = 5                              # random orientations per class
WIDTH = 0.01                          # solimp width of every pair
REPORT = {}

GT = {"plane": 0, "sphere": 2, "capsule": 3, "ellipsoid": 4}
CT_NAMES = ["NONE", "CAP_CAP", "SPH_SPH", "SPH_CAP", "PLANE_SPH", "PLANE_CAP", "PLANE_ELL", "CAP_ELL", "ELL_ELL"]
CAP, CAP2, SPH, SPH2 = (0.02, 0.04), (0.015, 0.05), (0.025,), (0.02,)
ELL, SPHEROID, ROUND = (0.03, 0.022, 0.016), (0.03, 0.03, 0.018), (0.022, 0.022, 0.022)


def _pp(condim, fr, margin, gap, power, mid, solref):
    return dict(condim=condim, friction="%g %g" % fr, margin=margin, gap=gap, solimp="0.85 0.97 %g %g %g" % (WIDTH, mid, power),
                solref="%g %g" % solref)


# class -> geom 1, geom 2 (None body: the world plane), pair parameters
ZOO = {
    "CAP_CAP": (("capsule", CAP), ("capsule", CAP2), _pp(3, (0.7, 1.3), 0.010, 0.004, 2.5, 0.5, (0.03, 0.8))),
    "SPH_SPH": (("sphere", SPH), ("sphere", SPH2), _pp(3, (1.3, 0.7), 0.006, 0.002, 1, 0.3, (0.02, 1))),
    "SPH_CAP": (("sphere", SPH), ("capsule", CAP), _pp(1, (0.7, 1.3), 0.008, 0.003, 2, 0.6, (0.015, 1.1))),
    "PLANE_SPH": (("plane", None), ("sphere", SPH), _pp(3, (0.7, 1.3), 0.006, 0.002, 1, 0.4, (0.02, 1))),
    "PLANE_CAP": (("plane", None), ("capsule", CAP), _pp(3, (0.7, 1.3), 0.010, 0.004, 2, 0.5, (0.04, 1.2))),
    "PLANE_ELL": (("plane", None), ("ellipsoid", ELL), _pp(1, (0.7, 1.3), 0.006, 0.002, 2.5, 0.5, (0.02, 1))),
    "CAP_ELL": (("capsule", CAP), ("ellipsoid", ELL), _pp(3, (0.7, 1.3), 0.008, 0.003, 2.5, 0.4, (0.02, 1))),
    "ELL_ELL": (("ellipsoid", ROUND), ("ellipsoid", SPHEROID), _pp(3, (1.3, 0.7), 0.006, 0.0, 1, 0.5, (0.03, 0.9))),
}
# the combined model: bodies in this order (geom ids follow them), pairs sorted by geom ids = model pair order.  Analytic (A) and
# ellipsoid (E) pairs interleave: floor-capA A, floor-ellB A, capA-ellB E, capA-capC A, ellB-ellE E, capC-ellE E, sphD-capC A
COMBO_GEOMS = [("floor", "plane", None), ("capA", "capsule", CAP), ("ellB", "ellipsoid", ELL), ("capC", "capsule", CAP),
               ("sphD", "sphere", SPH2), ("ellE", "ellipsoid", SPHEROID)]
COMBO_PAIRS = [("floor", "capA", _pp(3, (0.7, 1.3), 0.004, 0.0, 2, 0.5, (0.02, 1))),
               ("floor", "ellB", _pp(1, (0.7, 1.3), 0.006, 0.002, 1, 0.5, (0.02, 1))),
               ("capA", "ellB", _pp(3, (1.3, 0.7), 0.006, 0.0, 2.5, 0.5, (0.03, 0.9))),
               ("capA", "capC", _pp(3, (0.7, 1.3), 0.006, 0.002, 2, 0.5, (0.02, 1))),
               ("ellB", "ellE", _pp(3, (0.7, 1.3), 0.006, 0.0, 2, 0.5, (0.02, 1))),
               ("capC", "ellE", _pp(1, (0.7, 1.3), 0.006, 0.0, 2.5, 0.5, (0.02, 1))),
               ("sphD", "capC", _pp(3, (1.3, 0.7), 0.006, 0.0, 1, 0.5, (0.02, 1)))]


def _size(t, s):
    if t == "plane":
        return "0 0 1"
    return " ".join("%.17g" % v for v in s)


def zoo_xml(geoms, pairs):
    """MJCF of free bodies, one geom each (body None: a world geom), the explicit pairs and one force-free muscle on body 1."""
    world = "".join('<geom name="%s" type="%s" size="%s" contype="0" conaffinity="0"/>' % (n, t, _size(t, s)) for n, t, s in geoms if s is None)
    bodies, k = [], 0
    for n, t, s in geoms:
        if s is None:
            continue
        sites = '<site name="ms0" pos="0 0 0.005"/><site name="ms1" pos="0 0 -0.005"/>' if k == 0 else ""
        bodies.append('<body name="b%d" pos="%g 0 1"><freejoint/><geom name="%s" type="%s" size="%s" contype="0" conaffinity="0"/>%s</body>'
                      % (k, 0.3 * k, n, t, _size(t, s), sites))
        k += 1
    pr = "".join('<pair geom1="%s" geom2="%s" %s/>' % (a, b, " ".join('%s="%s"' % kv for kv in sorted(p.items()))) for a, b, p in pairs)
    return ('<mujoco model="zoo"><option timestep="0.002"/><worldbody>%s%s</worldbody>'
            '<tendon><spatial name="mt"><site site="ms0"/><site site="ms1"/></spatial></tendon>'
            '<actuator><muscle name="m0" tendon="mt" lengthrange="0.005 0.02" force="5" ctrlrange="0 1"/></actuator>'
            '<contact>%s</contact></mujoco>' % (world, "".join(bodies), pr))


def class_spec(ct):
    g1, g2, p = ZOO[ct]
    return [("g1", g1[0], g1[1]), ("g2", g2[0], g2[1])], [("g1", "g2", p)]


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
def quat_axis(axis, ang):
    a = np.asarray(axis, float); a = a / np.linalg.norm(a)
    return np.array([np.cos(ang / 2), *(np.sin(ang / 2) * a)])


def rand_quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def place(probe, qpos, slot, target, along=None, pair=None):
    """Move free body `slot` until the probe's signed distance of `pair` (of the closest contact when None) is `target`: along the
    contact normal, or along the unit vector `along`.  The probe model is the same geometry with a 10 m margin on every pair, so
    the oracle reports each pair at any distance."""
    for _ in range(20):
        probe.reset(); probe.set(qpos=qpos); probe.forward()
        d, cp = probe.f("con_dist"), probe.i("con_pair")
        ks = np.arange(len(d)) if pair is None else np.nonzero(cp == pair)[0]
        k = int(ks[np.argmin(d[ks])]); n = probe.f("con_frame")[9 * k:9 * k + 3]
        if abs(d[k] - target) < 1e-13:
            break
        u = n if along is None else np.asarray(along, float)
        qpos[7 * slot:7 * slot + 3] += (target - d[k]) / np.dot(n, u) * u      # the distance moves at rate n.u (envelope theorem)
    probe.reset(); probe.set(qpos=qpos); probe.forward()
    d, cp = probe.f("con_dist"), probe.i("con_pair")
    assert abs((d if pair is None else d[cp == pair]).min() - target) < 1e-10, (target, d)
    return qpos


def bands(p):
    """Signed distances each pose is placed at: beyond the margin, detected but inactive, just active, touching, shallow."""
    inc = p["margin"] - p["gap"]
    inactive = 0.5 * (inc + p["margin"]) if p["gap"] > 0 else inc - 0.0005
    return [p["margin"] + 0.01, inactive, inc - 0.002, 0.0, -0.003]


def class_configs(ct, probe, rng):
    """[(label, qpos)] for one class model: NGEN random orientations at every distance band, then the degenerate poses."""
    g1, g2, p = ZOO[ct]
    two = g1[0] != "plane"
    nb = 2 if two else 1
    slot = nb - 1                        # the body of geom 2 is the one that is moved
    out = []

    def pose(qs, dirs=None):
        q = np.zeros(7 * nb)
        for b in range(nb):
            q[7 * b + 3:7 * b + 7] = qs[b]
        if two:
            q[0:3] = [0.0, 0.0, 0.5]
            q[7:10] = q[0:3] + 0.2 * dirs
        else:
            q[0:3] = [0.0, 0.0, 0.2]
        return q

    for _ in range(NGEN):
        qs = [rand_quat(rng) for _ in range(nb)]
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        base = pose(qs, d)
        for b in bands(p):
            out.append(("generic", place(probe, base.copy(), slot, b)))
    I = np.array([1.0, 0, 0, 0])
    deg = []
    if ct == "CAP_CAP":
        # exactly parallel axes, side by side and axially shifted: the det < MYO_MINVAL branch, two contacts
        deg += [("parallel", [I, I], [1.0, 0, 0]), ("parallel-shifted", [I, I], [1.0, 0, 0.25])]
        # nearly parallel (det = sin^2 1e-7 = 1e-14, just above MYO_MINVAL), crossing point far beyond the ends: one contact at an end
        deg += [("near-parallel", [I, quat_axis([1, 0, 0], 1e-7)], [1.0, 0, 0.0])]
    elif ct == "SPH_CAP":
        deg += [("beyond-cap", [I, I], [0.3, 0.2, -1.0]), ("beyond-cap-axial", [I, I], [0.0, 0.0, -1.0])]
    elif ct == "PLANE_CAP":
        deg += [("upright", [I], None), ("lying", [quat_axis([1, 0, 0], np.pi / 2)], None),
                ("lying-diag", [quat_axis([1, 1, 0], np.pi / 2)], None)]
    elif ct == "PLANE_ELL":
        deg += [("tilted", [quat_axis([1, 2, 0.5], 0.7)], None), ("tilted-2", [quat_axis([0.3, -1, 0.2], 2.1)], None), ("aligned", [I], None)]
    elif ct == "CAP_ELL":
        deg += [("axis-through-centre", [I, I], [0.0, 0.0, -1.0]), ("axis-through-centre-tilted", [I, quat_axis([1, 1, 1], 0.9)], [0.0, 0.0, -1.0]),
                ("parallel-principal", [quat_axis([0, 1, 0], np.pi / 2), I], [0.01, 0.0, -1.0])]
    elif ct == "ELL_ELL":
        deg += [("round-vs-spheroid-axis", [I, I], [0.0, 0.0, 1.0]), ("round-vs-spheroid-equator", [I, I], [1.0, 0.0, 0.0]),
                ("round-vs-spheroid-tilted", [I, quat_axis([1, 0, 1], 0.6)], [0.4, 0.5, 0.7])]
    elif ct == "SPH_SPH":
        deg += [("aligned", [I, I], [0.0, 0.0, 1.0])]
    elif ct == "PLANE_SPH":
        deg += [("aligned", [I], None)]
    for label, qs, d in deg:
        d = None if d is None else np.asarray(d, float) / np.linalg.norm(d)
        base = pose(qs, d)
        if label == "near-parallel":      # lines cross at t = 0.2 on capsule 1, far beyond its end (the clipped, well-conditioned case)
            base[8] += 0.2 * np.sin(1e-7)
        axial = label.startswith("axis-through") or label in ("upright", "beyond-cap-axial")
        for b in (p["margin"] - p["gap"] - 0.002, -0.002):
            out.append((label, place(probe, base.copy(), slot, b, along=[0, 0, 1.0] if axial else None)))
    return out


def combo_config(probe, m):
    """The combined model's scene: capA lying on the floor and capC parallel beside it (two contacts each), sphD beyond capC's end
    cap, ellB against capA's side and held 5 mm above the floor (floor-ellB detected but inactive), ellE resting on ellB."""
    q = np.zeros(m.nq)
    lie = quat_axis([0, 1, 0], np.pi / 2)                       # capsule axis along x
    poses = [([0, 0, 0.016], lie), ([0, -0.045, 0.03], quat_axis([1, 2, 3], 0.4)), ([0, 0.04, 0.016], lie),
             ([0.079, 0.04, 0.016], [1.0, 0, 0, 0]), ([0.01, -0.035, 0.09], quat_axis([2, -1, 1], 1.1))]
    for b, (pos, qq) in enumerate(poses):
        q[7 * b:7 * b + 3] = pos; q[7 * b + 3:7 * b + 7] = qq
    place(probe, q, 1, 0.005, along=[0, 0, 1.0], pair=1)        # floor-ellB
    place(probe, q, 1, -0.001, along=[0, 1.0, 0], pair=2)       # capA-ellB (a move along y keeps the floor distance)
    place(probe, q, 4, -0.001, along=[0, 0, 1.0], pair=4)       # ellB-ellE
    return q


def combo_configs(probe, m, rng):
    """The scene and 15 copies with every body shifted by up to 0.5 mm."""
    q0 = combo_config(probe, m)
    out = [("scene", q0)]
    for _ in range(15):
        q = q0.copy()
        for b in range(m.nv // 6):
            q[7 * b:7 * b + 3] += rng.uniform(-5e-4, 5e-4, 3)
        out.append(("scene-shifted", q))
    return out


def regime_ok(o, m):
    """_in_regime for the iterative colliders only (a plane's size is not a depth scale)."""
    return _in_regime(o, m) or all(m.geom_type[int(a)] == GT["plane"] for a in o.i("con_geom1")[o.f("con_dist") < 0])


# ----------------------------------------------------------------------------- CPU: the zoo reaches every class and branch
def build_zoo(tmp, names=None):
    """{name: (model, program, info, probe oracle)}: the eight class models and the combined one ("COMBO")."""
    from myosuite_b200 import program
    zoo = {}
    specs = {ct: class_spec(ct) for ct in ZOO}
    specs["COMBO"] = (COMBO_GEOMS, COMBO_PAIRS)
    for name, (geoms, pairs) in specs.items():
        if names is not None and name not in names:
            continue
        m = compile_xml(zoo_xml(geoms, pairs), tmp, name)
        prog, info = program.build_program(m)
        probe_pairs = [(a, b, dict(p, margin=10.0, gap=0.0, condim=1)) for a, b, p in pairs]
        probe = oracle_of(compile_xml(zoo_xml(geoms, probe_pairs), tmp, name + "_probe"))
        zoo[name] = (m, prog, info, probe)
    return zoo


def test_zoo_coverage(tmp_path):
    """The zoo reaches every collider class but CT_NONE, both condims, mu1 != mu2 (neither 1) on condim-3 pairs, gap > 0 with
    margin > gap, solimp power 1, 2 and a non-integer one, more than one solref, and its configurations reach every distance band and
    the two-contact poses (counted on the oracle)."""
    zoo = build_zoo(tmp_path)
    classes, condims, powers, solrefs, gaps, mus = set(), set(), set(), set(), 0, set()
    for name, (m, prog, info, _) in zoo.items():
        assert m.nu == 1 and m.na == 1 and (m.nv <= 12 if name != "COMBO" else 24 < m.nv <= 30)
        assert len(prog["PPAIR"]) == m.npair and not info["dropped_pairs"]
        for row in prog["PPAIR"]:
            ct, dim, p = int(row[5]), int(row[2]), int(row[7])
            P = prog["PPAIR_d"][row[6]]
            classes.add(ct); condims.add(dim); powers.add(float(P[11])); solrefs.add(tuple(m.pair_solref[p]))
            assert P[9] == WIDTH and P[0] > P[1] >= 0
            gaps += P[1] > 0
            if dim == 3:
                assert P[2] != P[3] and 1.0 not in (P[2], P[3])
                mus.add((float(P[2]), float(P[3])))
        if name != "COMBO":
            assert [CT_NAMES[int(c)] for c in prog["PPAIR"][:, 5]] == [name]
    print("\nclasses %s, condims %s, solimp powers %s, solrefs %d, pairs with gap %d, condim-3 frictions %s"
          % ([CT_NAMES[c] for c in sorted(classes)], sorted(condims), sorted(powers), len(solrefs), gaps, sorted(mus)))
    assert classes == set(range(1, 9))
    assert condims == {1, 3} and powers == {1.0, 2.0, 2.5} and len(solrefs) >= 2 and gaps >= 3 and len(mus) == 2
    # model pair order of the combined model interleaves the two collider passes
    m, prog, info, _ = zoo["COMBO"]
    kinds = ["E" if CT_NAMES[int(r[5])] in ("CAP_ELL", "ELL_ELL") else "A" for r in sorted(prog["PPAIR"], key=lambda r: r[7])]
    assert "".join(kinds) == "AAEAEEA"
    # every class config lands in its band; both sides of solimp[3] are reached among the active contacts
    rng = np.random.default_rng(1)
    seen = dict(inactive=0, two=0, below_mid=0, above_mid=0, none=0)
    for ct in ZOO:
        m, prog, info, probe = zoo[ct]
        o = oracle_of(m); p = ZOO[ct][2]; inc = p["margin"] - p["gap"]
        cfgs = class_configs(ct, probe, rng)
        for label, q in cfgs:
            o.reset(); o.set(qpos=q); o.forward()
            d = o.f("con_dist")
            seen["none"] += o.ncon == 0
            seen["two"] += o.ncon == 2
            seen["inactive"] += int(np.sum((d >= inc) & (d <= p["margin"])))
            x = np.abs(d[d < inc] - inc) / WIDTH
            seen["below_mid"] += int(np.sum((x > 0) & (x < 1) & (x <= float(p["solimp"].split()[3]))))
            seen["above_mid"] += int(np.sum((x > float(p["solimp"].split()[3])) & (x < 1)))
        labels = {lb for lb, _ in cfgs}
        if ct == "CAP_CAP":
            for lb, q in cfgs:
                o.reset(); o.set(qpos=q); o.forward()
                if lb.startswith("parallel"):
                    assert o.ncon == 2, lb
                if lb == "near-parallel":
                    assert o.ncon == 1
        if ct == "PLANE_CAP":
            assert {"upright", "lying"} <= labels
    print("oracle over the class configs: %s" % seen)
    assert min(seen.values()) > 0


# ----------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def zoo(tmp_path_factory):
    z = build_zoo(tmp_path_factory.mktemp("zoo"))
    yield z
    if REPORT:
        print("\ncontact zoo vs oracle:")
        for k in sorted(REPORT):
            print("  %-28s %s" % (k, REPORT[k]))


MODELS = list(ZOO) + ["COMBO"]


def _configs(zoo, name):
    m, prog, info, probe = zoo[name]
    rng = np.random.default_rng(100 + MODELS.index(name))
    return combo_configs(probe, m, rng) if name == "COMBO" else class_configs(name, probe, rng)


def _state(m, qpos, seed, degenerate):
    rng = np.random.default_rng(seed)
    n = len(qpos)
    qvel = rng.normal(0, 0.2, (n, m.nv))
    for e in np.nonzero(degenerate)[0]:           # degenerate poses keep their symmetry on the first substeps: no spin
        for b in range(m.nv // 6):
            qvel[e, 6 * b + 3:6 * b + 6] = 0.0
    return qvel, rng.uniform(0, 1, (n, m.na)), rng.uniform(0, 1, (n, m.nu))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("ct", MODELS)
def test_zoo_forward_and_rollout(zoo, ct, rows):
    """One forward pass with taps (contact count, rows, ordered pair list, distances, qacc, all finite) on every config of the class,
    then 10 chained substeps from the same states."""
    import torch
    from myosuite_b200 import vec_env
    m, prog, info, _ = zoo[ct]
    cfgs = _configs(zoo, ct)
    labels = [lb for lb, _ in cfgs]; qpos = np.stack([q for _, q in cfgs]); n = len(qpos)
    qvel, act, ctrl = _state(m, qpos, 5, [lb != "generic" for lb in labels])
    env = vec_env.MyoVecEnv(None, n, model=m, taps=True, row_storage=rows)
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_")}
    o = oracle_of(m); pmi = env.prog_info["pair_model_index"]
    inc = m.pair_margin - m.pair_gap
    worst = dict(qacc=0.0, dist=0.0, qpos=0.0, qvel=0.0); cnt = dict(checked=0, contacts=0, two=0, inactive=0)
    for e in range(n):
        msg = "%s[%s] config %d (%s)" % (ct, rows, e, labels[e])
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        assert regime_ok(o, m), msg
        assert np.isfinite(t["tap_qacc"][e]).all() and np.isfinite(t["tap_contact_dist"][e]).all(), msg
        assert tuple(t["tap_ncon"][e, :2]) == (o.ncon, o.nefc), msg
        assert t["tap_ncon"][e, 3] == 0, msg
        nc = o.ncon
        assert [pmi[k] for k in t["tap_contact_pair"][e][:nc]] == [int(k) for k in o.i("con_pair")], msg
        od = o.f("con_dist")
        np.testing.assert_allclose(t["tap_contact_dist"][e][:nc], od, rtol=DIST_RTOL, atol=DIST_ATOL, err_msg=msg)
        worst["dist"] = max(worst["dist"], float(np.abs(t["tap_contact_dist"][e][:nc] - od).max()) if nc else 0.0)
        r = relerr(t["tap_qacc"][e], o.f("qacc")); worst["qacc"] = max(worst["qacc"], r)
        assert r < FWD_QACC, msg + ": qacc deviation %.2e" % r
        cnt["checked"] += 1; cnt["contacts"] += nc; cnt["two"] += nc == 2; cnt["inactive"] += int(np.sum(od >= inc[o.i("con_pair")]))
    assert cnt["checked"] == n
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 10); torch.cuda.synchronize()
    gq, gv = env.t["qpos"].cpu().numpy(), env.t["qvel"].cpu().numpy()
    assert np.isfinite(gq).all() and np.isfinite(gv).all()
    for e in range(n):
        msg = "%s[%s] config %d (%s), 10 substeps" % (ct, rows, e, labels[e])
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.step(10)
        worst["qpos"] = max(worst["qpos"], float(np.abs(gq[e] - o.f("qpos")).max())); worst["qvel"] = max(worst["qvel"], relerr(gv[e], o.f("qvel")))
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=ROLL_QPOS, err_msg=msg)
        assert relerr(gv[e], o.f("qvel")) < ROLL_QVEL, msg
    REPORT["%s[%s]" % (ct, rows)] = ("configs %d/%d checked (%d degenerate), contacts %d, two-contact %d, inactive %d; worst qacc %.1e, "
                                     "dist %.1e, 10-substep qpos %.1e qvel %.1e" % (cnt["checked"], n, sum(lb != "generic" for lb in labels),
                                                                                    cnt["contacts"], cnt["two"], cnt["inactive"], worst["qacc"],
                                                                                    worst["dist"], worst["qpos"], worst["qvel"]))
    print(REPORT["%s[%s]" % (ct, rows)])
    assert cnt["inactive"] > 0 or np.all(m.pair_gap == 0)
    if ct in ("CAP_CAP", "PLANE_CAP"):
        assert cnt["two"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("ct", MODELS)
def test_zoo_product_step(zoo, ct, rows):
    """The same states through env.step on a batch without taps, so that a product kernel runs, against oracle.step(frame_skip)."""
    import torch
    from myosuite_b200 import vec_env
    from oracle import env_oracle
    m, prog, info, _ = zoo[ct]
    cfgs = _configs(zoo, ct)
    labels = [lb for lb, _ in cfgs]; qpos = np.stack([q for _, q in cfgs]); n = len(qpos)
    qvel, act, _ = _state(m, qpos, 6, [lb != "generic" for lb in labels])
    env = vec_env.MyoVecEnv(None, n, model=m, row_storage=rows)
    assert not any(k.startswith("tap_") for k in env.t)
    li = env.batch.launch_info()
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    a = np.random.default_rng(7).uniform(-1, 1, (n, m.nu)).astype(np.float32)
    launches = env.batch.launches
    env.step(torch.as_tensor(a, device=env.device)); torch.cuda.synchronize()
    assert env.batch.launches == launches + 1 + li["regroup"]
    N = env.get_env_state()
    assert np.all(N["time"] == env.n_frames * m.opt_timestep) or np.allclose(N["time"], env.dt)
    o = oracle_of(m); worst = dict(qpos=0.0, qvel=0.0, qacc=0.0)
    for e in range(n):
        msg = "%s[%s] config %d (%s), product step" % (ct, rows, e, labels[e])
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=env_oracle.action_to_ctrl(a[e].astype(np.float64)))
        o.step(env.n_frames)
        assert np.isfinite(N["qpos"][e]).all() and np.isfinite(N["qacc_warmstart"][e]).all(), msg
        worst["qpos"] = max(worst["qpos"], float(np.abs(N["qpos"][e] - o.f("qpos")).max()))
        worst["qvel"] = max(worst["qvel"], relerr(N["qvel"][e], o.f("qvel"))); worst["qacc"] = max(worst["qacc"], relerr(N["qacc_warmstart"][e], o.f("qacc")))
        np.testing.assert_allclose(N["qpos"][e], o.f("qpos"), rtol=0, atol=MID["qpos"], err_msg=msg)
        assert relerr(N["qvel"][e], o.f("qvel")) < MID["qvel"], msg
        assert relerr(N["qacc_warmstart"][e], o.f("qacc")) < MID["qacc"], msg
        np.testing.assert_allclose(N["act"][e], o.f("act"), rtol=0, atol=1e-12, err_msg=msg)
    assert int(env.t["overflow"].sum().item()) == 0
    REPORT["%s[%s] product" % (ct, rows)] = ("%s kernel, %d warps/CTA, grid %d; %d configs, %d substeps; worst qpos %.1e qvel %.1e qacc %.1e"
                                             % ("w14" if li["use_w14"] else "k320", li["warps_per_cta"], li["grid"], n, env.n_frames,
                                                worst["qpos"], worst["qvel"], worst["qacc"]))
    print(REPORT["%s[%s] product" % (ct, rows)])


def _combo_full(zoo):
    """The combined scene, its full oracle contact list [(model pair, dist)] and the kernel's keep order (analytic pairs first, each
    pass in model pair order)."""
    m, prog, info, probe = zoo["COMBO"]
    q = combo_config(probe, m)
    o = oracle_of(m); o.reset(); o.set(qpos=q); o.forward()
    full = list(zip((int(p) for p in o.i("con_pair")), o.f("con_dist").copy()))
    ell = {int(r[7]) for r in prog["PPAIR"] if CT_NAMES[int(r[5])] in ("CAP_ELL", "ELL_ELL")}
    keep_order = [c for c in full if c[0] not in ell] + [c for c in full if c[0] in ell]
    return m, q, full, keep_order, ell


def test_combo_scene_structure(tmp_path):
    """The combined scene has the contacts the overflow test relies on: two from the floor-capA and from the parallel capA-capC pair,
    the floor-ellB pair detected but inactive, and ellipsoid contacts after the analytic ones."""
    zoo = build_zoo(tmp_path, ["COMBO"])
    m, q, full, keep, ell = _combo_full(zoo)
    pairs = [c[0] for c in full]
    print("\ncombined scene, oracle contacts (model pair, dist): %s" % [(p, "%.4f" % d) for p, d in full])
    assert pairs.count(0) == 2 and pairs.count(3) == 2 and 1 in pairs and 2 in pairs and 6 in pairs and len(full) >= 8
    d1 = [d for p, d in full if p == 1][0]
    assert 0.004 <= d1 <= 0.006                                   # floor-ellB: inside (margin - gap, margin]
    assert [c[0] for c in keep[:7]] == [0, 0, 1, 3, 3, 6, 2] and all(c[0] in ell for c in keep[6:])


MAXCON = {4: "straddle", 5: "whole", 7: "whole"}        # kept: 4 splits the parallel capsule pair, 5 ends before the ellipsoid pass, 7 reaches into it


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("maxcon", list(MAXCON))
def test_combo_overflow(zoo, maxcon, rows):
    """More contacts than maxcon: the overflow flag, ncon == maxcon, the kept contacts are the first maxcon of (analytic contacts in
    model pair order, then ellipsoid contacts in model pair order), reported in model pair order with the oracle's distances; qacc
    against an oracle of the model without the dropped pairs when whole pairs are kept; the product path's sticky overflow flag is set
    by step and cleared by reset."""
    import torch
    from myosuite_b200 import vec_env
    m, q, full, keep_order, ell = _combo_full(zoo)
    n = 4
    qpos = np.tile(q, (n, 1)); rng = np.random.default_rng(3)
    qvel, act, ctrl = rng.normal(0, 0.1, (n, m.nv)), rng.uniform(0, 1, (n, m.na)), rng.uniform(0, 1, (n, m.nu))
    env = vec_env.MyoVecEnv(None, n, model=m, taps=True, maxcon=maxcon, row_storage=rows)
    assert env.dims.maxcon == maxcon
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_")}
    pmi = env.prog_info["pair_model_index"]
    kept = keep_order[:maxcon]
    exp = sorted(kept, key=lambda c: c[0])                  # stable: the two contacts of a pair keep their collider order
    whole = all(sum(1 for c in kept if c[0] == p) == sum(1 for c in full if c[0] == p) for p in {c[0] for c in kept})
    assert whole == (MAXCON[maxcon] == "whole")
    for e in range(n):
        assert t["tap_ncon"][e, 3] == 1 and t["tap_ncon"][e, 0] == maxcon
        assert [pmi[k] for k in t["tap_contact_pair"][e][:maxcon]] == [c[0] for c in exp]
        np.testing.assert_allclose(t["tap_contact_dist"][e][:maxcon], [c[1] for c in exp], rtol=DIST_RTOL, atol=DIST_ATOL)
        assert np.isfinite(t["tap_qacc"][e]).all()
    worst = float("nan")
    if whole:
        keep_pairs = sorted({c[0] for c in kept})
        sub = [COMBO_PAIRS[p] for p in keep_pairs]
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            o = oracle_of(compile_xml(zoo_xml(COMBO_GEOMS, sub), d, "combo_kept"))
        worst = 0.0
        for e in range(n):
            o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
            assert o.ncon == maxcon
            r = relerr(t["tap_qacc"][e], o.f("qacc")); worst = max(worst, r)
            assert r < FWD_QACC
    # the product path: sticky per-env flag, set by step, cleared by the env's reset (the physics-only batch resets to qpos0)
    envp = vec_env.MyoVecEnv(None, n, model=m, maxcon=maxcon, row_storage=rows)
    envp.set_state(qpos=qpos, qvel=qvel, act=act)
    envp.step(torch.zeros(n, m.nu, device=envp.device)); torch.cuda.synchronize()
    assert np.all(envp.t["overflow"].cpu().numpy() == 1)
    assert np.isfinite(envp.t["qpos"].cpu().numpy()).all() and np.isfinite(envp.t["qvel"].cpu().numpy()).all()
    envp.reset(); torch.cuda.synchronize()
    assert np.all(envp.t["overflow"].cpu().numpy() == 0)
    np.testing.assert_array_equal(envp.t["qpos"].cpu().numpy(), np.tile(m.qpos0, (n, 1)))
    REPORT["COMBO maxcon %d[%s]" % (maxcon, rows)] = ("kept %s of %d contacts (%s); qacc vs the kept-pairs oracle %.1e"
                                                      % ([c[0] for c in exp], len(full), MAXCON[maxcon], worst))
    print(REPORT["COMBO maxcon %d[%s]" % (maxcon, rows)])
