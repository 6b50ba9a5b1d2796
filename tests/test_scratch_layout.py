"""The shared-memory scratch layout of the step kernel at every contact capacity.

Each env-warp works in one slice of shared memory.  Most of it is a scratch that `fill_devmodel` (myo_b200.cu) time-multiplexes
between the stages of a substep, and its layout is decided per batch from the model's sizes and the contact capacity `maxcon`: the
contact head (integer records, contact records) grows with maxcon, the body poses sit right behind it, PLACE puts each tendon and CRB
array into the free part of the head when it fits there and behind the poses otherwise, the solve stage reuses everything behind the
head, aref lives at the head of the Hessian region when it fits and the warm start in its tail when that is provably idle.  maxcon is
a public kwarg, so a user who changes it gets a layout of its own.

CPU: `myo_model_layout` reports what fill_devmodel decided.  The lifetime table below restates, from the phase code, which bytes each
stage reads or writes; the checks assert that no two regions that are live in a common stage overlap and that every region lies in
its reservation and in the slice, for every shipped model and zoo model at maxcon 1 .. 64 in both row storages.

GPU: no kernel arithmetic depends on maxcon except through the contacts it drops (rows are numbered by contact rank, lanes follow the
row index, the dense solver's order is chol_pad(nv)), so an env whose contacts all fit must give BIT-IDENTICAL results at every
capacity.  A difference means that a stage read a region another stage had overwritten, or that the arithmetic depends on the
layout.  The tests run one capacity per distinct layout signature plus 1, the largest and the default, on the debug kernel (taps) and
on the product kernels, and two more layout perturbations with identical physics (the hold task's eight extra persistent slots, and
extra world pairs that never touch)."""

import numpy as np
import pytest

import test_actuation_zoo as az
import test_contact_zoo as cz
from parity_helpers import relerr

ROWS = ["p48", "f64"]
JAC_BYTES = {"p48": 6, "f64": 8}
VARIANT = {"p48": None, "f64": "f64rows"}
CAPS = list(range(1, 65))
DEFAULT_MAXCON = 32
SHIPPED = ["myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso"]
PLACED = ("mom", "tlen", "tvel", "tfrc", "PL", "U", "cin", "crb", "bf")       # the PLACE decisions of fill_devmodel, in its order
MID = dict(qpos=2e-7, qvel=1e-5, qacc=1e-6)         # the mid-episode bounds of test_product_parity.py (oracle anchor)
REPORT = {}

# ----------------------------------------------------------------------------- the lifetime table
# Stages of one substep, in order.  "rank" is the first part of phase_constraints (equality and limit rows, the rank keys and the rank
# scan), "rows" the contact rows (Jacobians, masks, regularisers, aref; the contact taps read the records there).  "solve0" is the
# entry of phase_solve (warm start, J a - aref), "newton" its iterations, "euler" phase_integrate up to its (M + hB) solve, "store" the
# velocity / warm start / position update, the step epilogue (task_observe re-runs kinematics, tendons and actuation for the
# observation) and the store of the state.
STAGES = ("kin", "ten", "act", "crb", "col", "rank", "rows", "solve0", "newton", "euler", "store")


def span(a, b):
    return frozenset(STAGES[STAGES.index(a):STAGES.index(b) + 1])


ALL = frozenset(STAGES)
# Regions that share bytes on purpose although both are live in one stage: each Newton iteration and the integrator build EITHER the
# dense H or the tree-sparse Hs / LD / Dinv, never both (myo_solver.cuh:432-470, 505-514).
EXCLUSIVE = {frozenset(p) for p in (("H", "Hs"), ("H", "LD"), ("H", "Dinv"))}


def chol_pad(n):
    """the dense solver's order (myo_solver.cuh chol_pad)"""
    return n if n > 32 else 8 if n <= 8 else n if n in (23, 29) else (n + 3) & ~3


def model_dims(m, prog, lay):
    from myosuite_b200 import program as P
    d = prog["P_dims"]
    nlimrow = int(d[P.PD_NLIMROW]) if d[P.PD_NLIMROW] > 0 else 2 * int(d[P.PD_NLIM])
    out = dict(nq=m.nq, nv=m.nv, na=m.na, nM=m.nM, njnt=m.njnt, nbd=int(d[P.PD_NBD]), nnz=int(d[P.PD_NNZ]), nta=int(d[P.PD_NTA]),
               nsp=int(d[P.PD_NSP]), nwe=int(d[P.PD_NWE]), spA=int(d[P.PD_SPLIT_SP]), weA=int(d[P.PD_SPLIT_WE]), ngc=int(d[P.PD_NGC]),
               kcand=int(d[P.PD_NPAIR] - d[P.PD_NPAIR_ANALYTIC]), maxpath=int(d[P.PD_MAXPATH]), neq=int(d[P.PD_NEQ]), nlimrow=nlimrow,
               nwz=int(d[P.PD_NWE_SPH_IN] + d[P.PD_NWE_CYL_IN]), npair=int(d[P.PD_NPAIR]), mc=lay["maxcon"], neprm=lay["o_size"]["eprm"])
    out["maxefc"] = out["neq"] + nlimrow + 4 * out["mc"]
    out["nvp"] = chol_pad(m.nv)
    return out


def lifetime_table(d, jac_bytes, sines_at="gpose"):
    """[(region, layout field it is addressed from, byte offset in it, bytes, stages in which it is live)].  A region is live from
    the stage that writes it to the last stage that reads it.  Line numbers cite the phase code."""
    nv, nvp, mc, mp, nlr, efc = d["nv"], d["nvp"], d["mc"], d["maxpath"], d["nlimrow"], d["maxefc"]
    nsA, nwA = d["spA"], d["weA"]
    nsB, nwB = d["nsp"] - nsA, d["nwe"] - nwA
    cp = 8 * (mc + (mc + 1) // 2)                      # S_cpair: after the u64 masks and the i32 row words (myo_device.cuh:74)
    T = [
        # phase_kinematics: hinge sines / cosines, one lane-parallel pass, read by the level loop (myo_device.cuh:149-150,176)
        ("sines", sines_at, 0, 16 * d["njnt"], span("kin", "kin")),
        # body poses: written by the level loop (186-188), read by tendons (world_point 119, wrap_element 290), body inertia (196),
        # collision (geom_pose_all 471, geom_mat 483); phase_constraints takes its lever arms from dax / dan, not from the poses
        ("xpos", "xpos", 0, 24 * d["nbd"], span("kin", "col")),
        ("xmat", "xmat", 0, 72 * d["nbd"], span("kin", "col")),
        # tendon passes: one group at a time in U / PL (phase_tendon 330-335, wrap_element 307-325, phase_tendon_moments 342-354)
        ("U", "U", 0, 24 * max(nsA + 2 * nwA, nsB + 2 * nwB), span("ten", "ten")),
        ("PL", "PL", 0, 8 * max(nsA + nwA, nsB + nwB), span("ten", "ten")),
        # moments and tendon lengths / velocities / forces: tendon stage (349, 354, 364) to actuation (389, 406, 415); the walk
        # observation reads them after the re-run in task_observe (myo_b200.cu:169-172), i.e. in its own ten / act stages
        ("mom", "mom", 0, 8 * d["nnz"], span("ten", "act")),
        ("tlen", "tlen", 0, 8 * d["nta"], span("ten", "act")),
        ("tvel", "tvel", 0, 8 * d["nta"], span("ten", "act")),
        ("tfrc", "tfrc", 0, 8 * d["nta"], span("ten", "act")),
        # body inertia -> CRB -> bias (196-208, 422-436, 442-461)
        ("cin", "cin", 0, 80 * d["nbd"], span("crb", "crb")),
        ("crb", "crb", 0, 80 * d["nbd"], span("crb", "crb")),
        ("bf", "bf", 0, 48 * d["nbd"], span("crb", "crb")),
        # collision: geom poses (468-475) and the ellipsoid candidate list (701-709)
        ("gpose", "gpose", 0, 48 * d["ngc"], span("col", "col")),
        ("clist", "clist", 0, 4 * d["kcand"], span("col", "col")),
        # contact records: written by store_contact (669-677), read by phase_constraints (myo_solver.cuh:153,172) and the contact
        # taps (myo_b200.cu:66); the solve reuses the region for jar / jv
        ("con", "con", 0, 80 * mc, span("col", "rows")),
        # icon sub-fields (myo_solver.cuh:54-60, myo_device.cuh:74): S_cmask u64[maxcon] | S_crown i32[maxcon] | S_cpair i16[maxcon] |
        # S_lrow i16[nlimrow + 4] | S_drow u8[maxefc]; cpair from the colliders, the rest from phase_constraints, all read by the solve
        ("cmask", "icon", 0, 8 * mc, span("rows", "newton")),
        ("crown", "icon", 8 * mc, 4 * mc, span("rank", "newton")),
        ("cpair", "icon", cp, 2 * mc, span("col", "newton")),
        ("lrow", "icon", cp + 2 * mc, 2 * nlr, span("rank", "newton")),
        ("drow", "icon", cp + 2 * mc + 2 * (nlr + 4), efc, span("rank", "newton")),
        # rank keys of the contact ordering, in the Jacobian region before the Jacobians are written (myo_solver.cuh:146-157)
        ("keys", "conJ", 0, 4 * mc, span("rank", "rank")),
        # regularisers, equality Jacobian entries and aref (127, 137, 181-184); aref is last read at the solve's entry (415)
        ("D", "efD", 0, 8 * (d["neq"] + nlr + mc), span("rank", "newton")),
        ("eqJ", "eqJ", 0, 8 * d["neq"], span("rank", "newton")),
        ("aref", "efA", 0, 8 * efc, span("rank", "solve0")),
        # Newton: jar (414-415, 492), jv (424, 475), qacc a (413, read by the integrator 516), g | p (423, 435; chol_dense writes
        # chol_pad(nv) slots, 236), M a (414, 488, read by the integrator 503), M p (475)
        ("jar", "efR", 0, 8 * efc, span("solve0", "newton")),
        ("jv", "efV", 0, 8 * efc, span("newton", "newton")),
        ("a", "va", 0, 8 * nv, span("solve0", "store")),
        ("g|p", "vg", 0, 8 * nvp, span("newton", "euler")),
        ("Ma", "vMa", 0, 8 * nv, span("solve0", "euler")),
        ("Mp", "vMp", 0, 8 * nv, span("newton", "newton")),
        # Hessian and factors: Newton iterations (440-467) and the integrator (506, 511-513).  The unconstrained exit (409-411) factors
        # into LD / Dinv at the solve's entry; it runs only with nefc == 0, when aref, jar and the warm start hold nothing live, so its
        # writes are counted with the iterations.
        ("H", "H", 0, 8 * nvp * (nvp + 1) // 2, span("newton", "euler")),
        ("Hs", "Hs", 0, 8 * d["nM"], span("newton", "euler")),
        ("LD", "LD", 0, 8 * d["nM"], span("newton", "euler")),
        ("Dinv", "Dinv", 0, 8 * nv, span("newton", "euler")),
    ]
    if jac_bytes == 8:
        T.append(("jac", "conJ", 0, 24 * mp * mc, span("rows", "newton")))
    else:       # u32 high words, then the u16 middle words at 3 maxpath maxcon words (S_jac, myo_solver.cuh:37)
        T += [("jac_hi", "conJ", 0, 12 * mp * mc, span("rows", "newton")), ("jac_lo", "conJ", 12 * mp * mc, 6 * mp * mc, span("rows", "newton"))]
    # warm start: rewritten at the end of the integrator (516), read at the next solve's entry (413) or stored with the state.  A debug
    # forward pass without substeps runs no integrator and does not store it back (myo_b200.cu, store_qws), so the Newton stages may
    # reuse its bytes.
    T.append(("qws", "o:qws", 0, 8 * nv, span("kin", "solve0") | {"store"}))
    # persistent per-env arrays: live in every stage
    for name, n in (("qpos", d["nq"]), ("qvel", nv), ("act", d["na"]), ("dax", 3 * nv), ("dan", 3 * nv), ("qM", d["nM"]), ("fsm", nv),
                    ("eprm", d["neprm"]), ("wz", d["nwz"])):
        T.append((name, "o:" + name, 0, 8 * n, ALL))
    T.append(("cnt", "o:cnt", 0, 32, ALL))       # CNT_N int counters
    return T


def _field(lay, f):
    if f.startswith("o:"):
        return lay["o"][f[2:]], lay["o_size"][f[2:]]
    return lay["s"][f], lay["s_size"][f]


def placed(lay, T):
    """[(region, byte start, byte end, stages, reservation (start, end) in bytes)]"""
    out = []
    for name, f, off, nb, st in T:
        base, size = _field(lay, f)
        if name == "sines":         # not a field of its own: fill_devmodel extends the non-solve scratch for it (myo_b200.cu)
            res = (8 * base, 8 * lay["extNonSolve"])
        else:
            res = (8 * base, 8 * (base + size))
        out.append((name, 8 * base + off, 8 * base + off + nb, st, res))
    return out


def check_layout(lay, T):
    """(overlaps, bounds) violations: pairs of regions live in a common stage that share bytes, and regions outside their reservation,
    the slice, or their part of it (persistent before the scratch; the warm start in the Hessian tail only when qwsInH)."""
    R = [r for r in placed(lay, T) if r[2] > r[1]]
    bad_bounds = []
    scr, end = 8 * lay["o"]["scr"], 8 * lay["n_per_warp"]
    for name, a, b, st, (ra, rb) in R:
        if a < ra or b > rb:
            bad_bounds.append((name, "outside its reservation", (a, b), (ra, rb)))
        if a < 0 or b > end:
            bad_bounds.append((name, "outside the slice", (a, b), end))
        persistent = st == ALL
        if persistent and b > scr:
            bad_bounds.append((name, "persistent region in the scratch", (a, b), scr))
        if not persistent and name != "qws" and a < scr:
            bad_bounds.append((name, "scratch region before the scratch", (a, b), scr))
    if (8 * lay["o"]["qws"] >= scr) != bool(lay["qwsInH"]):
        bad_bounds.append(("qws", "placement disagrees with qwsInH", 8 * lay["o"]["qws"], scr))
    bad_overlap = []
    for i in range(len(R)):
        for j in range(i + 1, len(R)):
            n1, a1, b1, s1, _ = R[i]
            n2, a2, b2, s2, _ = R[j]
            if a1 < b2 and a2 < b1 and (s1 & s2) and frozenset((n1, n2)) not in EXCLUSIVE:
                bad_overlap.append((n1, n2, sorted(s1 & s2, key=STAGES.index), (a1, b1), (a2, b2)))
    return bad_overlap, bad_bounds


def signature(lay, T):
    """placement flags and the relative order of the region boundaries (ranks of the distinct byte offsets of every start and end)"""
    R = [r for r in placed(lay, T) if r[2] > r[1]]
    pts = sorted({p for r in R for p in (r[1], r[2])})
    rank = {p: k for k, p in enumerate(pts)}
    flags = tuple(int(lay["s"][f] < lay["head"]) for f in PLACED) + (lay["arefInH"], lay["qwsInH"])
    return flags + tuple((r[0], rank[r[1]], rank[r[2]]) for r in R)


# ----------------------------------------------------------------------------- the models
def far_pairs_xml(xml, body_geoms):
    """The same MJCF plus a world plane 5 m below and a world ellipsoid 4 m away, and one pair per body geom with each.  The compiler's
    reach bound (mjcf._build_collision_pairs) drops the plane pairs; the capsule-ellipsoid pairs survive it, so the iterative collider
    evaluates them every substep (more pairs, collision geoms and ellipsoid candidates) and they never touch.  The tests check that the
    contacts and their pair ids are those of the model without them."""
    world =('<geom name="xfloor" type="plane" size="0 0 1" pos="0 0 -5" contype="0" conaffinity="0"/>'
             '<geom name="xell" type="ellipsoid" size="0.02 0.03 0.04" pos="4 0 0" contype="0" conaffinity="0"/>')
    pairs = "".join('<pair geom1="xfloor" geom2="%s" margin="0.005"/>' % g for g, _ in body_geoms)
    pairs += "".join('<pair geom1="%s" geom2="xell" margin="0.005"/>' % g for g, t in body_geoms if t == "capsule")
    xml = xml.replace("</worldbody>", world + "</worldbody>", 1)
    if "</contact>" in xml:
        return xml.replace("</contact>", pairs + "</contact>", 1)
    return xml.replace("</mujoco>", "<contact>%s</contact></mujoco>" % pairs, 1)


WRAP_GEOMS = [("ca", "capsule"), ("cb", "capsule"), ("cd", "capsule"), ("cc", "capsule"), ("asph", "sphere")]
MUSCLE_GEOMS = [("ga", "capsule"), ("gb", "capsule"), ("gs", "sphere")]
SWEEP_GEOMS = [("cap", "capsule"), ("g1", "sphere"), ("g2", "sphere"), ("g4", "sphere")]


def build_models(tmp, names=None):
    """{name: dict(m, prog)} for the shipped models and the zoo models (the contact zoo's class and combined models, the actuation
    zoo's models, and WRAPX / MUSCLEX / SWEEP_16X: the same with far world pairs)."""
    from myosuite_b200 import assets, program
    out = {}
    want = lambda n: names is None or n in names
    for n in SHIPPED:
        if want(n):
            m = assets.load(n)
            out[n] = dict(m=m, prog=program.build_program(m)[0])
    if names is None or any(n in cz.MODELS for n in names):
        for n, (m, prog, info, probe) in cz.build_zoo(tmp, [n for n in cz.MODELS if want(n)]).items():
            out[n] = dict(m=m, prog=prog, probe=probe)
    if names is None or any(n in az.MODELS for n in names):
        for n, z in az.build_zoo(tmp, [n for n in az.MODELS if want(n)]).items():
            out[n] = dict(m=z["m"], prog=z["prog"], zoo=z)
    extra = {"WRAPX": lambda: far_pairs_xml(az.wrap_xml(), WRAP_GEOMS), "MUSCLEX": lambda: far_pairs_xml(az.muscle_xml(az.fit_lengthranges(tmp)), MUSCLE_GEOMS),
             "SWEEP_16X": lambda: far_pairs_xml(az.sweep_xml(16), SWEEP_GEOMS)}
    for n, mk in extra.items():
        if want(n):
            m = az.compile_xml(mk(), tmp, n)
            out[n] = dict(m=m, prog=program.build_program(m)[0])
    return out


def _cfg(maxcon, task=None):
    from myosuite_b200 import abi
    c = abi.MyoTaskCfg()
    c.maxcon = maxcon
    if task is not None:
        c.task = task
    return c


def layouts(m, prog, rows, task=None):
    """{maxcon asked: layout} for maxcon 1 .. 64 (the library clamps to min(64, 2 npair))"""
    from myosuite_b200 import abi, blob
    dm = abi.DeviceModel(*blob.pack(m, prog), variant=VARIANT[rows])
    return {c: dm.layout(_cfg(c, task)) for c in CAPS}


# ----------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    """{(model, cfg tag, rows): {maxcon: (layout, table)}} over every model (the hold model also with the hold task's cfg)"""
    from myosuite_b200 import abi
    models = build_models(tmp_path_factory.mktemp("layout"))
    out = {}
    for name, z in models.items():
        tasks = [(None, "physics")] + ([(abi.TASK_HOLD, "hold task")] if name == "myohand_hold" else [])
        for task, tag in tasks:
            for rows in ROWS:
                L = layouts(z["m"], z["prog"], rows, task)
                out[(name, tag, rows)] = {c: (lay, lifetime_table(model_dims(z["m"], z["prog"], lay), JAC_BYTES[rows])) for c, lay in L.items()}
    return models, out


def test_layout_query_agrees_with_dims(sweep):
    """myo_model_layout reports the slice size and capacity myo_model_dims reports, clamps maxcon as documented, and the lifetime
    table's dims agree with it (maxefc)."""
    from myosuite_b200 import abi, blob
    models, S = sweep
    for (name, tag, rows), per in S.items():
        m, prog = models[name]["m"], models[name]["prog"]
        if tag != "physics":
            continue
        dm = abi.DeviceModel(*blob.pack(m, prog), variant=VARIANT[rows])
        for c in (1, 7, 32, 64):
            lay = per[c][0]
            d = dm.dims(_cfg(c))
            assert lay["n_per_warp"] * 8 == d.smem_bytes_per_env and lay["maxcon"] == d.maxcon == min(c, 64, 2 * model_dims(m, prog, lay)["npair"])
            assert lay["maxefc"] == d.maxefc == model_dims(m, prog, lay)["maxefc"], (name, c)


def test_no_live_region_overlaps_and_all_in_bounds(sweep):
    """No two regions live in a common stage share a byte, and every region lies in its reservation and in [0, n_per_warp), for every
    model, cfg, row storage and maxcon 1 .. 64.  Prints the number of distinct layout signatures per model and storage."""
    models, S = sweep
    fails, sigs = [], {}
    for (name, tag, rows), per in S.items():
        s = set()
        for c, (lay, T) in per.items():
            ov, bd = check_layout(lay, T)
            fails += [(name, tag, rows, c, "overlap", x) for x in ov] + [(name, tag, rows, c, "bounds", x) for x in bd]
            s.add(signature(lay, T))
        sigs[(name, tag, rows)] = len(s)
    print("\ndistinct layout signatures over maxcon 1..64 (model, cfg, rows): %s" % {"%s/%s/%s" % k: v for k, v in sorted(sigs.items())})
    assert not fails, fails[:20]


def test_every_placement_branch_is_reached(sweep):
    """Every PLACE decision of fill_devmodel falls into the head and behind the poses, and arefInH and qwsInH take both values, somewhere
    in the sweep.  Prints where each branch is reached."""
    models, S = sweep
    seen = {}
    for (name, tag, rows), per in S.items():
        for c, (lay, T) in per.items():
            for f in PLACED:
                seen.setdefault((f, "head" if lay["s"][f] < lay["head"] else "behind K"), set()).add(name)
            for f in ("arefInH", "qwsInH"):
                seen.setdefault((f, bool(lay[f])), set()).add(name)
    print("\nplacement branches -> models reaching them:")
    for k in sorted(seen, key=str):
        print("  %-22s %s" % ("%s %s" % k, sorted(seen[k])))
    want = {(f, s) for f in PLACED for s in ("head", "behind K")} | {(f, b) for f in ("arefInH", "qwsInH") for b in (False, True)}
    assert want <= set(seen), want - set(seen)


def test_check_flags_the_old_sines_placement(sweep):
    """The check is strong enough to see the bug the kinematics phase had: the hinge sines parked at the head of the Hessian region
    overlap the body poses the level loop writes, on the shipped hand at small capacities."""
    models, S = sweep
    hit = {}
    for name in ("myohand_pose", "myohand_hold"):
        m, prog = models[name]["m"], models[name]["prog"]
        for c, (lay, _) in S[(name, "physics", "p48")].items():
            T = lifetime_table(model_dims(m, prog, lay), JAC_BYTES["p48"], sines_at="H")
            ov, _ = check_layout(lay, T)
            if any("sines" in (o[0], o[1]) and {"xpos", "xmat"} & {o[0], o[1]} for o in ov):
                hit.setdefault(name, []).append(c)
    print("\nold sines placement flagged at maxcon: %s" % hit)
    assert 1 in hit.get("myohand_pose", []) and 4 in hit.get("myohand_pose", []) and 1 in hit.get("myohand_hold", []), hit


def gpu_capacities(per):
    """one capacity per distinct layout signature (the smallest reaching it), plus 1, the largest (the reference) and the default"""
    first = {}
    for c in sorted(per):
        lay, T = per[c]
        first.setdefault(signature(lay, T), lay["maxcon"])
    top = per[64][0]["maxcon"]
    caps = sorted(set(first.values()) | {per[1][0]["maxcon"], top, per[DEFAULT_MAXCON][0]["maxcon"]})
    return [c for c in caps if c >= 1], top, len(first)


# ----------------------------------------------------------------------------- GPU
GPU_MODELS = ["myohand_pose", "myohand_hold", "myolegs", "COMBO", "SWEEP_16", "SWEEP_40", "WRAPX", "MUSCLEX"]
TASK_OF = {"myohand_pose": "myoHandPoseRandom-v0", "myohand_hold": "myoHandObjHoldRandom-v0", "myolegs": "myoLegStandRandom-v0"}
TAPS = ("tap_qacc", "tap_qfrc_smooth", "tap_qM", "tap_moment", "tap_ten_length", "tap_actuator_force")
STATE = ("qpos", "qvel", "act", "qacc_warmstart")
MIN_COMPARED = 32
POOL_ENVS = 192                     # task batch the shipped models' states come from (about 1 in 10 hand states has at most one contact)


@pytest.fixture(scope="module")
def gpu_models(tmp_path_factory):
    models = build_models(tmp_path_factory.mktemp("layout_gpu"), GPU_MODELS + ["WRAP", "SWEEP_16", "SWEEP_16X"])
    yield models
    if REPORT:
        print("\nscratch layout, bit-identity across capacities:")
        for k in sorted(REPORT):
            print("  %-34s %s" % (k, REPORT[k]))


def _lift_free(m, qpos, rng, top):
    """copies with every free body raised by 0 .. top (fewer contacts)"""
    q = qpos.copy()
    for j in range(m.njnt):
        if m.jnt_type[j] == 0:
            q[:, m.jnt_qposadr[j] + 2] += rng.uniform(0, top, len(q))
    return q


def state_pool(name, z):
    """qpos, qvel, act, qacc_warmstart, ctrl: reset states and states after 2, 4 and 8 steps of random actions at the default capacity
    (task batches for the shipped models; the zoo's configurations and 20 / 60 substeps for the zoo models), and lifted copies"""
    import torch
    from myosuite_b200 import vec_env
    m = z["m"]
    rng = np.random.default_rng(5)
    snaps = []
    if name in TASK_OF:
        env = vec_env.MyoVecEnv(TASK_OF[name], POOL_ENVS, seed=3, auto_reset=False)
        env.reset(seed=3)
        for k in range(9):
            if k in (0, 2, 4, 8):
                S = env.get_env_state()
                snaps.append([S[key] for key in STATE])
            env.step(torch.as_tensor(rng.uniform(-1, 1, (POOL_ENVS, m.nu)).astype(np.float32), device=env.device))
    else:
        if "zoo" in z:
            qpos, qvel, act = z["zoo"]["qpos"], z["zoo"]["qvel"], z["zoo"]["act"]
        elif name.startswith("WRAP") or name.startswith("MUSCLE"):          # the far-pair variants: the zoo's own configurations
            qpos = az.wrap_configs(m) if name.startswith("WRAP") else az.muscle_configs(m)[0]
            qvel, act = rng.normal(0, 0.5, (len(qpos), m.nv)), rng.uniform(0, 1, (len(qpos), m.na))
        else:       # the contact zoo's combined model
            qpos = np.array([q for _, q in cz._configs({name: (m, z["prog"], None, z["probe"])}, name)])
            qvel, act, _ = cz._state(m, qpos, 7, np.zeros(len(qpos), bool))
        n = len(qpos)
        env = vec_env.MyoVecEnv(None, n, model=m, taps=True)
        ctrl = rng.uniform(0, 1, (n, m.nu))
        env.set_state(qpos=qpos, qvel=qvel, act=act)
        for k in (0, 20, 40):
            if k:
                env.forward_debug(ctrl, k)
            S = env.get_env_state()
            snaps.append([S[key] for key in STATE])
    pool = [np.concatenate([s[i] for s in snaps]) for i in range(4)]
    if (m.jnt_type == 0).any():
        lifted = [_lift_free(m, pool[0], rng, top) for top in (0.05, 0.15)]
        pool = [np.concatenate(lifted + [pool[0]])] + [np.concatenate([p, p, p]) for p in pool[1:]]
    pool[2] = pool[2][:, :max(m.na, 1)]
    return dict(qpos=pool[0], qvel=pool[1], act=pool[2], qacc_warmstart=pool[3], ctrl=rng.uniform(0, 1, (len(pool[0]), m.nu)))


def batch_at(base, maxcon):
    """a batch of base's model and cfg at another capacity, bound to base's tensors (the contact taps sized for its capacity): one
    program per model, one batch per capacity"""
    import torch
    from myosuite_b200 import abi
    cfg = abi.MyoTaskCfg.from_buffer_copy(base.cfg)
    cfg.maxcon = maxcon
    b = abi.Batch(base.dev_model, base.device_index, base.num_envs, cfg)
    mc = base.dev_model.dims(cfg).maxcon
    t = {k: v for k, v in base.t.items() if k in abi.BUFFER_FIELDS}
    if "tap_contact_pair" in t:
        t["tap_contact_pair"] = torch.zeros(base.num_envs, max(mc, 1), dtype=torch.int32, device=base.device)
        t["tap_contact_dist"] = torch.zeros(base.num_envs, max(mc, 1), dtype=torch.float64, device=base.device)
    b.bind(**t)
    return b, t, mc


def forward_runner(m, rows, n):
    """run(maxcon, states, nsub): the debug kernel at that capacity, one forward pass with taps (nsub = 0) or nsub substeps, from the
    states and their warm starts; returns the taps and the state as numpy arrays"""
    import torch
    from myosuite_b200 import vec_env
    base = vec_env.MyoVecEnv(None, n, model=m, taps=True, row_storage=rows)

    def run(maxcon, st, nsub):
        b, t, mc = batch_at(base, maxcon)
        for k in STATE:
            v = torch.as_tensor(st[k], dtype=torch.float64, device=base.device)
            t[k][:, :v.shape[1]] = v
        ctrl = torch.as_tensor(st["ctrl"], dtype=torch.float64, device=base.device).contiguous()
        b.forward_debug(ctrl, nsub, stream=base._stream())
        torch.cuda.synchronize()
        out = {k: v.cpu().numpy().copy() for k, v in t.items() if k.startswith("tap_") or k in STATE}
        out["maxcon"] = mc
        return out
    return run


def run_forward(m, rows, maxcon, st, nsub):
    return forward_runner(m, rows, len(st["qpos"]))(maxcon, st, nsub)


def ndiff(a, b):
    """number of values whose bit patterns differ (0.0 vs -0.0 and NaN payloads count)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    u = np.dtype("u%d" % a.dtype.itemsize)
    return int(np.count_nonzero(a.view(u) != b.view(u)))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", GPU_MODELS)
def test_forward_bit_identical_across_capacities(gpu_models, name, rows):
    """At one capacity per layout signature (plus 1, the largest and the default): one forward pass with taps and 3 chained substeps,
    bit for bit against the largest capacity on every env whose contacts all fit.  Forward: qacc, qfrc_smooth, qM, tendon moments and
    lengths, actuator forces, ncon / nefc / Newton iterations, the ordered pair ids and distances, and the stored-back warm start.
    Substeps: qpos, qvel, act, warm start.  At the smallest and largest capacity a few compared envs are also checked against the
    oracle at the mid-episode bounds."""
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    z = gpu_models[name]; m = z["m"]
    per = {c: (lay, lifetime_table(model_dims(m, z["prog"], lay), JAC_BYTES[rows])) for c, lay in layouts(m, z["prog"], rows).items()}
    for c, (lay, T) in per.items():          # the host check first: no GPU run of a layout that addresses past the slice
        ov, bd = check_layout(lay, T)
        assert not ov and not bd, (c, ov[:3], bd[:3])
    caps, top, nsig = gpu_capacities(per)
    st = state_pool(name, z)
    n = len(st["qpos"])
    run = forward_runner(m, rows, n)
    ref0, ref3 = run(top, st, 0), run(top, st, 3)
    assert ref0["maxcon"] == top
    ncon_ref, seen_ref = ref0["tap_ncon"][:, 0], ref3["tap_phase_cycles"][:, 12]
    far = name in ("WRAPX", "MUSCLEX")
    if far:
        assert (ncon_ref == 0).all() and (seen_ref == 0).all()
    o = Oracle(*blob.pack(m))
    lines, total = [], 0
    for c in caps:
        g0, g3 = (ref0, ref3) if c == top else (run(c, st, 0), run(c, st, 3))
        ok0 = np.nonzero((ncon_ref <= c) & (g0["tap_ncon"][:, 3] == 0) & (ref0["tap_ncon"][:, 3] == 0))[0]
        ok3 = np.nonzero(seen_ref <= c)[0]      # max contacts over the 3 substeps at the reference (tap_phase_cycles[12])
        by = {k: ndiff(g0[k][ok0], ref0[k][ok0]) for k in TAPS + ("qacc_warmstart",)}
        by["ncon/nefc/niter"] = ndiff(g0["tap_ncon"][ok0, :3], ref0["tap_ncon"][ok0, :3])
        by["pair/dist"] = sum(ndiff(g0["tap_contact_pair"][e, :int(ncon_ref[e])], ref0["tap_contact_pair"][e, :int(ncon_ref[e])])
                              + ndiff(g0["tap_contact_dist"][e, :int(ncon_ref[e])], ref0["tap_contact_dist"][e, :int(ncon_ref[e])]) for e in ok0)
        by.update({"3 substeps " + k: ndiff(g3[k][ok3], ref3[k][ok3]) for k in STATE})
        # the forward pass advances nothing: every env stores back exactly the state it was given, warm start included
        by.update({"kept " + k: ndiff(g0[k][:, :st[k].shape[1]], np.asarray(st[k], np.float64)) for k in STATE})
        nd = sum(by.values())
        total += nd
        withc = int((ncon_ref[ok0] > 0).sum())
        lines.append("maxcon %d: %d / %d envs compared (%d with contacts, %d excluded for overflow), %d / %d over 3 substeps, %d differing"
                     % (c, len(ok0), n, withc, n - len(ok0), len(ok3), n, nd))
        assert nd == 0, "%s[%s] maxcon %d: %d values differ from maxcon %d: %s" % (name, rows, c, nd, top, {k: v for k, v in by.items() if v})
        assert len(ok0) >= MIN_COMPARED and len(ok3) >= MIN_COMPARED, lines[-1]
        assert far or withc > 0, lines[-1]
        # oracle anchor at the smallest and the largest capacity
        if c in (caps[0], top):
            anchor = [e for e in ok3 if ncon_ref[e] > 0][:4] + [e for e in ok3 if ncon_ref[e] == 0][:2]
            for e in anchor:
                o.reset(); o.set(qpos=st["qpos"][e], qvel=st["qvel"][e], act=st["act"][e][:m.na], ctrl=st["ctrl"][e]); o.forward()
                assert relerr(g0["tap_qacc"][e], o.f("qacc")) < MID["qacc"], (name, rows, c, e)
                o.reset(); o.set(qpos=st["qpos"][e], qvel=st["qvel"][e], act=st["act"][e][:m.na], ctrl=st["ctrl"][e]); o.f("wrap_warm")[:] = 1; o.step(3)
                np.testing.assert_allclose(g3["qpos"][e], o.f("qpos"), rtol=0, atol=MID["qpos"])
                assert relerr(g3["qvel"][e], o.f("qvel")) < MID["qvel"], (name, rows, c, e)
    REPORT["%s[%s] forward" % (name, rows)] = "%d signatures, capacities %s; %d differing values" % (nsig, caps, total)
    print("\n%s[%s]: %d layout signatures, capacities %s, reference maxcon %d\n  %s" % (name, rows, nsig, caps, top, "\n  ".join(lines)))


PRODUCT_KEYS = ("qpos", "qvel", "act", "qacc_warmstart", "time", "obs", "reward", "done", "truncated", "last_return")


def product_runner(task_id, rows, n):
    """run(maxcon, actions): a task batch at that capacity (product kernels: no taps bound), reset with one seed (episode counters
    rewound) and stepped with the actions; returns the outputs, the envs whose overflow flag rose on any step, the launch shape and the
    capacity"""
    import torch
    from myosuite_b200 import vec_env
    base = vec_env.MyoVecEnv(task_id, n, seed=11, row_storage=rows)
    assert not any(k.startswith("tap_") for k in base.t)

    def run(maxcon, actions):
        b, t, mc = batch_at(base, maxcon)
        for k in ("episode_count", "last_return", "overflow"):
            t[k].zero_()
        b.reset(seed=11, env_offset=0, stream=base._stream())
        ov = np.zeros(n, bool)
        for a in actions:
            t["action"].copy_(torch.as_tensor(a, device=base.device))
            b.step(stream=base._stream())
            ov |= t["overflow"].cpu().numpy() != 0
        torch.cuda.synchronize()
        return {k: t[k].cpu().numpy().copy() for k in PRODUCT_KEYS}, ov, b.launch_info(), mc
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", list(TASK_OF))
def test_product_step_bit_identical_across_capacities(gpu_models, name, rows):
    """Task batches with the same seed and 3 steps of the same actions at each capacity: state, obs, reward, done, truncated and last
    return bit for bit against the largest capacity on every env whose overflow flag never rose.  The launch shape (kernel, warps per
    CTA, rounds) changes with the capacity; the results must not."""
    z = gpu_models[name]; m = z["m"]
    per = {c: (lay, lifetime_table(model_dims(m, z["prog"], lay), JAC_BYTES[rows])) for c, lay in layouts(m, z["prog"], rows).items()}
    caps, top, _ = gpu_capacities(per)
    n = 1024
    rng = np.random.default_rng(21)
    actions = [rng.uniform(-1, 1, (n, m.nu)).astype(np.float32) for _ in range(3)]
    run = product_runner(TASK_OF[name], rows, n)
    ref, ov_ref, li_ref, mc = run(top, actions)
    assert mc == top
    lines, shapes = [], set()
    for c in caps:
        got, ov, li, _ = (ref, ov_ref, li_ref, top) if c == top else run(c, actions)
        shapes.add((li["use_w14"], li["warps_per_cta"], li["rounds"]))
        ok = np.nonzero(~ov & ~ov_ref)[0]
        nd = sum(ndiff(got[k][ok], ref[k][ok]) for k in PRODUCT_KEYS)
        lines.append("maxcon %d: %s kernel, %d warps/CTA, %d rounds; %d / %d envs compared, %d differing"
                     % (c, "w14" if li["use_w14"] else "k320", li["warps_per_cta"], li["rounds"], len(ok), n, nd))
        assert nd == 0, "%s[%s] maxcon %d: %d values differ" % (name, rows, c, nd)
        # (task states keep many contacts: below the default capacity few envs get through 3 steps without dropping one)
        assert len(ok) >= (MIN_COMPARED if c >= min(DEFAULT_MAXCON, top) else 1), lines[-1]
    REPORT["%s[%s] product" % (name, rows)] = "capacities %s, %d launch shapes; 0 differing values" % (caps, len(shapes))
    print("\n%s[%s] product kernel:\n  %s" % (name, rows, "\n  ".join(lines)))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
def test_hold_task_slots_do_not_change_physics(gpu_models, rows):
    """The hold task batch (eight persistent env_prm slots shift every offset behind them) against the physics-only batch of the same
    model, with env_prm holding the model's own object size: one forward pass with taps and 5 substeps, bit for bit."""
    import torch
    from myosuite_b200 import vec_env
    z = gpu_models["myohand_hold"]; m = z["m"]
    st = state_pool("myohand_hold", z)
    n = len(st["qpos"])
    for c in (4, DEFAULT_MAXCON):
        res = []
        for hold in (False, True):
            env = (vec_env.MyoVecEnv(TASK_OF["myohand_hold"], n, taps=True, auto_reset=False, row_storage=rows, maxcon=c) if hold
                   else vec_env.MyoVecEnv.from_model("myohand_hold", n, taps=True, row_storage=rows, maxcon=c))
            if hold:
                g = int(env.cfg.task_i[1])
                env.t["env_prm"][:, 3:6] = torch.as_tensor(env.prog["PG_d"][g][12:15], device=env.device)
            r = {}
            for nsub in (0, 5):
                env.set_state(qpos=st["qpos"], qvel=st["qvel"], act=st["act"])
                env.t["qacc_warmstart"].copy_(torch.as_tensor(st["qacc_warmstart"], device=env.device))
                env.forward_debug(st["ctrl"], nsub); torch.cuda.synchronize()
                r.update({"%s/%d" % (k, nsub): v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_") and k != "tap_phase_cycles" or k in STATE})
            res.append((r, env.dims.smem_bytes_per_env))
        (a, sa), (b, sb) = res
        assert sb > sa
        nd = sum(ndiff(a[k], b[k]) for k in a)
        assert nd == 0, (c, [k for k in a if ndiff(a[k], b[k])])
        REPORT["hold slots[%s] maxcon %d" % (rows, c)] = "%d envs, slice %d -> %d bytes; 0 differing values" % (n, sa, sb)
        print("\nhold task slots [%s] maxcon %d: %d envs, slice %d -> %d bytes, 0 differing values" % (rows, c, n, sa, sb))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("pair", [("WRAP", "WRAPX"), ("SWEEP_16", "SWEEP_16X")])
def test_far_pairs_do_not_change_physics(gpu_models, pair, rows):
    """A hinge-tree zoo model against the same model plus world geoms and pairs that never touch (more pairs, collision geoms and
    ellipsoid candidates, a larger capacity): one forward pass with taps and 3 substeps, bit for bit; the extra pairs make no contact."""
    base, ext = (gpu_models[p] for p in pair)
    mb, mx = base["m"], ext["m"]
    assert mx.npair > mb.npair and mx.ngeom > mb.ngeom
    st = state_pool(pair[0], base)
    nb = len(st["qpos"])
    for nsub in (0, 3):
        a = run_forward(mb, rows, DEFAULT_MAXCON, st, nsub)
        b = run_forward(mx, rows, DEFAULT_MAXCON, st, nsub)
        assert (b["tap_ncon"][:, 0] == a["tap_ncon"][:, 0]).all() and (b["tap_ncon"][:, 3] == 0).all()
        k = a["maxcon"]           # (0 without pairs: nothing written)
        assert np.array_equal(b["tap_contact_pair"][:, :k], a["tap_contact_pair"][:, :k]) and (b["tap_contact_pair"][:, k:] == -1).all()
        keys = (TAPS + ("qacc_warmstart",)) if nsub == 0 else STATE
        nd = sum(ndiff(a[k_], b[k_]) for k_ in keys)
        assert nd == 0, (pair, rows, nsub, [k_ for k_ in keys if ndiff(a[k_], b[k_])])
    REPORT["far pairs %s[%s]" % (pair[1], rows)] = "npair %d -> %d, maxcon %d -> %d; %d envs, 0 differing values" % (mb.npair, mx.npair, a["maxcon"], b["maxcon"], nb)
