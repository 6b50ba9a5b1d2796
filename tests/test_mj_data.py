"""The mjData readout (myo_batch_data, MyoVecEnv.data, MyoEnv.mj_data) against the CPU oracle's mj_forward.

CPU: the myo_data_buffers field order against abi.py, the export, the host maps the readout relies on (program pair -> model geoms,
parents before children, the per-task site sources) for every shipped and zoo model, and the named views of MyoEnv.mj_data on stub data.

GPU, on both row storages: every registered base task at its benchmarked launch shape after a reset and random-action steps, envs
checked against the oracle set to their rows (warm start, time, env_prm); the contact and actuation zoo models through
MyoVecEnv.from_model; the sites the tasks move per episode; the quantities the observation also holds; and that a readout changes
nothing: bound state, I/O rows and later steps stay bit-identical."""
import os
import re
import ctypes

import numpy as np
import pytest

from parity_helpers import _in_regime, relerr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = ["p48", "f64"]
POSE_ATOL = 1e-12          # xpos, xquat, xmat, site_xpos (absolute)
LEN_REL = 5e-12            # actuator_length, relative to the env's largest entry (the legs' wrapped paths measure 2.0e-12 on an H100)
FRC_REL = 1e-10            # actuator_velocity, actuator_force, qfrc_actuator
QACC_MID = 1e-6            # the qacc tap's mid-episode bound (test_gpu_parity.py), held by at least QACC_SHARE of the checked envs ...
QACC_MAX = 1e-5            # ... and every env within the north-star bound (checking every env of 4096 reaches the tail: 1.9e-6 measured)
QACC_SHARE = 0.99
DIST_ATOL = 1e-12          # analytic colliders; the iterative (ellipsoid) ones are held to test_gpu_parity.py's 1e-7 relative / 1e-11
POSFRAME_ATOL = 1e-10      # contact pos / frame of the analytic colliders
ITER_TOL = 1e-7            # pos / frame of the iterative colliders (their witness points come out of a Newton iteration)
WARM = 6
SEED = 11
REPORT = {}

# base task -> (env id, n_env): the launch shapes bench.py and test_product_parity.py run
CASES = {
    "elbow": ("myoElbowPose1D6MRandom-v0", 4096),
    "hand_pose": ("myoHandPoseRandom-v0", 4096),
    "reach": ("myoHandReachRandom-v0", 4096),
    "hold": ("myoHandObjHoldRandom-v0", 2048),
    "walk_fatigue": ("myoFatiLegWalk-v0", 2048),
    "stand": ("myoLegStandRandom-v0", 2048),
    "torso": ("myoTorsoPoseFixed-v0", 661),
}
PLANE, ELLIPSOID = 0, 4


# ----------------------------------------------------------------------------- CPU
def _header_struct(name):
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    body = src[:src.index("} %s;" % name)]
    body = body[body.rindex("typedef struct {") + len("typedef struct {"):]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"\*\s*(\w+)\s*;", body), body.count(";")


def test_data_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_data_buffers")
    assert len(fields) == decls                                     # every member is a pointer
    assert abi.DATA_FIELDS == fields
    assert [n for n, _ in abi.MyoDataBuffers._fields_] == fields and ctypes.sizeof(abi.MyoDataBuffers) == 8 * len(fields)
    assert set(abi.DATA_SHAPES) == set(fields) - {"site_source"}
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert src.index("} myo_buffers;") < src.index("} myo_data_buffers;")      # declared after myo_buffers, which is unchanged
    assert _header_struct("myo_buffers")[0] == abi.BUFFER_FIELDS


def _header_region_list(macro):
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    body = re.search(r"#define %s\(X\)((?:.*\\\n)*.*)" % macro, src).group(1)
    return tuple(re.findall(r"X\((\w+)\)", body))


def test_layout_regions_match_header():
    """The names and slot order of myo_model_layout's regions: the X-macro lists the library is built from against abi.LAYOUT_*."""
    from myosuite_b200 import abi
    assert _header_region_list("MYO_LAYOUT_PERSISTENT") == abi.LAYOUT_PERSISTENT
    assert _header_region_list("MYO_LAYOUT_SCRATCH") == abi.LAYOUT_SCRATCH
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    assert int(re.search(r"#define MYO_LAYOUT_N (\d+)", src).group(1)) == abi.LAYOUT_N == 93


def test_data_export():
    from myosuite_b200 import abi, build
    assert "myo_batch_data" in abi.EXPORTS
    L = ctypes.CDLL(build.build())
    assert hasattr(L, "myo_batch_data") and hasattr(abi.lib("f64rows"), "myo_batch_data")
    assert abi.lib().myo_version() == 2


def _zoo_models(tmp):
    import test_actuation_zoo as AZ
    import test_contact_zoo as CZ
    (tmp / "c").mkdir(); (tmp / "a").mkdir()
    out = {"contact/" + k: v[0] for k, v in CZ.build_zoo(tmp / "c").items()}
    out.update({"actuation/" + k: v["m"] for k, v in AZ.build_zoo(tmp / "a", names=["WRAP", "MUSCLE", "LIM_CROSS", "SWEEP_40"]).items()})
    return out


def _check_maps(m, prog, info):
    """The facts myo_batch_data's host setup reads from the blob: bodies after their parents (one level sweep), the program pair's two geoms
    are the model pair's geom1 / geom2 in that order, and the contact rank is the model pair index."""
    assert all(m.body_parentid[b] < b for b in range(1, m.nbody))
    gid = info["geom_model_ids"]
    for row in prog["PPAIR"]:
        p = int(row[7])
        assert (gid[int(row[0])], gid[int(row[1])]) == (int(m.pair_geom1[p]), int(m.pair_geom2[p]))
    assert list(prog["PPAIR"][:, 7]) == info["pair_model_index"]


def test_host_maps_every_model(tmp_path):
    from myosuite_b200 import assets, program
    models = {k: assets.load(k) for k in assets.MODEL_XML}
    models.update(_zoo_models(tmp_path))
    for name, m in models.items():
        prog, info = program.build_program(m)
        _check_maps(m, prog, info)
    print("\nhost maps checked on %d models: %s" % (len(models), sorted(models)))


def test_site_sources_every_task():
    """Per-task site sources: every registered base task (and the pose variants with visualised targets) moves exactly the sites the
    reference moves, each of them on the world body, with in-range indices."""
    from myosuite_b200 import abi, assets, program, tasks, vec_env
    seen = {}
    for eid in vec_env.registered_ids():
        steps, kw, entry = vec_env.env_spec(eid)
        kind = tasks.task_of(entry)
        if kind is None:
            continue
        m = assets.load(vec_env._MODEL_OF_XML[kw["model_path"]])
        c = tasks.configure(entry, m, program.build_program(m)[1], kw, steps)
        src = tasks.site_sources(c.task, m, kw, c.tip_names)
        moved = [] if src is None else list(np.nonzero(src[:, 0])[0])
        for s in moved:
            k, ix = src[s]
            assert m.site_bodyid[s] == 0, (eid, m.id2name("site", s))
            if k == abi.SITE_TARGET:
                assert c.task in ("reach", "stand") and 0 <= ix and ix + 3 <= m.nq
                assert m.id2name("site", s) == c.tip_names[ix // 3] + "_target"
            elif k == abi.SITE_ENV_PRM:
                assert c.task == "hold" and ix == 0 and m.id2name("site", s) == "goal"
            else:
                assert k == abi.SITE_AT_TARGET_POSE and c.task == "pose" and m.id2name("site", s) == m.id2name("site", ix) + "_target"
        if c.task in ("reach", "stand"):
            assert len(moved) == len(c.tip_names) > 0
        if c.task == "hold":
            assert len(moved) == 1
        if c.task == "pose":
            assert len(moved) == len(kw.get("viz_site_targets") or ())
        seen[c.task] = seen.get(c.task, 0) + len(moved)
    print("\nmoved sites per task over the registry: %s" % seen)
    assert seen.get("pose", 0) > 0 and seen.get("reach", 0) > 0 and seen.get("stand", 0) > 0 and seen.get("hold", 0) > 0


class _StubVec:
    """What _DataView reads of a MyoVecEnv: CPU tensors in place of the device rows, counting the readouts."""

    def __init__(self, m):
        import torch
        from myosuite_b200 import abi, vec_env
        self.torch, self.mj_model, self.state_version, self.calls = torch, m, 0, 0
        self.DATA_FIELDS = vec_env.MyoVecEnv.DATA_FIELDS
        rng = np.random.default_rng(0)
        self.t = {"qpos": torch.as_tensor(rng.normal(size=(1, m.nq))), "qvel": torch.as_tensor(rng.normal(size=(1, m.nv))),
                  "act": torch.as_tensor(rng.uniform(size=(1, max(m.na, 1)))), "time": torch.tensor([0.25], dtype=torch.float64)}
        size = dict(nbody=m.nbody, nsite=m.nsite, nu=m.nu, nv=m.nv, maxcon=4)
        self.out = {}
        for f in self.DATA_FIELDS:
            _, dt, shape = abi.DATA_SHAPES[f]
            shape = (1,) + tuple(size[x] if isinstance(x, str) else x for x in shape)
            self.out[f] = (torch.as_tensor(rng.normal(size=shape)) if dt == "f64" else torch.as_tensor(rng.integers(0, 5, size=shape), dtype=torch.int32))
        self.out["ncon"][:] = 2

    def data(self, *fields):
        self.calls += 1
        return self.out


def test_named_views_on_stub_data():
    from myosuite_b200 import assets, mjcf, vec_env
    m = assets.load("myolegs")
    v = _StubVec(m)
    d = vec_env._DataView(v)
    o = {k: x[0].numpy() for k, x in v.out.items()}
    b = m.name2id("body", "pelvis")
    assert np.array_equal(d.body("pelvis").xpos, o["xpos"][b]) and np.array_equal(d.body(b).xquat, o["xquat"][b])
    assert np.array_equal(d.body("pelvis").xmat, o["xmat"][b])
    s = 3
    assert np.array_equal(d.site(m.id2name("site", s)).xpos, o["site_xpos"][s]) and np.array_equal(d.site_xpos[s], o["site_xpos"][s])
    a = 5
    act = d.actuator(m.id2name("actuator", a))
    assert act.length[0] == o["actuator_length"][a] and act.velocity[0] == o["actuator_velocity"][a] and act.force[0] == o["actuator_force"][a]
    root = [j for j in range(m.njnt) if m.jnt_type[j] == mjcf.JNT_FREE][0]
    hinge = [j for j in range(m.njnt) if m.jnt_type[j] == mjcf.JNT_HINGE][0]
    jr, jh = d.joint(m.id2name("joint", root)), d.joint(m.id2name("joint", hinge))
    qa, da = m.jnt_qposadr[root], m.jnt_dofadr[root]
    assert np.array_equal(jr.qpos, v.t["qpos"][0, qa:qa + 7].numpy()) and np.array_equal(jr.qvel, v.t["qvel"][0, da:da + 6].numpy())
    assert np.array_equal(jr.qacc, o["qacc"][da:da + 6]) and jh.qpos.shape == (1,) and jh.qacc[0] == o["qacc"][m.jnt_dofadr[hinge]]
    assert d.ncon == 2 and d.time == 0.25
    c = d.contact
    assert np.array_equal(c.geom1, o["contact_geom"][:2, 0]) and np.array_equal(c.geom2, o["contact_geom"][:2, 1])
    assert np.array_equal(c.dist, o["contact_dist"][:2]) and c.pos.shape == (2, 3) and c.frame.shape == (2, 9)
    assert np.array_equal(d.act, v.t["act"][0, :m.na].numpy()) and np.array_equal(d.actuator_length, o["actuator_length"])
    assert v.calls == 1                       # one readout for all of the above
    v.state_version += 1
    d.qpos
    assert v.calls == 2
    x = d.xpos; x[:] = 0                      # copies: the cached values stay
    assert not np.all(d.xpos == 0)
    with pytest.raises(AttributeError):
        d.not_a_field


# ----------------------------------------------------------------------------- GPU helpers
def _oracle_expect(o, m, site_src, target, prm, o_target):
    """Expected site_xpos of one env: the oracle's poses, with the sites the task moves placed from their per-env sources."""
    xpos, xmat = o.f("xpos").reshape(-1, 3), o.f("xmat").reshape(-1, 3, 3)
    out = o.f("site_xpos").reshape(-1, 3).copy()
    if site_src is None:
        return out
    for s in np.nonzero(site_src[:, 0])[0]:
        k, ix = site_src[s]
        if k == 1:
            loc = target[ix:ix + 3]
        elif k == 2:
            loc = prm[ix:ix + 3]
        else:
            loc = o_target[ix]
        b = m.site_bodyid[s]
        out[s] = xpos[b] + xmat[b] @ loc
    return out


def _contact_force_ref(o, m):
    """mj_contactForce of the oracle's contacts, decoded in numpy from efc_force (mju_decodePyramid: the normal force is the sum of the
    pyramid edges, tangent i is (edge 2i - edge 2i+1) mu_i).  The contact rows close the row list, in contact order: none for a contact
    beyond margin - gap, one for condim 1, four pyramid edges for condim 3."""
    pair, dist, f = o.i("con_pair"), o.f("con_dist"), o.f("efc_force")
    active = dist < m.pair_margin[pair] - m.pair_gap[pair]
    out, r = np.zeros((len(pair), 6)), o.nefc - int(np.sum(np.where(active, np.where(m.pair_dim[pair] == 1, 1, 4), 0)))
    for c, p in enumerate(pair):
        if not active[c]:
            continue
        if m.pair_dim[p] == 1:
            out[c, 0] = f[r]; r += 1
        else:
            e = f[r:r + 4]; r += 4
            out[c, 0] = e.sum(); out[c, 1] = (e[0] - e[1]) * m.pair_friction[p, 0]; out[c, 2] = (e[2] - e[3]) * m.pair_friction[p, 1]
    assert r == o.nefc
    return out


def compare_env(env, D, S, e, o, worst, qacc_tol=QACC_MAX, o_target=None, regime=_in_regime):
    """Every readout field of env e against the oracle set to its rows; returns False (skipped) outside the contact regime."""
    m = env.mj_model
    o.reset()
    o.set(qpos=S["qpos"][e], qvel=S["qvel"][e], act=S["act"][e, :m.na], qacc_warmstart=S["qacc_warmstart"][e], ctrl=np.zeros(m.nu))
    o.f("time")[:] = S["time"][e]
    o.forward()
    if not regime(o, m):
        return False
    msg = "%s env %d" % (env.env_id or "model", e)
    for k, ref in (("xpos", o.f("xpos")), ("xquat", o.f("xquat")), ("xmat", o.f("xmat"))):
        g = D[k][e].reshape(-1)
        worst[k] = max(worst.get(k, 0.0), float(np.abs(g - ref).max()))
        np.testing.assert_allclose(g, ref, rtol=0, atol=POSE_ATOL, err_msg=msg + " " + k)
    src = None if env._site_source is None else env._site_source.cpu().numpy()
    prm = S["env_prm"][e] if "env_prm" in S else None
    exp = _oracle_expect(o, m, src, S["target"][e], prm, o_target)
    worst["site_xpos"] = max(worst.get("site_xpos", 0.0), float(np.abs(D["site_xpos"][e] - exp).max()) if m.nsite else 0.0)
    np.testing.assert_allclose(D["site_xpos"][e], exp, rtol=0, atol=POSE_ATOL, err_msg=msg + " site_xpos")
    for k, tol in (("actuator_length", LEN_REL), ("actuator_velocity", FRC_REL), ("actuator_force", FRC_REL), ("qfrc_actuator", FRC_REL)):
        ref = o.f(k); g = D[k][e]
        err = float(np.abs(g - ref).max() / max(np.abs(ref).max(), 1e-300)) if ref.size else 0.0
        worst[k] = max(worst.get(k, 0.0), err)
        assert err <= tol, "%s %s: %.2e" % (msg, k, err)
    r = relerr(D["qacc"][e], o.f("qacc")); worst["qacc"] = max(worst.get("qacc", 0.0), r)
    worst["qacc_over_mid"] = worst.get("qacc_over_mid", 0) + int(r >= QACC_MID)
    assert r < qacc_tol, "%s qacc %.2e" % (msg, r)
    nc = o.ncon
    assert D["ncon"][e] == nc, msg
    assert [tuple(x) for x in D["contact_geom"][e, :nc]] == list(zip(o.i("con_geom1"), o.i("con_geom2"))), msg
    assert np.all(D["contact_geom"][e, nc:] == -1) and np.all(D["contact_dist"][e, nc:] == 0) and np.all(D["contact_force"][e, nc:] == 0), msg
    it = np.array([m.geom_type[g2] == ELLIPSOID and m.geom_type[g1] != PLANE for g1, g2 in zip(o.i("con_geom1"), o.i("con_geom2"))], dtype=bool)
    gd, od = D["contact_dist"][e, :nc], o.f("con_dist")
    gp, op = D["contact_pos"][e, :nc], o.f("con_pos").reshape(-1, 3)
    gf, of = D["contact_frame"][e, :nc], o.f("con_frame").reshape(-1, 9)
    if np.any(~it):
        worst["dist"] = max(worst.get("dist", 0.0), float(np.abs(gd - od)[~it].max()))
        worst["pos_frame"] = max(worst.get("pos_frame", 0.0), float(max(np.abs(gp - op)[~it].max(), np.abs(gf - of)[~it].max())))
        np.testing.assert_allclose(gd[~it], od[~it], rtol=0, atol=DIST_ATOL, err_msg=msg + " dist")
        np.testing.assert_allclose(gp[~it], op[~it], rtol=0, atol=POSFRAME_ATOL, err_msg=msg + " pos")
        np.testing.assert_allclose(gf[~it], of[~it], rtol=0, atol=POSFRAME_ATOL, err_msg=msg + " frame")
    if np.any(it):
        worst["dist_iter"] = max(worst.get("dist_iter", 0.0), float(np.abs(gd - od)[it].max()))
        np.testing.assert_allclose(gd[it], od[it], rtol=1e-7, atol=1e-11, err_msg=msg + " dist (iterative)")
        np.testing.assert_allclose(gp[it], op[it], rtol=0, atol=ITER_TOL, err_msg=msg + " pos (iterative)")
        np.testing.assert_allclose(gf[it], of[it], rtol=0, atol=ITER_TOL, err_msg=msg + " frame (iterative)")
    if nc:
        ref = _contact_force_ref(o, m)
        scale = max(np.abs(ref[:, 0]).max(), 1e-300)
        err = float(np.abs(D["contact_force"][e, :nc] - ref).max() / scale) if scale > 1e-300 else float(np.abs(D["contact_force"][e, :nc]).max())
        worst["contact_force"] = max(worst.get("contact_force", 0.0), err)
        assert err < qacc_tol, "%s contact_force %.2e" % (msg, err)
        worst["contacts"] = worst.get("contacts", 0) + nc
    return True


def _host(D):
    return {k: v.cpu().numpy().copy() for k, v in D.items()}


def _oracle_targets(env, o_t, target):
    """World positions of every site at the kinematics of the target pose (for the pose task's markers)."""
    o_t.reset(); o_t.set(qpos=target); o_t.forward()
    return o_t.f("site_xpos").reshape(-1, 3).copy()


# ----------------------------------------------------------------------------- GPU: registered tasks against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_data_vs_oracle(case, rows):
    """After a reset and WARM random-action steps (auto-reset on): every env (every 4th and the 64 most contact-heavy ones on the f64
    row storage, whose launch shape differs only in the step kernels) against the oracle's mj_forward at its rows."""
    import torch
    from test_product_parity import Oracles
    from myosuite_b200 import vec_env
    eid, n = CASES[case]
    env = vec_env.MyoVecEnv(eid, n, seed=SEED, row_storage=rows)
    m = env.mj_model
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(WARM):
        env.step((torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device))
    D = _host(env.data())
    torch.cuda.synchronize()
    S = env.get_env_state()
    if rows == "f64":
        top = np.argsort(D["ncon"], kind="stable")[::-1][:64]
        envs = sorted(set(range(0, n, 4)) | set(int(e) for e in top))
    else:
        envs = range(n)
    oracles, o_t = Oracles(env), None
    src = None if env._site_source is None else env._site_source.cpu().numpy()
    if src is not None and np.any(src[:, 0] == 3):
        from oracle.oracle_py import Oracle
        o_t = Oracle(env.I, env.D)
    worst, checked, skipped = {}, 0, 0
    for e in envs:
        o = oracles.get(S["env_prm"][e] if "env_prm" in S else None)
        ot = _oracle_targets(env, o_t, S["target"][e]) if o_t is not None else None
        if compare_env(env, D, S, e, o, worst, o_target=ot):
            checked += 1
        else:
            skipped += 1
    REPORT["%s[%s]" % (case, rows)] = "checked %d, skipped (contact regime) %d; worst %s" % (
        checked, skipped, ", ".join("%s %.1e" % (k, v) if isinstance(v, float) else "%s %d" % (k, v) for k, v in sorted(worst.items())))
    print("\n%s[%s] %s" % (case, rows, REPORT["%s[%s]" % (case, rows)]))
    assert skipped <= 0.25 * len(envs) and checked > 0
    assert worst.get("qacc_over_mid", 0) <= (1 - QACC_SHARE) * checked


# ----------------------------------------------------------------------------- GPU: synthetic models
@pytest.fixture(scope="module")
def zoos(tmp_path_factory):
    import test_actuation_zoo as AZ
    import test_contact_zoo as CZ
    tmp = tmp_path_factory.mktemp("data_zoo")
    (tmp / "c").mkdir(); (tmp / "a").mkdir()
    return CZ.build_zoo(tmp / "c"), AZ.build_zoo(tmp / "a")


ZOO_CASES = ["contact/" + k for k in ("CAP_CAP", "SPH_SPH", "SPH_CAP", "PLANE_SPH", "PLANE_CAP", "PLANE_ELL", "CAP_ELL", "ELL_ELL", "COMBO")] + \
            ["actuation/" + k for k in ("WRAP", "MUSCLE", "LIM_TREE", "LIM_CROSS", "SWEEP_40")]


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("name", ZOO_CASES)
def test_data_zoo(zoos, name, rows):
    """Every collider class, condim 1 and 3, every wrap class, muscles, limits and equalities through MyoVecEnv.from_model."""
    import torch
    import test_contact_zoo as CZ
    from myosuite_b200 import vec_env
    kind, key = name.split("/")
    if kind == "contact":
        m = zoos[0][key][0]
        cfgs = CZ._configs({key: zoos[0][key]}, key) if key != "COMBO" else CZ._configs(zoos[0], key)
        labels = [lb for lb, _ in cfgs]; qpos = np.stack([q for _, q in cfgs])
        qvel, act, _ = CZ._state(m, qpos, 5, [lb != "generic" for lb in labels])
        qacc_tol = CZ.FWD_QACC
    else:
        z = zoos[1][key]; m, qpos, qvel, act = z["m"], z["qpos"], z["qvel"], z["act"]
        qacc_tol = 1e-7
    n = len(qpos)
    env = vec_env.MyoVecEnv(None, n, model=m, row_storage=rows)
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    D = _host(env.data()); torch.cuda.synchronize()
    S = env.get_env_state()
    from oracle.oracle_py import Oracle
    from myosuite_b200 import blob
    o = Oracle(*blob.pack(m))
    worst, checked = {}, 0
    for e in range(n):
        checked += bool(compare_env(env, D, S, e, o, worst, qacc_tol=qacc_tol, regime=CZ.regime_ok))
    REPORT["zoo %s[%s]" % (name, rows)] = "checked %d of %d; worst %s" % (checked, n, ", ".join(
        "%s %.1e" % (k, v) if isinstance(v, float) else "%s %d" % (k, v) for k, v in sorted(worst.items())))
    print("\n" + REPORT["zoo %s[%s]" % (name, rows)])
    assert checked >= 0.75 * n


# ----------------------------------------------------------------------------- GPU: per-episode sites and the observation
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["reach", "stand", "hold", "hand_pose"])
def test_per_episode_sites(case):
    import torch
    from oracle.oracle_py import Oracle
    from myosuite_b200 import vec_env
    eid, n = CASES[case]
    n = 256
    env = vec_env.MyoVecEnv(eid, n, seed=SEED)
    m = env.mj_model
    env.reset(seed=SEED)
    env.step(torch.zeros(n, m.nu, device=env.device))
    D = _host(env.data("site_xpos")); S = env.get_env_state()
    src = env._site_source.cpu().numpy()
    moved = np.nonzero(src[:, 0])[0]
    assert len(moved) > 0
    o = Oracle(env.I, env.D)
    for s in moved:
        k, ix = src[s]
        for e in range(n):
            if k == 1:
                assert np.array_equal(D["site_xpos"][e, s], S["target"][e, ix:ix + 3])
            elif k == 2:
                assert np.array_equal(D["site_xpos"][e, s], S["env_prm"][e, ix:ix + 3])
            elif e < 64:
                o.reset(); o.set(qpos=S["target"][e]); o.forward()
                np.testing.assert_allclose(D["site_xpos"][e, s], o.f("site_xpos").reshape(-1, 3)[ix], rtol=0, atol=POSE_ATOL)
    assert len(np.unique(D["site_xpos"][:, moved[0]], axis=0)) > n // 2        # per env, not the model's site_pos


def _f32_close(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.all(np.abs(a.astype(np.float64) - b.astype(np.float64)) <= np.spacing(np.maximum(np.abs(a), np.abs(b))))


@pytest.mark.gpu
def test_data_against_obs():
    """Where the observation holds the same quantity: reach tip positions, the walk torso's xquat and the walk muscle length, velocity and
    force (after the obs's clip and scale), equal after the f32 cast (within one f32 ulp of rounding-boundary cases)."""
    import torch
    from myosuite_b200 import tasks, vec_env
    n = 512
    env = vec_env.MyoVecEnv("myoHandReachRandom-v0", n, seed=SEED)
    m = env.mj_model
    env.reset(seed=SEED)
    for _ in range(3):
        env.step(torch.rand(n, m.nu, device=env.device) * 2 - 1)
    D = _host(env.data("site_xpos")); obs = env.t["obs_full"].cpu().numpy()
    ntip = len(env.tip_names); base = m.nq + m.nv
    tips = np.stack([D["site_xpos"][:, m.name2id("site", t)] for t in env.tip_names], 1).reshape(n, -1)
    assert _f32_close(obs[:, base:base + 3 * ntip], tips)
    exact = np.mean(obs[:, base:base + 3 * ntip] == tips.astype(np.float32))

    env = vec_env.MyoVecEnv("myoFatiLegWalk-v0", n, seed=SEED)
    m = env.mj_model
    env.reset(seed=SEED)
    for _ in range(3):
        env.step(torch.rand(n, m.nu, device=env.device) * 2 - 1)
    D = _host(env.data("xquat", "actuator_length", "actuator_velocity", "actuator_force")); obs = env.t["obs_full"].cpu().numpy()
    lay, o = dict(tasks.obs_layout("walk", m.nq, m.nv, m.na)), {}
    off = 0
    for k, w in tasks.obs_layout("walk", m.nq, m.nv, m.na):
        o[k] = obs[:, off:off + w]; off += w
    assert _f32_close(o["torso_angle"], D["xquat"][:, m.name2id("body", "torso")])
    assert _f32_close(o["muscle_length"], D["actuator_length"])
    assert _f32_close(o["muscle_velocity"], np.clip(D["actuator_velocity"], -100, 100))
    assert _f32_close(o["muscle_force"], np.clip(D["actuator_force"] / 1000.0, -100, 100))
    print("\nreach tips equal to obs bit for bit in %.4f of the entries (the rest within one f32 ulp)" % exact)


# ----------------------------------------------------------------------------- GPU: no side effects
BOUND = ("qpos", "qvel", "act", "qacc_warmstart", "time", "step_count", "episode_count", "ep_return", "last_return", "obs", "reward", "done",
         "truncated", "final_obs", "overflow", "fatigue", "target", "env_prm")


def _same(x, y):
    """bit-equal, NaN where NaN"""
    if x.is_floating_point():
        return torch_equal_bits(x, y)
    return bool((x == y).all())


def torch_equal_bits(x, y):
    import torch
    return torch.equal(x.contiguous().view(torch.int64 if x.element_size() == 8 else torch.int32), y.contiguous().view(torch.int64 if y.element_size() == 8 else torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("eid,n", [("myoHandPoseRandom-v0", 999), ("myoFatiLegWalk-v0", 333), ("myoHandObjHoldRandom-v0", 517)])
def test_no_side_effects(eid, n):
    """A readout leaves every bound tensor bit-identical; twin batches with and without a readout between their 50 steps (auto-resets
    included) stay bit-identical; n_env is not a multiple of any launch's grid x warps."""
    import torch
    from myosuite_b200 import vec_env
    a_env, b_env = (vec_env.MyoVecEnv(eid, n, seed=SEED) for _ in range(2))
    m = a_env.mj_model
    for env in (a_env, b_env):
        env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    ends = 0
    for step in range(50):
        act = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(a_env.device)
        before = {k: a_env.t[k].clone() for k in BOUND if k in a_env.t}
        a_env.data()
        torch.cuda.synchronize()
        for k, v in before.items():
            assert _same(v, a_env.t[k]), (step, k)
        a_env.step(act); b_env.step(act.clone())
        torch.cuda.synchronize()
        ends += int((a_env.t["done"] | a_env.t["truncated"]).sum())
        for k in BOUND:
            if k in a_env.t:
                assert _same(a_env.t[k], b_env.t[k]), (step, k)
    print("\n%s n %d: 50 twin steps bit-identical, %d episode ends" % (eid, n, ends))
    assert ends > 0 or eid.startswith("myoHandPose")


@pytest.mark.gpu
def test_unrequested_fields_keep_sentinel():
    import torch
    from myosuite_b200 import abi, vec_env
    env = vec_env.MyoVecEnv("myoHandPoseRandom-v0", 100, seed=SEED)
    env.reset(seed=SEED)
    full = env.data()                                        # every buffer allocated and written once
    torch.cuda.synchronize()
    sent = {k: torch.full_like(v, float("nan")) if v.dtype == torch.float64 else torch.full_like(v, -7) for k, v in full.items()}
    for ask in (("xpos",), ("actuator_force",), ("qacc", "contact_geom")):
        for v in sent.values():
            v.fill_(float("nan")) if v.dtype == torch.float64 else v.fill_(-7)
        n0 = env.batch.launches
        env.batch.data(stream=env._stream(), **{k: sent[k] for k in ask})
        torch.cuda.synchronize()
        assert env.batch.launches == n0 + 1
        for k, v in sent.items():
            if k in ask:
                assert torch.equal(v, full[k]), k           # the same state gives the same values, bit for bit
            else:
                assert (v.isnan().all() if v.dtype == torch.float64 else (v == -7).all()), (ask, k)
    n0 = env.batch.launches
    env.batch.data(stream=env._stream())                      # nothing requested: no launch
    assert env.batch.launches == n0
    assert set(full) == set(abi.DATA_SHAPES)


# ----------------------------------------------------------------------------- GPU: MyoEnv.mj_data
@pytest.mark.gpu
def test_myoenv_mj_data():
    from myosuite_b200 import vec_env
    env = vec_env.MyoEnv("myoLegStandRandom-v0", seed=3)
    m = env.mj_model
    d = env.unwrapped.mj_data
    L = env.vec.batch
    env.reset()
    n0 = L.launches
    sid = m.name2id("site", env.vec.tip_names[0])
    tip, pel, al = d.site_xpos[sid], d.body("pelvis").xpos, d.actuator_length
    assert L.launches == n0 + 1                               # one readout for the state
    assert tip.shape == (3,) and pel.shape == (3,) and al.shape == (m.nu,) and np.isfinite(al).all()
    d.qacc, d.contact, d.joint(m.id2name("joint", 0)).qpos
    assert L.launches == n0 + 1
    env.step(env.action_space.sample())
    n1 = L.launches
    assert n1 > n0 + 1                                        # the step's own launches
    d.body("pelvis").xquat, d.site_xpos
    assert L.launches == n1 + 1
    # the stand task's tip position is in its observation (tip_pos after qpos and qvel)
    base = m.nq + m.nv
    np.testing.assert_allclose(env._last["obs_full"][base:base + 3], d.site_xpos[sid], rtol=0, atol=1e-6)
    env.forward(); d.xpos
    assert L.launches == n1 + 3


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nmjData readout vs oracle:")
        for k in sorted(REPORT):
            print("  %-32s %s" % (k, REPORT[k]))
