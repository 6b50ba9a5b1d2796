"""Every registered muscle-condition variant (myoSarc* / myoFati* / myoReaf*) against the reference's action path and the oracle.

The conditions are wired per id: sarcopenia halves gainprm[:, 2] in a copy of the model on the host (vec_env.condition_model), fatigue
runs the 3CC-r compartments in the kernel's action prologue with the model's own time constants, and reafferentation redirects the
EIP action to EPL and zeroes EIP in that prologue, with the ids from tasks.configure.

CPU: env_oracle's action path against tests/golden/variants.npz (the reference's own BaseV0.initializeConditions / BaseV0.step), the
packed blob of every Sarc id against its base id's, every shipped actuator a muscle (the kernel's remap has no muscle mask), and the
reafferentation ids of every Reaf id.
GPU: every variant id through the product kernel at a multi-round launch shape, replayed on the oracle (parity_helpers.StepCheck, the
replay of test_product_parity.py), the Reaf ids also on the f64-row build; reafferentation bit for bit against a rollout of the
redirected ctrl; the single env of make(id) against the oracle and against env 0 of a batch."""
import os
import time

import numpy as np
import pytest

import parity_helpers as PH
import philox_ref as P

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "variants.npz"))
MODELS = ("myoelbow_1dof6muscles", "myohand_pose", "myohand_hold", "myolegs", "myotorso")


def _ids(cond):
    from myosuite_b200 import vec_env
    return [i for i in vec_env.registered_ids() if vec_env.env_spec(i)[1].get("muscle_condition") == cond]


def _model_of(env_id):
    from myosuite_b200 import assets, vec_env
    return assets.load(vec_env._MODEL_OF_XML[vec_env.env_spec(env_id)[1]["model_path"]])


def _base(env_id):
    from myosuite_b200 import vec_env
    return vec_env.registry()["variants"][env_id]["base"]


# ----------------------------------------------------------------------------- CPU: the reference's action path
@pytest.mark.parametrize("norm", ["norm", "raw"])
def test_reafferentation_matches_reference(norm):
    """BaseV0.step of the reafferentation condition: sigmoid (when normalize_act), then EPL = EIP and EIP = 0 (base_v0.py:83-108)."""
    from oracle import env_oracle
    epl, eip = (int(x) for x in G["reaf_ids"])
    m = _model_of("myoReafHandPoseRandom-v0")
    assert (m.name2id("actuator", "EPL"), m.name2id("actuator", "EIP")) == (epl, eip)
    A, want = G["reaf_%s_float64_action" % norm], G["reaf_%s_float64_ctrl" % norm]
    got = np.stack([env_oracle.action_to_ctrl(a, norm == "norm", reaf=(epl, eip)) for a in A])
    assert np.all(got[:, eip] == 0) and np.all(want[:, eip] == 0)
    if norm == "raw":           # no transcendental: bit for bit
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(got[:, epl], A[:, eip])
    else:                       # the same numpy sigmoid; at most one ulp apart where a vectorised exp of another width is used
        np.testing.assert_array_max_ulp(got, want, maxulp=1)
        np.testing.assert_array_max_ulp(got[:, epl], 1.0 / (1.0 + np.exp(-5.0 * (A[:, eip] - 0.5))), maxulp=1)
    # the rows that put EIP / EPL at -1, 0.5, 1: the EPL entry follows EIP, not its own action
    assert len({(a[eip], a[epl]) for a in A[:9]}) == 9 and not np.array_equal(want[:9, epl], want[:9, eip])
    # float32 actions: the reference computes in float32; the f64 remap agrees to f32 round-off, the moves stay exact
    A32, want32 = G["reaf_%s_float32_action" % norm], G["reaf_%s_float32_ctrl" % norm]
    got32 = np.stack([env_oracle.action_to_ctrl(a.astype(np.float64), norm == "norm", reaf=(epl, eip)) for a in A32])
    assert np.all(want32[:, eip] == 0)
    if norm == "raw":
        np.testing.assert_array_equal(got32, want32)
    else:
        np.testing.assert_allclose(got32, want32, rtol=0, atol=2e-7)
    # the redirect must come after the sigmoid: zeroing EIP before it would leave sigmoid(0) ~ 0.076 there
    if norm == "norm":
        pre = 1.0 / (1.0 + np.exp(-5.0 * (0.0 - 0.5)))
        assert abs(pre - 0.0759) < 1e-3 and np.all(np.abs(want[:, eip] - pre) > 0.07)


def test_action_to_ctrl_muscle_mask():
    """The optional muscle mask: the sigmoid only on masked entries (base_v0.py:84-90); an all-true mask is the default."""
    from oracle import env_oracle
    a = G["reaf_norm_float64_action"][12]
    mask = np.arange(len(a)) % 3 != 0
    got = env_oracle.action_to_ctrl(a, True, muscle=mask)
    np.testing.assert_array_equal(got[~mask], a[~mask])
    np.testing.assert_array_equal(got[mask], env_oracle.action_to_ctrl(a, True)[mask])
    np.testing.assert_array_equal(env_oracle.action_to_ctrl(a, True, muscle=np.ones(len(a), bool)), env_oracle.action_to_ctrl(a, True))
    np.testing.assert_array_equal(env_oracle.action_to_ctrl(a, False, muscle=mask), a)


@pytest.mark.parametrize("model", MODELS)
def test_every_actuator_is_a_muscle(model):
    """The kernel applies the sigmoid and fatigue to every actuator, the reference only where actuator_dyntype == mjDYN_MUSCLE (4):
    the same only while every actuator of a shipped model is a muscle."""
    from myosuite_b200 import assets
    m = assets.load(model)
    assert m.nu > 0 and m.na == m.nu and np.all(np.asarray(m.actuator_dyntype) == 4)


def test_fatigue_chain_torso_matches_reference():
    """BaseV0.step of the fatigue condition on the torso's 210 muscles with the model's own tauact / taudeact."""
    from oracle import env_oracle
    m = _model_of("myoFatiTorsoPoseFixed-v0")
    f = env_oracle.Fatigue(m.nu, dt=m.opt_timestep * 10, tauact=m.actuator_dynprm[:, 0], taudeact=m.actuator_dynprm[:, 1])
    got = np.stack([f.compute_act(env_oracle.action_to_ctrl(a))[0].copy() for a in G["fati_torso_action"]])
    want = G["fati_torso_ctrl"]
    assert want.shape == (60, 210) and np.ptp(want[-1]) > 0.05          # the compartments moved and differ between muscles
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-15)


@pytest.mark.parametrize("model", MODELS)
def test_sarcopenia_model_matches_reference(model):
    """vec_env.condition_model against the reference's initializeConditions: gainprm bit for bit (column 2 halved), biasprm untouched."""
    from myosuite_b200 import assets, vec_env
    m = assets.load(model)
    s = vec_env.condition_model(m, "sarcopenia")
    np.testing.assert_array_equal(s.actuator_gainprm, G["sarc_%s_gainprm" % model])
    np.testing.assert_array_equal(s.actuator_biasprm, G["sarc_%s_biasprm" % model])
    np.testing.assert_array_equal(s.actuator_gainprm[:, 2], 0.5 * m.actuator_gainprm[:, 2])
    np.testing.assert_array_equal(m.actuator_gainprm, assets.load(model).actuator_gainprm)            # the shipped model is not modified
    for cond in ("", "fatigue", "reafferentation"):
        assert vec_env.condition_model(m, cond) is m


@pytest.mark.parametrize("eid", _ids("sarcopenia"))
def test_sarcopenia_blob(eid):
    """The blob a Sarc batch packs equals its base id's except where gainprm[:, 2] is packed (found by packing the base model with that
    column tripled), and there it is exactly half; the integer part is equal."""
    import copy
    from myosuite_b200 import blob, program, vec_env
    m = _model_of(eid)
    _, kw, _ = vec_env.env_spec(eid); _, kw_b, _ = vec_env.env_spec(_base(eid))
    assert kw["muscle_condition"] == "sarcopenia" and kw_b.get("muscle_condition", "") == ""

    def pack(mm):
        return blob.pack(mm, program.build_program(mm)[0])
    Ib, Db = pack(vec_env.condition_model(m, kw_b.get("muscle_condition", "")))
    Is, Ds = pack(vec_env.condition_model(m, kw["muscle_condition"]))
    m3 = copy.deepcopy(m); m3.actuator_gainprm[:, 2] *= 3.0
    I3, D3 = pack(m3)
    off = np.nonzero(D3 != Db)[0]
    assert np.array_equal(Is, Ib) and np.array_equal(I3, Ib) and len(off) >= m.nu
    np.testing.assert_array_equal(np.delete(Ds, off), np.delete(Db, off))
    np.testing.assert_array_equal(Ds[off], 0.5 * Db[off])


@pytest.mark.parametrize("eid", _ids("reafferentation"))
def test_reafferentation_ids(eid):
    """cfg.reaf_dst / reaf_src of every Reaf id are the EPL / EIP actuators of its model (base_v0.py:78-79); no other id sets them."""
    from myosuite_b200 import program, tasks, vec_env
    steps, kw, entry = vec_env.env_spec(eid)
    m = _model_of(eid)
    c = tasks.configure(entry, m, program.build_program(m)[1], kw, steps)
    assert (c.cfg.reaf_dst, c.cfg.reaf_src) == (m.name2id("actuator", "EPL"), m.name2id("actuator", "EIP"))
    assert m.id2name("actuator", c.cfg.reaf_dst) == "EPL" and m.id2name("actuator", c.cfg.reaf_src) == "EIP"
    assert (c.cfg.reaf_dst, c.cfg.reaf_src) == tuple(int(x) for x in G["reaf_ids"])
    b_steps, b_kw, b_entry = vec_env.env_spec(_base(eid))
    cb = tasks.configure(b_entry, m, program.build_program(m)[1], b_kw, b_steps)
    assert cb.cfg.reaf_dst == cb.cfg.reaf_src == -1


def test_every_variant_id_has_a_case():
    from myosuite_b200 import vec_env
    ids = _ids("sarcopenia") + _ids("fatigue") + _ids("reafferentation")
    assert (len(_ids("sarcopenia")), len(_ids("fatigue")), len(_ids("reafferentation"))) == (11, 11, 6)
    assert sorted(ids) == sorted(vec_env.registry()["variants"])
    assert sorted(c[0] for c in CASES.values() if c[2] == {}) == sorted(ids)
    assert sorted(c[0] for c in CASES.values() if c[2]) == sorted(_ids("reafferentation"))
    assert all(b in BASE_SHAPE for b in map(_base, ids))


# ----------------------------------------------------------------------------- GPU: every variant id through a product kernel
# base id -> (n_env, expected launch_info subset, envs reset right before the checked step): the shapes of test_product_parity.py's
# cases on an H100 SXM (132 SMs), at least 2 rounds and 2 warps per CTA.  A variant runs its base's model (sarcopenia changes values
# only), so it gets its base's shape.
HAND_SHAPE = (4096, dict(use_w14=1, warps_per_cta=11, rounds=3, regroup=1), 0)
BASE_SHAPE = {
    "myoElbowPose1D6MRandom-v0": (4096, dict(use_w14=1, warps_per_cta=14, rounds=3, regroup=0, balanced=0), 0),
    "myoElbowPose1D6MFixed-v0": (4096, dict(use_w14=1, warps_per_cta=14, rounds=3, regroup=0, balanced=0), 0),
    "myoHandPoseRandom-v0": HAND_SHAPE, "myoHandPoseFixed-v0": HAND_SHAPE, "myoHandReachRandom-v0": HAND_SHAPE, "myoHandReachFixed-v0": HAND_SHAPE,
    "myoHandObjHoldRandom-v0": (2048, dict(use_w14=0, warps_per_cta=8, rounds=2, regroup=1), 0),
    "myoHandObjHoldFixed-v0": (2048, dict(use_w14=0, warps_per_cta=8, rounds=2, regroup=1), 0),
    "myoLegWalk-v0": (2048, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1), 0),
    "myoLegStandRandom-v0": (2048, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1), 48),
    "myoTorsoPoseFixed-v0": (661, dict(use_w14=0, warps_per_cta=3, rounds=2, regroup=1), 0),
}
# the f64-row build runs fewer warps per CTA where the rows do not fit beside them
F64_SHAPE = {"myoHandObjHoldRandom-v0": (2048, dict(use_w14=0, warps_per_cta=8, rounds=2, regroup=1), 0),
             "myoHandObjHoldFixed-v0": (2048, dict(use_w14=0, warps_per_cta=8, rounds=2, regroup=1), 0)}
_VARIANTS = sorted(__import__("json").load(open(os.path.join(os.path.dirname(HERE), "myosuite_b200", "assets", "registry.json")))["variants"].items())
# case -> (env id, n_env, env kwargs, expected launch_info subset, envs reset right before the checked step)
CASES = {eid: (eid,) + (lambda s: (s[0], {}, s[1], s[2]))(BASE_SHAPE[v["base"]]) for eid, v in _VARIANTS}
CASES.update({eid + "/f64": (eid,) + (lambda s: (s[0], {"row_storage": "f64"}, s[1], s[2]))(F64_SHAPE.get(v["base"], BASE_SHAPE[v["base"]]))
              for eid, v in _VARIANTS if v["variants"]["muscle_condition"] == "reafferentation"})
REPORT = []


@pytest.fixture(scope="module")
def report():
    t0 = time.time()
    yield REPORT
    print("\nmuscle-condition variants vs oracle (%.0f s for the module):" % (time.time() - t0))
    for line in REPORT:
        print("  " + line)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_variant_step_vs_oracle(case, report, monkeypatch):
    """The replay of test_product_parity.py on one variant id: reset, 6 warm steps, a quarter of the envs at the TimeLimit, the selected
    envs of the checked step replayed on the oracle with the id's action path (reafferentation pair, fatigue compartments)."""
    eid, n, kw, expect, n_first = CASES[case]
    for k in PH.LAUNCH_ENV:
        monkeypatch.delenv(k, raising=False)
    line, res = PH.replay_product_step(case.replace("myo", "").replace("-v0", ""), eid, n, kw, expect, n_first=n_first, report=report)
    assert res["cnt"]["reset"] >= 16 and res["cnt"]["phys"] >= 32


# ----------------------------------------------------------------------------- GPU: reafferentation without the oracle
REAF_N = 256


@pytest.mark.gpu
@pytest.mark.parametrize("eid", _ids("reafferentation"))
def test_reafferentation_equals_rollout_of_redirected_ctrl(eid, report):
    """With normalize_act off the remap has no transcendental: 3 steps of the Reaf batch with actions a are bit-identical to a rollout
    on the base batch of ctrl = a with EPL = a_EIP and EIP = 0, from the same state (qpos, qvel, act, warm start, time)."""
    import torch
    from myosuite_b200 import vec_env
    n = REAF_N
    reaf = vec_env.MyoVecEnv(eid, n, seed=PH.SEED, normalize_act=False, auto_reset=False)
    base = vec_env.MyoVecEnv(_base(eid), n, seed=PH.SEED, normalize_act=False, auto_reset=False)
    m = reaf.mj_model
    assert np.array_equal(reaf.I, base.I) and np.array_equal(reaf.D, base.D)
    epl, eip = PH.reaf_pair(reaf)
    assert (epl, eip) == (m.name2id("actuator", "EPL"), m.name2id("actuator", "EIP")) and PH.reaf_pair(base) is None
    reaf.reset(seed=PH.SEED)
    g = torch.Generator(device="cpu").manual_seed(PH.SEED)
    for _ in range(PH.WARM):
        reaf.step((torch.rand(n, m.nu, generator=g) * 2 - 1).to(reaf.device))
    S = {k: reaf.t[k].clone() for k in ("qpos", "qvel", "qacc_warmstart", "time")}
    S["act"] = reaf.t["act"][:, :m.na].contiguous().clone()
    if "env_prm" in reaf.t:                 # the hold task's per-env object sizes of the episodes the reset drew
        base.t["env_prm"].copy_(reaf.t["env_prm"])
    # actions in (0, 1), inside ctrlrange, with |a_EIP - a_EPL| > 0.2 on every env: a lost, swapped or misplaced redirect changes ctrl
    acts = torch.rand(3, n, m.nu, generator=g, dtype=torch.float32)
    acts[:, :, eip] = 0.05 + 0.3 * torch.rand(3, n, generator=g); acts[:, :, epl] = 0.65 + 0.3 * torch.rand(3, n, generator=g)
    assert bool(torch.all((acts[:, :, eip] - acts[:, :, epl]).abs() > 0.2))
    ctrl = acts.double().permute(1, 0, 2).contiguous()
    ctrl[:, :, epl] = ctrl[:, :, eip]; ctrl[:, :, eip] = 0.0
    ctrl = ctrl.to(base.device).contiguous()
    out = base.rollout(ctrl, substeps=base.frame_skip, initial_state=S, fields=base.ROLLOUT_FIELDS)
    reaf.t["overflow"].zero_()
    diff = {}
    for t in range(3):
        reaf.step(acts[t].to(reaf.device))
        for k, s in (("qpos", "qpos"), ("qvel", "qvel"), ("act", "act"), ("qacc", "qacc_warmstart"), ("time", "time")):
            ref = reaf.t[s][:, :m.na] if k == "act" else reaf.t[s]
            if not torch.equal(out[k][:, t], ref):
                diff.setdefault(k, []).append(t)
    torch.cuda.synchronize()
    assert not diff, diff
    assert torch.equal(out["overflow"] != 0, reaf.t["overflow"] != 0)
    report.append("reaf-rollout %-26s n %d: 3 steps bit-equal to a rollout of the redirected ctrl (EPL %d <- EIP %d)" % (eid, n, epl, eip))


# ----------------------------------------------------------------------------- GPU: the single env of make(id)
SINGLE_IDS = sorted(BASE_SHAPE) + ["myoReafHandPoseRandom-v0", "myoFatiTorsoPoseFixed-v0"]


def test_reach_reward_dict_of_one_env():
    """The single env's obs_dict carries time as a [1] array: the reach reward terms stay scalars (make(id) of the reach ids raised
    in get_reward_dict when the penalty term took the time's shape)."""
    from myosuite_b200 import tasks
    od = tasks.obs_dict_from_vec("reach", np.zeros(23 + 23 + 30 + 39, np.float32), np.array([1.0]), 23, 23, 39, 5)
    r = tasks.reward_dict("reach", od, tasks.DEFAULT_WEIGHTS["reach"], {"ntip": 5, "far_th": 0.35, "dt": 0.02})
    assert all(np.shape(v) == () for v in r.values()), {k: np.shape(v) for k, v in r.items()}
    assert r["penalty"] == 0 and r["dense"] == 8.0          # d = 0: both bonus terms


def _single_step(case, v, a, oracles):
    """One step of the single env's batch v with action row a, replayed on the oracle (StepCheck of env 0)."""
    import torch
    S = v.get_env_state()
    ov0 = v.t["overflow"].cpu().numpy().copy()
    v.step(torch.as_tensor(a[None], device=v.device))
    torch.cuda.synchronize()
    t = v.t
    ret = tuple(t[k].cpu().numpy().copy() for k in ("obs", "reward", "done", "truncated", "last_return"))
    C = PH.StepCheck(case, v, S, a[None], ret, v.get_env_state(), ov0, t["overflow"].cpu().numpy().copy(), {0: (0, 0, 0)}, oracles)
    assert C.check(0, {"single"}), (case, C.cnt)
    return C


@pytest.mark.gpu
@pytest.mark.parametrize("eid", SINGLE_IDS)
def test_single_env_vs_oracle(eid, report):
    """make(id): one env in one warp of one CTA.  Two steps, a step that hits the TimeLimit (the env keeps its state: MyoEnv runs
    without auto-reset, the caller resets), reset() against the reset RNG's replay, two more steps; every step replayed on the oracle.
    Env 0 of a batch of the variant shape, stepped with the same rows, is bit-identical where both run the same kernel."""
    import torch

    import myosuite_b200
    from myosuite_b200 import vec_env
    t0 = time.time()
    env = myosuite_b200.make(eid, seed=PH.SEED)
    v = env.vec
    info = v.batch.launch_info()
    assert (info["warps_per_cta"], info["grid"], info["rounds"]) == (1, 1, 1), info
    base = _base(eid) if eid in vec_env.registry()["variants"] else eid
    n, expect, _ = BASE_SHAPE[base]
    batch = vec_env.MyoVecEnv(eid, n, seed=PH.SEED, auto_reset=False)
    binfo = batch.batch.launch_info()
    assert {k: binfo[k] for k in expect} == expect, binfo
    same_kernel = binfo["use_w14"] == info["use_w14"]
    batch.reset(seed=PH.SEED)
    m = v.mj_model
    rng = np.random.default_rng(PH.SEED)
    oracles = PH.Oracles(v)
    worst = dict(qpos=0.0, qvel=0.0, qacc=0.0, obs=0.0, reward=0.0)
    identical = True
    bg = torch.Generator(device="cpu").manual_seed(PH.SEED)
    for k in range(5):
        if k == 2:                          # the third step hits the TimeLimit
            env.set_env_state({"step_count": np.array(v.max_episode_steps - 1)})
            batch.t["step_count"][0] = v.max_episode_steps - 1
        if k == 3:                          # the caller's reset after the truncation: the draws of the env's next episode
            S = v.get_env_state()
            env.reset()
            batch.reset(mask=torch.as_tensor(np.eye(1, n, 0, dtype=np.uint8)[0], device=batch.device))
            N = v.get_env_state()
            assert N["episode_count"][0] == S["episode_count"][0] + 1 and N["step_count"][0] == 0 and N["time"][0] == 0
            P.compare_reset(v, N, P.replay_env(v, v.seed_value, S["episode_count"][[0]], [0]), eid + " reset", rows=[0])
        a = rng.uniform(-1, 1, m.nu).astype(np.float32)
        C = _single_step(eid, v, a, oracles)
        PH.check_map(PH.slot_table(info, 1, PH.perm_or_none(v, info)), 1)         # the slot map (load-sorted or fixed) steps env 0
        assert bool(C.trunc[0]) == (k == 2)
        for key in worst:
            worst[key] = max(worst[key], C.worst[key])
        rows = (torch.rand(n, m.nu, generator=bg) * 2 - 1)
        rows[0] = torch.as_tensor(a)
        batch.step(rows.to(batch.device))
        for key in ("qpos", "qvel", "act", "qacc_warmstart", "time", "obs", "reward"):
            same = torch.equal(batch.t[key][0], v.t[key][0])
            if same_kernel:
                assert same, (eid, k, key)
            identical = identical and same
    kern = lambda i: "w14" if i["use_w14"] else "k320"
    mp = lambda i: "regroup" if i["regroup"] else ("balanced" if i["balanced"] else "contiguous")
    line = ("single %-26s warps 1  grid 1  rounds 1  %s %s  5 steps (TimeLimit, reset, 2 more) worst: qpos %.1e  qvel %.1e  qacc %.1e  obs %.1e  "
            "reward %.1e;  env 0 of n %d (%s %s, %d warps x %d rounds): %s  [%.1f s]"
            % (eid, kern(info), mp(info), worst["qpos"], worst["qvel"], worst["qacc"], worst["obs"], worst["reward"], n, kern(binfo), mp(binfo),
               binfo["warps_per_cta"], binfo["rounds"],
               "same kernel, bit-identical" if same_kernel else ("other kernel, %s" % ("bit-identical" if identical else "not bit-identical")), time.time() - t0))
    report.append(line)
    print(line)
