"""The leg stand task, myoLegStandRandom-v0 and its Sarc / Fati variants (the ReachEnvV0 of walk_v0.py on the legs model).

CPU: registry, the host obs_dict / rwd_dict, the CPU reference of the task (tests/stand_oracle.py) and the host-computed target centre
against tests/golden/stand.npz, which the reference's own methods produced (tests/golden/make_golden_stand.py).
GPU: the kernel's obs / reward / done on the golden states, the distribution of the randomised reset, the product step kernel against the
oracle at the benchmark shape (first steps after a reset and in-kernel auto-resets included) and the gym contract."""
import copy
import os
import pickle
import time

import numpy as np
import pytest

from myosuite_b200 import gym_api, vec_env
from stand_oracle import STAND_WEIGHTS, stand_obs_reward, stand_reset_qpos

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STAND = "myoLegStandRandom-v0"
IDS = (STAND, "myoSarcLegStandRandom-v0", "myoFatiLegStandRandom-v0")
NQ, NV, NA, DT = 35, 34, 80, 0.01


@pytest.fixture(scope="module")
def Z():
    return np.load(os.path.join(G, "stand.npz"))


def _oracle(m):
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    return Oracle(*blob.pack(m))


def _observe(o, m, q, v, a):
    o.reset(); o.set(qpos=q, qvel=v, act=a, ctrl=np.zeros(m.nu)); o.forward()


# ------------------------------------------------------------------------------------------------ CPU
def test_registry_ids_and_kwargs():
    ids = vec_env.registered_ids()
    assert set(IDS) <= set(ids) and "myoReafLegStandRandom-v0" not in ids        # Reaf variants exist for myoHand ids only
    steps, kw, entry = vec_env.env_spec(STAND)
    assert steps == 150 and entry.endswith("walk_v0:ReachEnvV0")
    assert kw == {"model_path": "simhive/myo_sim/leg/myolegs.xml", "joint_random_range": [-0.2, 0.2],
                  "target_reach_range": {"pelvis": [[-0.05, -0.05, 0], [0.05, 0.05, 0]]}, "normalize_act": True, "far_th": 0.44}
    assert vec_env.env_spec("myoSarcLegStandRandom-v0")[1]["muscle_condition"] == "sarcopenia"
    assert vec_env.env_spec("myoFatiLegStandRandom-v0")[1]["muscle_condition"] == "fatigue"
    vec_env.MyoVecEnv._check_kwargs(kw)
    assert gym_api.DEFAULT_WEIGHTS["stand"] == STAND_WEIGHTS
    assert gym_api.obs_layout("stand", NQ, NV, NA, 1) == gym_api.obs_layout("reach", NQ, NV, NA, 1)
    assert sum(w for _, w in gym_api.obs_layout("stand", NQ, NV, NA, 1)) == 155


def _f64_obs_dict(models, Z):
    """obs_dict of the golden states in f64 (the reference's own precision), from the oracle."""
    m = models["myolegs"]; o = _oracle(m); sid = m.name2id("site", "pelvis")
    d = {k: [] for k in ("qpos", "qvel", "tip_pos", "reach_err", "act")}
    for q, v, a, tg in zip(Z["obs_qpos"], Z["obs_qvel"], Z["obs_act"], Z["obs_targets"]):
        _observe(o, m, q, v, a)
        tip = o.f("site_xpos").reshape(-1, 3)[sid].copy()
        for k, x in (("qpos", o.f("qpos").copy()), ("qvel", o.f("qvel") * DT), ("tip_pos", tip), ("reach_err", tg - tip), ("act", o.f("act").copy())):
            d[k].append(x)
    return dict({k: np.array(x) for k, x in d.items()}, time=Z["obs_time"])


def test_host_dicts_vs_reference_golden(models, Z):
    # the obs_dict is a view of the observation vector
    od = gym_api.obs_dict_from_vec("stand", Z["obs"], Z["obs_time"], NQ, NV, NA, ntip=1)
    assert list(od) == ["time", "qpos", "qvel", "tip_pos", "reach_err", "act"]
    np.testing.assert_array_equal(np.concatenate([od[k] for k in list(od)[1:]], -1), Z["obs"])
    cfg = {"ntip": 1, "far_th": 0.44, "dt": DT}
    # the reward terms: f64 inputs reproduce the reference to round-off ...
    r = gym_api.reward_dict("stand", _f64_obs_dict(models, Z), gym_api.DEFAULT_WEIGHTS["stand"], cfg)
    for k in ("reach", "bonus", "act_reg", "penalty", "sparse", "dense"):
        np.testing.assert_allclose(r[k], Z["obs_" + k], rtol=1e-12, atol=1e-12, err_msg=k)
    for k in ("solved", "done"):
        assert np.array_equal(np.asarray(r[k], bool), Z["obs_" + k].astype(bool)), k
    # ... and the f32 observation the host sees gives the same flags and the reward to f32 round-off
    r = gym_api.reward_dict("stand", od, gym_api.DEFAULT_WEIGHTS["stand"], cfg)
    np.testing.assert_allclose(r["dense"], Z["obs_dense"], rtol=2e-5, atol=2e-5)
    for k in ("solved", "done"):
        assert np.array_equal(np.asarray(r[k], bool), Z["obs_" + k].astype(bool)), k
    # the golden spans both sides of every threshold: d = 0.05, 0.1, 0.44 and time = 2 dt
    d = -Z["obs_sparse"]; armed = Z["obs_time"] > 2 * DT
    for th in (0.05, 0.1):
        assert np.any(d < th) and np.any(d > th)
    assert np.any(armed & (d > 0.44)) and np.any(armed & (d < 0.44)) and np.any(~armed & (d > 0.44)) and np.any(~armed)
    from myosuite_b200 import task_info
    inf = task_info.info_from_obs("stand", Z["obs"], NQ, NV, NA, ntip=1)
    assert np.array_equal(inf["solved"], Z["obs_solved"].astype(bool))


def test_oracle_stand_obs_reward_vs_reference_golden(models, Z):
    m = models["myolegs"]; o = _oracle(m)
    for i, (q, v, a, tg, tm) in enumerate(zip(Z["obs_qpos"], Z["obs_qvel"], Z["obs_act"], Z["obs_targets"], Z["obs_time"])):
        _observe(o, m, q, v, a)
        obs, r = stand_obs_reward(m, o, DT, ["pelvis"], tg[None], tm, far_th=0.44)
        np.testing.assert_array_equal(obs, Z["obs"][i])
        for k in ("reach", "bonus", "act_reg", "penalty", "sparse", "dense"):
            assert r[k] == pytest.approx(Z["obs_" + k][i], rel=1e-12, abs=1e-12), (i, k)
        assert r["done"] == bool(Z["obs_done"][i]) and r["solved"] == bool(Z["obs_solved"][i])


def test_reset_mirror_bit_equal_to_reference(models, Z):
    m = models["myolegs"]
    for u, q in zip(Z["reset_u"], Z["reset_qpos"]):
        assert np.array_equal(stand_reset_qpos(m, m.key_qpos[0], u[m.jnt_qposadr]), q)
    Q = Z["reset_qpos"]; k0 = m.key_qpos[0]
    assert np.all(Q[:, 0] == 0) and np.all(Q[:, 1:7] == k0[1:7])           # free root: x pinned by its [0, 0] range, the rest untouched
    assert np.any(np.all(Q == Q[:1], axis=0) == False)                      # noqa: E712  (the draws differ)


def test_target_centre_vs_reference_golden(models, Z):
    m = models["myolegs"]
    c = vec_env.stand_target_centre(m, ["pelvis"], m.key_qpos[0])
    assert c.shape == (1, 3)
    np.testing.assert_allclose(np.broadcast_to(c, Z["target_centre"].shape), Z["target_centre"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(c[0], [0.0, 0.0, 0.92], atol=1e-12)
    lo, hi = np.array([-0.05, -0.05, 0.0]), np.array([0.05, 0.05, 0.0])
    np.testing.assert_allclose(Z["target"], c + (lo + (hi - lo) * Z["target_u"]), rtol=0, atol=1e-15)
    assert np.all(Z["target"][:, 2] == Z["target_centre"][:, 2])
    # a tip site that the randomised draw can move makes the centre non-constant: refused
    m2 = copy.deepcopy(m); m2.jnt_range[0] = [-1.0, 1.0]
    with pytest.raises(NotImplementedError):
        vec_env.stand_target_centre(m2, ["pelvis"], m2.key_qpos[0])


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_stand_golden_on_device(Z):
    """obs / reward / done of the kernel epilogue on the golden states (the reference's own get_obs_dict / get_reward_dict)."""
    import torch
    n = len(Z["obs"])
    env = vec_env.MyoVecEnv(STAND, n, auto_reset=False)
    assert env.obs_dim == 155 and env.act_dim == 80 and env.dt == pytest.approx(DT) and env.max_episode_steps == 150 and env.task == "stand"
    env.set_state(qpos=Z["obs_qpos"], qvel=Z["obs_qvel"], act=Z["obs_act"])
    env.t["target"][:, :3] = torch.as_tensor(Z["obs_targets"], device=env.device)
    env.t["time"][:] = torch.as_tensor(Z["obs_time"], device=env.device)
    env.refresh_obs(); torch.cuda.synchronize()
    np.testing.assert_allclose(env.t["obs"].cpu().numpy(), Z["obs"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(env.t["reward"].cpu().numpy(), Z["obs_dense"], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), Z["obs_done"].astype(bool))


def _binom_ok(k, n, p):
    return abs(k - n * p) <= 6 * np.sqrt(n * p * (1 - p)) + 1


@pytest.mark.gpu
def test_stand_reset_distribution():
    """4096 resets against the reference's rule: every joint's first coordinate init + U(-0.2, 0.2) clipped to jnt_range; target xy
    U(+-0.05) around the constant centre, z exact; zero velocity and activation; reproducible under reset(seed=s), distinct streams
    across env_offset."""
    import torch
    from scipy import stats
    n = 4096
    env = vec_env.MyoVecEnv(STAND, n, seed=11)
    m = env.mj_model; k0 = m.key_qpos[0]
    env.reset(seed=11); torch.cuda.synchronize()
    S = env.get_env_state()
    Q, T = S["qpos"], S["target"][:, :3]
    assert np.all(Q[:, 0] == 0.0) and np.all(Q[:, 1:7] == k0[1:7])
    assert np.all(S["qvel"] == 0) and np.all(S["act"] == 0) and np.all(S["time"] == 0) and np.all(S["step_count"] == 0)
    worst_p = 1.0
    for j in range(1, m.njnt):
        qa = m.jnt_qposadr[j]; lo, hi = m.jnt_range[j]; a, b = k0[qa] - 0.2, k0[qa] + 0.2
        x = Q[:, qa]
        assert np.all(x >= lo) and np.all(x <= hi), j
        p_lo, p_hi = np.clip((lo - a) / 0.4, 0, 1), np.clip((b - hi) / 0.4, 0, 1)
        n_lo, n_hi = int(np.sum(x == lo)), int(np.sum(x == hi))
        assert _binom_ok(n_lo, n, p_lo) and _binom_ok(n_hi, n, p_hi), (j, n_lo, n * p_lo, n_hi, n * p_hi)
        inner = x[(x > lo) & (x < hi)]
        ilo, ihi = max(lo, a), min(hi, b)
        if len(inner) > 20:
            p = stats.kstest(inner, stats.uniform(loc=ilo, scale=ihi - ilo).cdf).pvalue
            worst_p = min(worst_p, p)
            assert p > 1e-5, (j, p)
    c = env.target_center[0]
    assert np.all(T[:, 2] == c[2])
    for k in range(2):
        assert np.all(np.abs(T[:, k] - c[k]) <= 0.05)
        assert stats.kstest(T[:, k], stats.uniform(loc=c[k] - 0.05, scale=0.1).cdf).pvalue > 1e-5
    obs = env.t["obs"].cpu().numpy()
    np.testing.assert_array_equal(obs[:, :NQ], Q.astype(np.float32))
    # reproducible under reset(seed=s); a different seed or env_offset gives other draws
    env.reset(seed=11); torch.cuda.synchronize()
    assert np.array_equal(env.get_env_state()["qpos"], Q) and np.array_equal(env.get_env_state()["target"][:, :3], T)
    env.reset(seed=12); torch.cuda.synchronize()
    assert np.mean(np.all(env.get_env_state()["qpos"] == Q, axis=1)) < 0.01
    off = vec_env.MyoVecEnv(STAND, 64, seed=11, env_offset=64)
    off.reset(seed=11); torch.cuda.synchronize()
    Qo = off.get_env_state()["qpos"]
    assert np.array_equal(Qo, Q[64:128])                                    # the stream belongs to the global env index
    assert np.mean(np.all(Qo == Q[:64], axis=1)) < 0.1
    print("reset distribution: worst KS p-value over the interior of the %d joints: %.3g" % (m.njnt - 1, worst_p))


@pytest.mark.gpu
@pytest.mark.parametrize("env_id", IDS)
def test_stand_gym_contract(env_id):
    import myosuite_b200 as myo
    env1 = myo.make(env_id, seed=5).unwrapped
    obs0, _ = env1.reset()
    assert obs0.shape == (155,) and obs0.dtype == np.float32 and env1.observation_space.shape == (155,) and env1.action_space.shape == (80,)
    u = 0.1 * np.random.default_rng(0).uniform(0, 1, 80)
    obs1, rwd1, done1, trunc1, info1 = env1.step(u)
    assert obs1.shape == (155,) and isinstance(rwd1, float) and isinstance(done1, bool)
    od = env1.get_obs_dict(); rd = env1.get_reward_dict(od)
    assert list(od) == ["time", "qpos", "qvel", "tip_pos", "reach_err", "act"]
    assert {"reach", "bonus", "act_reg", "penalty", "sparse", "solved", "done", "dense"} <= set(rd)
    np.testing.assert_allclose(np.concatenate([np.ravel(od[k]) for k in env1.obs_keys]), obs1)
    host = gym_api.reward_dict("stand", od, env1.rwd_keys_wt, env1._task_cfg)["dense"]
    assert float(host) == pytest.approx(rwd1, rel=2e-5, abs=2e-5)          # host recomputation from the f32 observation vs the device's f64 reward
    # set_env_state: the target row drives reach_err
    st = env1.get_env_state()
    st2 = copy.deepcopy(st); st2["target"][:3] = st["target"][:3] + np.array([0.3, 0.0, 0.0])
    env1.set_env_state(st2)
    np.testing.assert_allclose(env1.obs_dict["reach_err"], od["reach_err"] + np.array([0.3, 0, 0], np.float32), atol=1e-6)
    env1.set_env_state(st)
    np.testing.assert_allclose(env1.obs_dict["reach_err"], od["reach_err"], atol=0)
    # pickle round trip
    env2 = pickle.loads(pickle.dumps(env1)).unwrapped
    assert env2.env_id == env_id
    np.testing.assert_array_equal(env2.get_env_state()["qpos"], st["qpos"])
    np.testing.assert_array_equal(env2.get_env_state()["target"], st["target"])
    o2, r2, *_ = env2.step(u); o1, r1, *_ = env1.step(u)
    np.testing.assert_allclose(o2, o1, atol=1e-6); assert r2 == pytest.approx(r1, abs=1e-5)
    # seeded resets reproduce
    env2.seed(5); a, _ = env2.reset(); env1.seed(5); b, _ = env1.reset()
    np.testing.assert_array_equal(a, b)
    if "Fati" in env_id:
        assert "fatigue" in env1.get_env_state()


# ---- the product step kernel against the oracle at the benchmark shape
STAND_CASES = {
    "stand": (STAND, 2048, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1)),
    "stand_fatigue": ("myoFatiLegStandRandom-v0", 2048, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1)),
}
N_FIRST = 48              # envs reset just before the checked step: it is their first step, from a state whose joint couplings are broken
REPORT = []


@pytest.fixture(scope="module")
def report():
    yield
    if REPORT:
        print("\nleg stand, product kernel vs oracle:")
        for line in REPORT:
            print("  " + line)


def _stand_task_obs(env, o, tnow, target):
    """obs, dense reward, done of the oracle's current state, and the distance of d to the nearest threshold it is compared with."""
    m, far_th = env.mj_model, float(env.kwargs["far_th"])
    o.set(ctrl=np.zeros(m.nu)); o.forward()
    obs, r = stand_obs_reward(m, o, env.dt, env.tip_names, target[:3].reshape(1, 3), tnow, far_th=far_th)
    d = -r["sparse"]
    ths = [0.05, 0.1] + ([far_th] if tnow > 2 * env.dt else [])
    return obs, r["dense"], r["done"], min(abs(d - t) for t in ths)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(STAND_CASES))
def test_stand_product_step_vs_oracle(case, monkeypatch, report):
    """test_product_parity.py's replay on the stand task: launch shape, slot map on every step, a quarter of the envs forced to the
    TimeLimit (in-kernel auto-resets), plus envs reset right before the checked step, so that the step from a freshly randomised state
    (couplings violated) is held to the mid-episode bounds too."""
    import torch
    from oracle import env_oracle
    from parity_helpers import _in_regime, relerr
    from test_product_parity import (ACT_ATOL, FATIGUE_RTOL, LAUNCH_ENV, MAX_SKIP_REGIME, N_RESET, QACC_REL, QPOS_ATOL, QVEL_REL, SEED,
                                     THRESHOLD_MARGIN, WARM, Oracles, check_map, load_state, perm_or_none, select, slot_table)
    eid, n, expect = STAND_CASES[case]
    for k in LAUNCH_ENV:
        monkeypatch.delenv(k, raising=False)
    t0 = time.time()
    env = vec_env.MyoVecEnv(eid, n, seed=SEED)
    m = env.mj_model
    info = env.batch.launch_info()
    assert {k: info[k] for k in expect} == expect, info
    env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    for _ in range(WARM):
        env.step((torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device))
        check_map(slot_table(info, n, perm_or_none(env, info)), n)
    rng = np.random.default_rng(SEED)
    trunc_set = rng.choice(n, n // 4, replace=False)
    first_set = rng.choice(np.setdiff1d(np.arange(n), trunc_set), N_FIRST, replace=False)
    mask = np.zeros(n, np.uint8); mask[first_set] = 1
    env.reset(mask=torch.as_tensor(mask, device=env.device))
    S0 = env.get_env_state()
    sc = S0["step_count"].copy(); sc[trunc_set] = env.max_episode_steps - 1
    env.set_env_state({"step_count": sc})
    S = env.get_env_state()
    assert np.all(S["step_count"][first_set] == 0) and np.all(S["time"][first_set] == 0) and np.all(S["qacc_warmstart"][first_set] == 0)
    ov0 = env.t["overflow"].cpu().numpy().copy()
    a = (torch.rand(n, m.nu, generator=g) * 2 - 1).numpy().astype(np.float32)
    oracles = Oracles(env)

    obs, rew, done, trunc, info_d = env.step(torch.as_tensor(a, device=env.device))
    torch.cuda.synchronize()
    obs, rew, done, trunc = (x.cpu().numpy().copy() for x in (obs, rew, done, trunc))
    last_ret, ov = info_d["last_return"].cpu().numpy().copy(), env.t["overflow"].cpu().numpy().copy()
    N = env.get_env_state()
    T = slot_table(info, n, perm_or_none(env, info))
    check_map(T, n)
    assert np.all(trunc[trunc_set])
    chosen = select(T, rng, [], rng.choice(trunc_set, N_RESET, replace=False))
    for e in first_set:
        chosen.setdefault(int(e), set()).add("first-step")
    where = {int(e): (r, w, c) for (r, w, c), e in np.ndenumerate(T) if e >= 0}
    worst = {k: 0.0 for k in ("qpos", "qvel", "qacc", "obs", "reward", "qpos_first", "qvel_first", "qacc_first")}
    cnt = dict(checked=0, phys=0, first=0, reset=0, threshold=0, overflow=0, regime=0)
    tr = env.t["target_range"].cpu().numpy()
    k0 = m.key_qpos[0]

    def check(e, why):
        msg = "%s env %d (round, warp, cta) %s, checked as %s" % (case, e, where[e], sorted(why))
        if ov0[e] or ov[e]:
            cnt["overflow"] += 1
            return
        o = oracles.get(); load_state(o, env, S, e)
        fat = None
        if "fatigue" in S:
            fat = env_oracle.Fatigue(m.nu, dt=env.dt, tauact=m.actuator_dynprm[:, 0], taudeact=m.actuator_dynprm[:, 1])
            fat.MA, fat.MR, fat.MF = (S["fatigue"][e, k].copy() for k in range(3))
        ctrl = env_oracle.action_to_ctrl(a[e].astype(np.float64), bool(env.cfg.normalize_act))
        o.set(ctrl=fat.compute_act(ctrl)[0].copy() if fat is not None else ctrl)
        in_regime = True
        for _ in range(env.n_frames):
            o.step(1); in_regime = in_regime and _in_regime(o, m)
        if not in_regime:
            cnt["regime"] += 1
            return
        tnow = float(S["time"][e])
        for _ in range(env.n_frames):
            tnow += m.opt_timestep
        qpos, qvel, act, qacc = (o.f(k).copy() for k in ("qpos", "qvel", "act", "qacc"))
        x_obs, x_rw, x_done, margin = _stand_task_obs(env, o, tnow, S["target"][e])
        x_trunc = int(S["step_count"][e]) + 1 >= env.max_episode_steps
        if margin > THRESHOLD_MARGIN:
            worst["reward"] = max(worst["reward"], abs(float(rew[e]) - x_rw))
            assert rew[e] == pytest.approx(x_rw, rel=1e-5, abs=1e-5), msg
            assert bool(done[e]) == bool(x_done), msg
        else:
            cnt["threshold"] += 1
        assert bool(trunc[e]) == x_trunc, msg
        R = np.float32(S["ep_return"][e]) + rew[e]
        if done[e] or trunc[e]:
            assert last_ret[e] == R, msg
            cnt["reset"] += 1
            q = N["qpos"][e]
            assert np.all(N["act"][e] == 0) and np.all(N["qacc_warmstart"][e] == 0) and N["time"][e] == 0 and np.all(N["qvel"][e] == 0), msg
            assert N["step_count"][e] == 0 and N["episode_count"][e] == S["episode_count"][e] + 1 and N["ep_return"][e] == 0, msg
            assert q[0] == 0 and np.all(q[1:7] == k0[1:7]), msg
            adr = m.jnt_qposadr[1:]
            assert np.all(q[adr] >= m.jnt_range[1:, 0]) and np.all(q[adr] <= m.jnt_range[1:, 1]) and np.all(np.abs(q[adr] - k0[adr]) <= 0.2 + 1e-12), msg
            assert np.all(N["target"][e][:3] >= tr[:3, 0]) and np.all(N["target"][e][:3] <= tr[:3, 1]), msg
            if "fatigue" in N:
                assert np.all(N["fatigue"][e, 0] == 0) and np.all(N["fatigue"][e, 1] == 1) and np.all(N["fatigue"][e, 2] == 0), msg
            o = oracles.get(); load_state(o, env, N, e)
            np.testing.assert_allclose(obs[e], _stand_task_obs(env, o, 0.0, N["target"][e])[0], rtol=2e-6, atol=2e-6, err_msg=msg)
        else:
            first = "first-step" in why
            cnt["phys"] += 1; cnt["first"] += first
            sfx = "_first" if first else ""
            worst["qpos" + sfx] = max(worst["qpos" + sfx], float(np.abs(N["qpos"][e] - qpos).max()))
            worst["qvel" + sfx] = max(worst["qvel" + sfx], relerr(N["qvel"][e], qvel))
            worst["qacc" + sfx] = max(worst["qacc" + sfx], relerr(N["qacc_warmstart"][e], qacc))
            np.testing.assert_allclose(N["qpos"][e], qpos, rtol=0, atol=QPOS_ATOL, err_msg=msg)
            assert relerr(N["qvel"][e], qvel) < QVEL_REL, msg
            assert relerr(N["qacc_warmstart"][e], qacc) < QACC_REL, msg
            np.testing.assert_allclose(N["act"][e, :m.na], act, rtol=0, atol=ACT_ATOL, err_msg=msg)
            if fat is not None:
                np.testing.assert_allclose(N["fatigue"][e], np.stack([fat.MA, fat.MR, fat.MF]), rtol=FATIGUE_RTOL, atol=1e-15, err_msg=msg)
            assert N["time"][e] == tnow and N["step_count"][e] == S["step_count"][e] + 1 and N["ep_return"][e] == R, msg
            worst["obs"] = max(worst["obs"], float(np.abs(obs[e] - x_obs).max()))
            np.testing.assert_allclose(obs[e], x_obs, rtol=2e-6, atol=2e-6, err_msg=msg)
        cnt["checked"] += 1

    for e in sorted(chosen):
        check(e, chosen[e])
    REPORT.append("%-14s %-26s n %4d  %s  warps %d  grid %d  rounds %d  checked %d of %d (physics %d, of them first steps after a reset %d; "
                  "auto-reset %d; skipped: deep penetration %d, contact overflow %d; near a threshold %d)  worst: qpos %.1e qvel %.1e qacc %.1e "
                  "(first steps: qpos %.1e qvel %.1e qacc %.1e)  obs %.1e  reward %.1e  [%.1f s]"
                  % (case, eid, n, "w14" if info["use_w14"] else "k320", info["warps_per_cta"], info["grid"], info["rounds"], cnt["checked"], len(chosen),
                     cnt["phys"], cnt["first"], cnt["reset"], cnt["regime"], cnt["overflow"], cnt["threshold"], worst["qpos"], worst["qvel"], worst["qacc"],
                     worst["qpos_first"], worst["qvel_first"], worst["qacc_first"], worst["obs"], worst["reward"], time.time() - t0))
    print(REPORT[-1])
    assert cnt["reset"] >= N_RESET and cnt["first"] >= N_FIRST // 2 and cnt["phys"] >= 32
    assert cnt["regime"] <= MAX_SKIP_REGIME * len(chosen) and cnt["overflow"] <= 3
