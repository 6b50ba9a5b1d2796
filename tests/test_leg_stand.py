"""The leg stand task, myoLegStandRandom-v0 and its Sarc / Fati variants (the ReachEnvV0 of walk_v0.py on the legs model).

CPU: registry, the host obs_dict / rwd_dict / info, the oracle's reach rule with the stand shape (env_oracle.reach_obs_reward), the reset
rule (philox_ref.stand_reset_qpos) and the host-computed target centre against tests/golden/stand.npz, which the reference's own methods
produced (tests/golden/make_golden_stand.py).
GPU: the kernel's obs / reward / done on the golden states, the distribution of the randomised reset and the gym contract.  The product
step kernel is checked against the oracle at the benchmark shape in tests/test_product_parity.py (cases stand, stand_fatigue)."""
import copy
import os
import pickle

import numpy as np
import pytest

from myosuite_b200 import gym_api, tasks, vec_env
from philox_ref import stand_reset_qpos

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STAND = "myoLegStandRandom-v0"
IDS = (STAND, "myoSarcLegStandRandom-v0", "myoFatiLegStandRandom-v0")
NQ, NV, NA, DT = 35, 34, 80, 0.01
STAND_WEIGHTS = {"reach": 1.0, "bonus": 4.0, "penalty": 50, "act_reg": 1}        # walk_v0.py:18-24


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


def test_host_dicts_and_info_vs_reference_golden(models, Z):
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
    inf = tasks.info_from_obs("stand", Z["obs"], NQ, NV, NA, ntip=1)
    assert np.array_equal(inf["solved"], Z["obs_solved"].astype(bool))


def test_oracle_stand_obs_reward_vs_reference_golden(models, Z):
    """The oracle's reach rule with the kernel's stand shape (cfg.reach_shape) against the reference's own stand reward."""
    from oracle import env_oracle
    m = models["myolegs"]; o = _oracle(m)
    for i, (q, v, a, tg, tm) in enumerate(zip(Z["obs_qpos"], Z["obs_qvel"], Z["obs_act"], Z["obs_targets"], Z["obs_time"])):
        _observe(o, m, q, v, a)
        obs, r = env_oracle.reach_obs_reward(m, o, DT, ["pelvis"], tg[None], tm, far_th=0.44, shape=tasks.STAND_SHAPE, weights=STAND_WEIGHTS)
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

