"""The observation of the state an episode ended in (myo_buffers.final_obs, MyoVecEnv.step's info["final_obs"]) and PPO's bootstrapping of
time-limit truncations with it.

CPU: gae with bootstrapping against a per-env textbook loop, gae without it against the function it replaced, and the C-ABI field order.
GPU: twin batches of one id and seed, one with auto-reset and one without, driven by the same actions at the benchmarked launch shapes.
An env that ends for the first time has the same state in both, so the auto-reset twin's final_obs row must be bit-equal to the other
twin's obs row, and every output of that step must agree; rows that never ended must keep identical obs and an untouched (NaN) final_obs."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAND = "myoHandPoseRandom-v0"
SEED = 11


# ------------------------------------------------------------------------------------------------ CPU
def _gae_without_boot(rewards, values, dones, last_value, gamma, lam):
    """gae as it was before the boot argument (the default path must stay bit-identical to it)."""
    import torch
    T = rewards.shape[0]
    adv = torch.zeros_like(rewards)
    nxt, run = last_value, torch.zeros_like(last_value)
    for t in range(T - 1, -1, -1):
        live = 1.0 - dones[t].to(rewards.dtype)
        delta = rewards[t] + gamma * nxt * live - values[t]
        run = delta + gamma * lam * live * run
        adv[t] = run
        nxt = values[t]
    return adv, adv + values


def _episode_ends(T, n, rng):
    """done / truncated [T, n] covering terminations, pure truncations, both on the same step, and truncations at the last unroll step."""
    done = rng.uniform(size=(T, n)) < 0.15
    trunc = rng.uniform(size=(T, n)) < 0.15
    done[:, 0], trunc[:, 0] = False, False                     # env 0: never ends
    done[:, 1], trunc[:, 1] = False, np.arange(T) % 4 == 3     # env 1: pure truncations only, the last at t = T - 1
    done[:, 2], trunc[:, 2] = np.arange(T) % 3 == 1, False     # env 2: terminations only
    done[:, 3], trunc[:, 3] = False, False
    done[5, 3] = trunc[5, 3] = True                            # env 3: terminated and truncated on one step (no bootstrap)
    trunc[T - 1, 4], done[T - 1, 4] = True, False              # env 4: truncated on the last step
    return done, trunc


def test_gae_bootstrap_matches_textbook_loop():
    import torch
    from myosuite_b200.ppo import gae
    rng = np.random.default_rng(0); T, n, g, l = 16, 9, 0.97, 0.95
    r, v, lv, fv = rng.normal(size=(T, n)), rng.normal(size=(T, n)), rng.normal(size=n), rng.normal(size=(T, n))
    done, trunc = _episode_ends(T, n, rng)
    e, b = done | trunc, trunc & ~done
    assert (done & trunc).any() and b[T - 1].any() and b.any() and (done & ~trunc).any()
    adv = np.zeros((T, n))
    for k in range(n):                                         # delta_t = r_t + g [(1 - e_t) V_{t+1} + b_t Vf_t] - V_t ; run_t = delta_t + g l (1 - e_t) run_{t+1}
        run, nxt = 0.0, lv[k]
        for t in range(T - 1, -1, -1):
            live = 0.0 if e[t, k] else 1.0
            delta = r[t, k] + g * (live * nxt + (1.0 if b[t, k] else 0.0) * fv[t, k]) - v[t, k]
            run = delta + g * l * live * run
            adv[t, k] = run; nxt = v[t, k]
    fv_masked = torch.where(torch.tensor(b), torch.tensor(fv), 0.0)
    a, ret = gae(torch.tensor(r), torch.tensor(v), torch.tensor(e), torch.tensor(lv), g, l, boot=(torch.tensor(b), fv_masked))
    np.testing.assert_allclose(a.numpy(), adv, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ret.numpy(), adv + v, rtol=1e-12, atol=1e-12)
    # the bootstrap changes exactly the steps of truncated episodes and those before them in the same episode
    a0, _ = gae(torch.tensor(r), torch.tensor(v), torch.tensor(e), torch.tensor(lv), g, l)
    assert not torch.equal(a0[:, 1], a[:, 1]) and torch.equal(a0[:, 0], a[:, 0]) and torch.equal(a0[:, 2], a[:, 2]) and torch.equal(a0[:, 3], a[:, 3])


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_gae_without_bootstrap_is_unchanged(dtype):
    import torch
    from myosuite_b200.ppo import gae
    rng = np.random.default_rng(1); T, n, g, l = 20, 64, 0.97, 0.95
    dt = getattr(torch, dtype)
    r, v, lv = (torch.tensor(rng.normal(size=s), dtype=dt) for s in ((T, n), (T, n), (n,)))
    done, trunc = _episode_ends(T, n, rng)
    e = torch.tensor(done | trunc)
    ref = _gae_without_boot(r, v, e, lv, g, l)
    for got in (gae(r, v, e, lv, g, l), gae(r, v, e, lv, g, l, boot=None),
                gae(r, v, e, lv, g, l, boot=(torch.zeros(T, n, dtype=torch.bool), torch.tensor(rng.normal(size=(T, n)), dtype=dt)))):
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


def _header_buffer_fields():
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    body = src[:src.index("} myo_buffers;")]
    body = body[body.rindex("typedef struct {") + len("typedef struct {"):]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"\*\s*(\w+)\s*;", body), body.count(";")


def test_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_buffer_fields()
    assert len(fields) == decls                                # every member is a pointer
    assert abi.BUFFER_FIELDS == fields and fields[-1] == "final_obs"
    assert [n for n, _ in abi.MyoBuffers._fields_] == fields
    assert ctypes.sizeof(abi.MyoBuffers) == 8 * len(fields)
    assert abi.lib().myo_version() == 2


# ------------------------------------------------------------------------------------------------ GPU: twin batches
# case -> (env id, n_env, env kwargs, expected launch_info subset: the shapes test_product_parity.py checks), step cap
TWINS = {
    "hand_pose": (HAND, 4096, {}, dict(use_w14=1, warps_per_cta=11, rounds=3), 6),
    "hand_pose_f64rows": (HAND, 4096, {"row_storage": "f64"}, dict(use_w14=1, warps_per_cta=11, rounds=3), 6),
    "reach": ("myoHandReachRandom-v0", 4096, {}, dict(use_w14=1, warps_per_cta=11, rounds=3), 105),
    "elbow": ("myoElbowPose1D6MRandom-v0", 4096, {}, dict(use_w14=1, warps_per_cta=14, rounds=3), 6),
    "hold": ("myoHandObjHoldRandom-v0", 2048, {}, dict(use_w14=0, warps_per_cta=8, rounds=2), 80),
    "walk": ("myoFatiLegWalk-v0", 2048, {}, dict(use_w14=0, warps_per_cta=6, rounds=3), 300),
    "stand": ("myoLegStandRandom-v0", 2048, {}, dict(use_w14=0, warps_per_cta=6, rounds=3), 155),
}
TERMINATING = ("reach", "hold", "walk", "stand")          # tasks whose episodes also end by termination: >= N_MIN of each kind are checked
N_MIN = 32
LAUNCH_ENV = ("MYO_B200_REGROUP", "MYO_B200_W14", "MYO_B200_WARPS_PER_CTA")
REPORT = []


@pytest.fixture(scope="module")
def report():
    yield REPORT
    print("\nfinal_obs twins (first endings checked):")
    for line in REPORT:
        print("  " + line)


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32 if x.dtype == np.float32 else np.uint8)


def _twins(eid, n, kw, monkeypatch):
    from myosuite_b200 import vec_env
    for k in LAUNCH_ENV:
        monkeypatch.delenv(k, raising=False)
    auto = vec_env.MyoVecEnv(eid, n, seed=SEED, **kw)
    noauto = vec_env.MyoVecEnv(eid, n, seed=SEED, auto_reset=False, **kw)
    return auto, noauto


def _near_limit(envs, frac=4, seed=SEED):
    """step_count of about 1 / frac of the envs set 1-3 steps below the limit (same state on every env of `envs`)."""
    n, lim = envs[0].num_envs, envs[0].max_episode_steps
    rng = np.random.default_rng(seed)
    sel = rng.choice(n, n // frac, replace=False)
    sc = envs[0].get_env_state()["step_count"].copy()
    sc[sel] = lim - rng.integers(1, 4, size=sel.size)
    for e in envs:
        e.set_env_state({"step_count": sc})


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(TWINS))
def test_final_obs_twins(case, monkeypatch, report):
    import torch
    from myosuite_b200 import tasks
    eid, n, kw, expect, cap = TWINS[case]
    auto, noauto = _twins(eid, n, kw, monkeypatch)
    for e in (auto, noauto):
        info = e.batch.launch_info()
        assert {k: info[k] for k in expect} == expect, info
    m = auto.mj_model
    for e in (auto, noauto):
        e.reset(seed=SEED)
    _near_limit((auto, noauto))
    assert np.array_equal(_bits(auto.t["obs"].cpu().numpy()), _bits(noauto.t["obs"].cpu().numpy()))
    info_args = (m.nq, m.nv, m.na)
    info_kw = dict(pose_thd=float(auto.cfg.pose_thd), ntip=len(auto.tip_names) or None)
    g = torch.Generator(device=auto.device).manual_seed(SEED)
    ended = np.zeros(n, bool)
    n_term = n_trunc = n_both = steps = 0
    for steps in range(1, cap + 1):
        a = torch.rand(n, m.nu, device=auto.device, generator=g) * 2 - 1
        oa, ra, da, ta, ia = auto.step(a)
        ob, rb, db, tb, ib = noauto.step(a)
        assert ia["final_obs"].data_ptr() == auto.t["final_obs"].data_ptr()
        A = {k: auto.t[k].cpu().numpy() for k in ("obs", "final_obs", "reward", "done", "truncated", "last_return")}
        B = {k: noauto.t[k].cpu().numpy() for k in ("obs", "final_obs", "reward", "done", "truncated", "last_return")}
        live = ~ended
        end_a = (A["done"] | A["truncated"]).astype(bool)
        for k in ("reward", "done", "truncated", "last_return"):          # every env not ended before: the same step in both twins
            assert np.array_equal(_bits(A[k][live]), _bits(B[k][live])), (case, steps, k)
        first = end_a & live
        still = live & ~end_a
        assert np.array_equal(_bits(A["final_obs"][first]), _bits(B["obs"][first])), (case, steps)
        assert np.array_equal(_bits(A["obs"][still]), _bits(B["obs"][still])), (case, steps)
        assert np.isnan(A["final_obs"][still]).all(), (case, steps)          # no stray stores into rows of envs that never ended
        end_b = (B["done"] | B["truncated"]).astype(bool)                   # without auto-reset the copy equals obs, on every ending row
        assert np.array_equal(_bits(B["final_obs"][end_b]), _bits(B["obs"][end_b])), (case, steps)
        assert np.isnan(B["final_obs"][~end_b & live]).all()
        fi = auto.final_task_info()
        ref = tasks.info_from_obs(auto.task, noauto.t["obs_full"], *info_args, **info_kw)
        if ref is None:
            assert fi is None and auto.task == "walk"
        else:                       # rwd_sparse / solved of the ended states: those of the no-auto twin's obs
            fm = torch.as_tensor(first, device=auto.device)
            assert torch.equal(fi["rwd_sparse"][fm], ref["rwd_sparse"][fm]) and torch.equal(fi["solved"][fm], ref["solved"][fm])
        d, t_ = A["done"][first].astype(bool), A["truncated"][first].astype(bool)
        n_term += int(d.sum()); n_trunc += int((t_ & ~d).sum()); n_both += int((t_ & d).sum())
        ended |= end_a
        if case in TERMINATING and n_trunc >= N_MIN and n_term >= N_MIN:          # (the pose cases run their cap: every near-limit env ends)
            break
    line = "%-18s %-26s n %4d  steps %3d  first endings %4d: terminated %4d, truncated only %4d, both %d" % (
        case, eid, n, steps, int(ended.sum()), n_term, n_trunc, n_both)
    report.append(line)
    print(line)
    assert n_trunc >= N_MIN, line
    if case in TERMINATING:
        assert n_term >= N_MIN, line


# ------------------------------------------------------------------------------------------------ GPU: the public interface around it
@pytest.mark.gpu
def test_final_obs_custom_obs_keys():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv(HAND, 512, seed=SEED, obs_keys=["qpos", "pose_err"])
    cols = env._obs_cols
    assert cols is not None and env.obs_dim < env.full_obs_dim
    env.reset(seed=SEED)
    _near_limit((env,), frac=2)
    g = torch.Generator(device=env.device).manual_seed(SEED)
    ended = torch.zeros(env.num_envs, dtype=torch.bool, device=env.device)
    for _ in range(3):
        obs, _, done, trunc, info = env.step(torch.rand(env.num_envs, env.act_dim, device=env.device, generator=g) * 2 - 1)
        fo = info["final_obs"]
        assert fo.shape == (env.num_envs, env.obs_dim) and fo.shape == obs.shape
        full = env.t["final_obs_full"].index_select(1, cols)
        assert np.array_equal(_bits(fo.cpu().numpy()), _bits(full.cpu().numpy()))
        ended |= (done | trunc).bool()
    assert int(ended.sum()) >= env.num_envs // 4 and not torch.isnan(info["final_obs"][ended]).any()


@pytest.mark.gpu
def test_reset_and_observe_leave_final_obs_alone():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 512, seed=SEED)
    env.reset(seed=SEED)
    _near_limit((env,), frac=2)
    g = torch.Generator(device=env.device).manual_seed(SEED)
    for _ in range(3):
        env.step(torch.rand(env.num_envs, env.act_dim, device=env.device, generator=g) * 2 - 1)
    before = env.t["final_obs"].cpu().numpy().copy()
    ended = ~np.isnan(before).any(1)
    assert ended.sum() >= env.num_envs // 4
    obs0 = env.t["obs"].cpu().numpy().copy()
    mask = torch.zeros(env.num_envs, dtype=torch.uint8, device=env.device); mask[::3] = 1
    for call in (lambda: env.reset(mask=mask), env.refresh_obs, env.reset, lambda: env.reset(seed=SEED + 1)):
        call()
        assert np.array_equal(_bits(env.t["final_obs"].cpu().numpy()), _bits(before))
    assert not np.array_equal(env.t["obs"].cpu().numpy(), obs0)          # (the calls did write obs)


@pytest.mark.gpu
def test_physics_only_batch_binds_no_final_obs():
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv.from_model("myoelbow_1dof6muscles", 32)
    assert "final_obs" not in env.t and env.final_task_info() is None
    *_, info = env.step(torch.zeros(32, env.act_dim, device=env.device))
    assert info["final_obs"] is None
    from myosuite_b200 import abi
    with pytest.raises(abi.MyoError, match="final_obs"):          # the copy's source is obs: binding final_obs without it is refused
        env.batch.bind(obs=None, final_obs=torch.zeros(32, 1, device=env.device))


@pytest.mark.gpu
def test_ppo_bootstrap_truncated_improves_elbow_pose():
    """The budget and bound of test_ppo.py's test_ppo_improves_elbow_pose, with time-limit truncations bootstrapped."""
    from myosuite_b200 import ppo, vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 1024, seed=3)
    agent = ppo.PPO(env, unroll=20, minibatches=8, epochs=4, seed=3, bootstrap_truncated=True)
    hist = agent.train(40 * 20 * 1024)
    first = np.mean([h["reward_per_step"] for h in hist[:3]]); last = np.mean([h["reward_per_step"] for h in hist[-3:]])
    print("PPO elbow, truncations bootstrapped: reward/step %.3f -> %.3f over %d env-steps, %.0f env-steps/s incl. updates"
          % (first, last, hist[-1]["steps"], hist[-1]["steps_per_s"]))
    assert last > first + 0.5 and all(np.isfinite(h["value_loss"]) for h in hist)
