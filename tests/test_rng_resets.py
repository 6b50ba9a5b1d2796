"""The reset random number generator: Philox4x32-10 streams keyed (seed, global env, episode, lane), and the draws env_reset takes from them.

CPU: tests/philox_ref.py against the Random123 known-answer vectors, the uniform's edges, and the stream key: unchanged below 2^20 envs,
injective over its domain (env < 2^47, episode < 2^44, lane < 32).
GPU: resets of every task branch against philox_ref.replay_reset -- bit for bit where the kernel's expression admits no contraction
(fatigue state, stand joint offsets, walk keyframe row), else to a few ulps (nvcc may fuse lo + u span into an FMA) -- at seed, env id and
episode boundaries of the key, for an in-kernel auto-reset, and the rejection of seeds and env offsets outside the key's domain.
The statistical reset tests (test_leg_stand.py, test_gpu_env.py) check the distributions the reference specifies; these check the generator."""
import numpy as np
import pytest

import philox_ref as P



# ------------------------------------------------------------------------------------------------ CPU
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_R(10)."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        np.testing.assert_array_equal(P.philox4x32(np.array(ctr), np.array(key)), np.array(want, dtype=np.uint32))
    # vectorised over streams: the same answers in one call
    got = P.philox4x32(np.array([c for c, _, _ in cases]), np.array([k for _, k, _ in cases]))
    np.testing.assert_array_equal(got, np.array([w for _, _, w in cases], dtype=np.uint32))


def test_uniform_edges():
    assert P.uniform53(0, 0) == 0.0
    assert P.uniform53(0xffffffff, 0xffffffff) == 1.0 - 2.0 ** -53
    assert P.uniform53(0x80000000, 0) == 0.5                               # a's top bit is the uniform's first bit
    assert P.uniform53(0, 0x40) == 2.0 ** -53                              # b's bit 6 is the last one kept
    assert P.uniform53(0x1f, 0x3f) == 0.0                                  # the dropped low bits of both words
    u = P.uniforms(1, np.arange(64)[:, None], 0, np.arange(32)[None, :], 8)
    assert u.min() >= 0.0 and u.max() < 1.0 and len(np.unique(u)) == u.size


def _key_words(seed, env, episode, lane):
    ctr, key = P.stream_key(seed, env, episode, lane)
    return np.concatenate([key, ctr[..., 1:]], axis=-1)                  # (k0, k1, c1, c2, c3); c0 is the draw counter


def test_key_unchanged_below_2_20_envs():
    """Every stream of an env id below 2^20 (all that the goldens, policy replays and benchmark dumps use) is the one it always was:
    c1 = lane, c2 = env ^ episode << 20, c3 = env >> 32 ^ episode >> 12 ^ 'MYOB'."""
    rng = np.random.default_rng(0)
    env = rng.integers(0, 1 << 20, 4096, dtype=np.uint64); ep = rng.integers(0, 1 << 44, 4096, dtype=np.uint64)
    lane = rng.integers(0, 32, 4096, dtype=np.uint64); seed = rng.integers(0, 1 << 64, 4096, dtype=np.uint64, endpoint=False)
    M = np.uint64(P.M32)
    want = np.stack([seed & M, seed >> np.uint64(32), lane, env ^ ((ep << np.uint64(20)) & M), (ep >> np.uint64(12)) & M ^ np.uint64(P.KEY_TAG)], -1)
    np.testing.assert_array_equal(_key_words(seed, env, ep, lane), want)


def _assert_injective(seed, env, episode, lane):
    t = np.unique(np.stack(np.broadcast_arrays(*(np.asarray(x, dtype=np.uint64) for x in (seed, env, episode, lane))), -1).reshape(-1, 4), axis=0)
    k = np.unique(_key_words(t[:, 0], t[:, 1], t[:, 2], t[:, 3]), axis=0)
    assert len(k) == len(t), "%d distinct (seed, env, episode, lane) share %d keys" % (len(t), len(k))
    return len(t)


def test_key_injective_structured_pairs():
    """Env k ^ (x << 20) at episode e and env k at episode e ^ x: the same key before c1 carried env bits 20 and up."""
    rng = np.random.default_rng(1)
    k = rng.integers(0, 1 << 20, 512, dtype=np.uint64); x = rng.integers(1, 1 << 12, 512, dtype=np.uint64)
    e = rng.integers(0, 1 << 12, 512, dtype=np.uint64); lane = rng.integers(0, 32, 512, dtype=np.uint64)
    a = _key_words(7, k ^ (x << np.uint64(20)), e, lane); b = _key_words(7, k, e ^ x, lane)
    assert not np.any(np.all(a == b, axis=1))
    # the first episode of global env 2^20 and the second of env 0
    assert not np.array_equal(_key_words(0, 1 << 20, 0, 3), _key_words(0, 0, 1, 3))


def test_key_injective_at_boundaries():
    envs = [0, 1, 31, 32, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, (1 << 21) + 5, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 32) + (1 << 20),
            (1 << 46) + 3, P.ENV_LIMIT - 1]
    episodes = [0, 1, 4095, 4096, 4097, (1 << 20) + 1, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, P.EPISODE_LIMIT - 1]
    n = _assert_injective(np.array([0, 1, (1 << 32) - 1, 1 << 32, (1 << 64) - 1], dtype=np.uint64)[:, None, None, None],
                          np.array(envs, dtype=np.uint64)[None, :, None, None], np.array(episodes, dtype=np.uint64)[None, None, :, None],
                          np.array([0, 1, 30, 31], dtype=np.uint64)[None, None, None, :])
    assert n == 5 * len(envs) * len(episodes) * 4


def test_key_injective_random_tuples():
    """10^6 tuples from the domain: a third anywhere, a third with small env ids and episodes (where the structured collisions live), a
    third around env 2^32."""
    rng = np.random.default_rng(2)
    s = 1_000_000 // 3
    seed = rng.choice(np.array([0, 5, (1 << 32) + 5, (1 << 64) - 1], dtype=np.uint64), 3 * s)
    env = np.concatenate([rng.integers(0, P.ENV_LIMIT, s, dtype=np.uint64), rng.integers(0, 1 << 24, s, dtype=np.uint64),
                          rng.integers((1 << 32) - (1 << 22), (1 << 32) + (1 << 22), s, dtype=np.uint64)])
    ep = np.concatenate([rng.integers(0, P.EPISODE_LIMIT, s, dtype=np.uint64), rng.integers(0, 1 << 6, s, dtype=np.uint64),
                         rng.integers(0, 1 << 14, s, dtype=np.uint64)])
    lane = rng.integers(0, 32, 3 * s, dtype=np.uint64)
    n = _assert_injective(seed, env, ep, lane)
    assert n > 0.9 * 3 * s


# ------------------------------------------------------------------------------------------------ GPU
# task branches of env_reset; every fatigue case draws the fatigue state after the task's own draws (several counters on every lane)
CASES = {
    "hand_pose_fatigue": ("myoFatiHandPoseRandom-v0", dict(fatigue_reset_random=True)),
    "elbow_pose": ("myoElbowPose1D6MRandom-v0", {}),
    "hand_reach_fatigue": ("myoFatiHandReachRandom-v0", dict(fatigue_reset_random=True)),
    "hold_random_fatigue": ("myoFatiHandObjHoldRandom-v0", dict(fatigue_reset_random=True)),
    "hold_fixed_fatigue": ("myoFatiHandObjHoldFixed-v0", dict(fatigue_reset_random=True)),
    "stand_fatigue": ("myoFatiLegStandRandom-v0", dict(fatigue_reset_random=True)),
    "walk_random": ("myoLegWalk-v0", dict(reset_type="random")),
    "walk_random_fatigue": ("myoFatiLegWalk-v0", dict(reset_type="random", fatigue_reset_random=True)),
}
OFFSETS = (0, (1 << 20) - 16, (1 << 32) - 16, P.ENV_LIMIT - 32)      # batches of 32 straddle 2^20 and 2^32; the last ends at the limit
N = 32
_ENVS = {}


def _env(case, n=N):
    if (case, n) not in _ENVS:
        from myosuite_b200 import vec_env
        eid, kw = CASES[case]
        _ENVS[case, n] = vec_env.MyoVecEnv(eid, n, auto_reset=True, **kw)
    return _ENVS[case, n]


def _reset_and_compare(env, label, seed=None, episode=None):
    """reset(seed) (episode counters rewound to 0) or, with seed None, a reset at the current episode counts (set to `episode` first)."""
    import torch
    if seed is None:
        if episode is not None:
            env.t["episode_count"].fill_(episode)
        ep = env.t["episode_count"].cpu().numpy().copy()
        env.reset()
    else:
        ep = np.zeros(env.num_envs, np.int64)
        env.reset(seed=seed)
    torch.cuda.synchronize()
    S = env.get_env_state()
    np.testing.assert_array_equal(S["episode_count"], ep + 1)
    R = P.replay_env(env, env.seed_value, ep)
    P.compare_reset(env, S, R, "%s seed %d env_offset %d" % (label, env.seed_value, env.env_offset))
    return S, R


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_reset_matches_replay(case):
    """Every task branch, at the first and a later episode, for env ids below 2^20, straddling it, and at the top of the domain."""
    env = _env(case, 64 if case.startswith("walk") else N)     # 64 walk envs: both keyframe rows come up
    for off in (0, (1 << 20) - 16, P.ENV_LIMIT - env.num_envs):
        env.env_offset = off
        _, R = _reset_and_compare(env, case, seed=123)
        _reset_and_compare(env, case + " episode 1")
        _reset_and_compare(env, case, episode=4096)
        if "key" in R:
            assert 0 < R["key"].mean() < 1


@pytest.mark.gpu
@pytest.mark.parametrize("env_offset", OFFSETS)
def test_key_boundaries_through_reset(env_offset):
    """Seeds whose halves are at their limits and episode counts at the bits where c2 and c3 split the episode, at each env id boundary."""
    env = _env("hand_pose_fatigue")
    env.env_offset = env_offset
    seen = []
    for seed in (0, (1 << 32) - 1, 1 << 32, (1 << 64) - 1):
        S, _ = _reset_and_compare(env, "seed boundary", seed=seed)
        seen.append(S["fatigue"])
    for episode in (4095, 4096, 1 << 32):
        S, _ = _reset_and_compare(env, "episode %d" % episode, episode=episode)
        seen.append(S["fatigue"])
    for i in range(len(seen)):                                 # every (seed, episode) gives every env its own draws
        for j in range(i):
            assert not np.any(np.all(seen[i] == seen[j], axis=(1, 2))), (i, j)


@pytest.mark.gpu
def test_auto_reset_matches_replay():
    """TimeLimit auto-reset inside the step kernel draws from the stream of the episode count the env had before the step."""
    import torch
    from myosuite_b200 import vec_env
    n = 64
    env = vec_env.MyoVecEnv("myoFatiHandPoseRandom-v0", n, seed=7, env_offset=(1 << 20) - n // 2, fatigue_reset_random=True)
    env.reset(seed=7)
    g = torch.Generator(device="cpu").manual_seed(0)
    env.step((torch.rand(n, env.act_dim, generator=g) * 2 - 1).to(env.device))
    S0 = env.get_env_state()
    forced = np.arange(0, n, 2)
    sc = S0["step_count"].copy(); sc[forced] = env.max_episode_steps - 1
    env.set_env_state({"step_count": sc})
    obs, rew, done, trunc, _ = env.step((torch.rand(n, env.act_dim, generator=g) * 2 - 1).to(env.device))
    torch.cuda.synchronize()
    S = env.get_env_state()
    reset = (trunc | done).cpu().numpy().astype(bool)
    assert np.all(reset[forced])
    np.testing.assert_array_equal(S["episode_count"][reset], S0["episode_count"][reset] + 1)
    np.testing.assert_array_equal(S["step_count"][reset], 0)
    R = P.replay_env(env, 7, S0["episode_count"])
    R = {k: v[reset] for k, v in R.items()}
    P.compare_reset(env, S, R, "auto-reset", rows=reset)


@pytest.mark.gpu
def test_env_2_20_does_not_replay_env_0():
    """Global env 2^20 in its first episode and env 0 in its second drew the same streams while the key ignored env bits 20 and up."""
    import torch
    env = _env("hand_pose_fatigue")
    env.env_offset = 0
    env.reset(seed=5); env.reset(); torch.cuda.synchronize()
    A = env.get_env_state()
    env.env_offset = 1 << 20
    env.reset(seed=5); torch.cuda.synchronize()
    B = env.get_env_state()
    assert np.all(A["episode_count"] == 2) and np.all(B["episode_count"] == 1)
    same = [np.array_equal(A[k][e], B[k][e]) for k in ("fatigue", "qpos", "target") for e in range(env.num_envs)]
    assert not any(same), "%d of %d rows equal" % (sum(same), len(same))


@pytest.mark.gpu
def test_reset_rejects_seeds_and_env_ids_outside_the_key_domain():
    """ctypes would wrap seed 2^64 to 0 and -1 to 2^64 - 1; env ids at or past 2^47 would share streams."""
    import torch
    from myosuite_b200 import make, vec_env
    n = 4
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", n)
    top = P.ENV_LIMIT - n
    for seed in (1 << 64, -1):
        with pytest.raises(ValueError, match=r"seed must be in \[0, 2\*\*64\)"):
            env.reset(seed=seed)
    for off in (-1, top + 1, P.ENV_LIMIT):
        with pytest.raises(ValueError, match="env_offset"):
            env.batch.reset(seed=0, env_offset=off)
    with pytest.raises(ValueError, match="env_offset"):
        vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", n, env_offset=-1).reset()
    # the library refuses them as well
    L = env.batch.L
    for off in (-1, top + 1):
        assert L.myo_batch_reset(env.batch.handle, None, 0, off, None) != 0
        assert b"env_offset" in L.myo_last_error()
    env.batch.reset(seed=(1 << 64) - 1, env_offset=top)                  # the top of the domain is accepted
    torch.cuda.synchronize()
    # the single-env facade goes through the same check
    e1 = make("myoElbowPose1D6MRandom-v0", seed=1).unwrapped
    e1.seed(1 << 64)
    with pytest.raises(ValueError, match=r"seed must be in \[0, 2\*\*64\)"):
        e1.reset()
