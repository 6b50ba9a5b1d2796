"""Host reference of the simulator's random resets: Philox4x32-10 in numpy, the per-(seed, env, episode, lane) stream key of
`philox_init`, the 53-bit uniform of `philox_uniform`, and the order in which each lane of `env_reset` consumes its stream
(myosuite_b200/csrc/myo_b200.cu).  Test infrastructure: tests/test_rng_resets.py pins the generator to the Random123 known-answer
vectors and the device resets to `replay_reset`; `replay_env` / `compare_reset` hold a batch's reset state to the replay (there and
in the in-kernel auto-resets of tests/test_product_parity.py)."""
import numpy as np

M32 = 0xFFFFFFFF
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57          # round multipliers
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85          # key schedule (Weyl) increments
KEY_TAG = 0x4D594F42                                   # "MYOB", xor-ed into c3
ENV_LIMIT = 1 << 47                                    # the key is injective for env < 2^47, episode < 2^44, lane < 32
EPISODE_LIMIT = 1 << 44
LANES = 32


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def philox4x32(ctr, key, rounds=10):
    """Philox4x32-R of counters ctr [..., 4] under keys key [..., 2] (uint32 words); returns uint32 [..., 4].  The 32 x 32 -> 64-bit
    products are exact in uint64."""
    c = [_u64(ctr)[..., i] for i in range(4)]
    k0, k1 = _u64(key)[..., 0], _u64(key)[..., 1]
    for _ in range(rounds):
        p0, p1 = c[0] * np.uint64(PHILOX_M0), c[2] * np.uint64(PHILOX_M1)
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & np.uint64(M32), (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & np.uint64(M32)]
        k0, k1 = (k0 + np.uint64(PHILOX_W0)) & np.uint64(M32), (k1 + np.uint64(PHILOX_W1)) & np.uint64(M32)
    return np.stack(c, axis=-1).astype(np.uint32)


def stream_key(seed, env, episode, lane):
    """philox_init: (ctr [..., 4], key [..., 2]) of the stream of a lane, broadcast over the arguments.
    k0, k1 = seed lo, hi ; c0 = draw counter (0) ; c1 = lane | (env >> 20) << 5 ; c2 = env lo ^ episode << 20 ;
    c3 = env hi ^ episode >> 12 ^ KEY_TAG, every word truncated to 32 bits."""
    seed, env, episode, lane = np.broadcast_arrays(_u64(seed), _u64(env), _u64(episode), _u64(lane))
    m, s20, s12, s32 = np.uint64(M32), np.uint64(20), np.uint64(12), np.uint64(32)
    c1 = (lane | (((env >> s20) & m) << np.uint64(5))) & m
    c2 = (env & m) ^ ((episode << s20) & m)
    c3 = ((env >> s32) & m) ^ ((episode >> s12) & m) ^ np.uint64(KEY_TAG)
    ctr = np.stack([np.zeros_like(c1), c1, c2, c3], axis=-1)
    key = np.stack([seed & m, seed >> s32], axis=-1)
    return ctr, key


def uniform53(a, b):
    """philox_uniform's double in [0, 1) from two output words: ((a >> 5) << 26 | b >> 6) 2^-53."""
    hi, lo = _u64(a) >> np.uint64(5), _u64(b) >> np.uint64(6)
    return ((hi << np.uint64(26)) | lo).astype(np.float64) * 2.0 ** -53


def uniforms(seed, env, episode, lane, count, rounds=10):
    """The first `count` uniforms of each stream, in the order philox_uniform returns them: (o0, o1) then (o2, o3) of counter 0, then of
    counter 1, ...  Shape: broadcast shape of the arguments + (count,)."""
    ctr, key = stream_key(seed, env, episode, lane)
    out = []
    for j in range((count + 1) // 2):
        c = ctr.copy(); c[..., 0] = j                  # the counter never carries into c1: a lane draws far fewer than 2^32 blocks
        o = philox4x32(c, key, rounds)
        out += [uniform53(o[..., 0], o[..., 1]), uniform53(o[..., 2], o[..., 3])]
    return np.stack(out[:count], axis=-1)


def stand_reset_qpos(m, init_qpos, u, joint_random_range=(-0.2, 0.2)):
    """ReachEnvV0.generate_qpos (walk_v0.py:152-167) on given uniforms u ~ U[0, 1), one per joint in joint order: the first qpos
    coordinate of every joint += U(lo, hi) (numpy's low + (high - low) u), clipped to jnt_range whether or not the joint is limited."""
    lo, hi = joint_random_range
    adr = m.jnt_qposadr
    q = np.array(init_qpos, dtype=np.float64, copy=True)
    q[adr] += lo + (hi - lo) * np.asarray(u, dtype=np.float64)
    q[adr] = np.clip(q[adr], m.jnt_range[:, 0], m.jnt_range[:, 1])
    return q


class _LaneDraws:
    """Per-lane cursors over precomputed uniforms [n_env, 32, count]; every env of a reset consumes the same number of draws per lane."""

    def __init__(self, seed, env, episode, count):
        self.u = uniforms(seed, _u64(env)[:, None], _u64(episode)[:, None], np.arange(LANES)[None, :], count)
        self.pos = [0] * LANES

    def __call__(self, lane):
        x = self.u[:, lane, self.pos[lane]]
        self.pos[lane] += 1
        return x


def replay_reset(m, task, seed, env, episode, init_qpos, init_qvel=None, target_range=None, reset_random=False, joint_random=(0.0, 0.0),
                 ntip=0, hold_d=None, fatigue_random=False):
    """env_reset of the global envs `env` [n] at episode counts `episode` [n] (what episode_count held before the reset), lane by lane in
    the kernel's order: walk (random reset), pose, stand joint offsets, reach targets, hold, fatigue.  Returns what the branches taken
    write: qpos [n, nq] always; "key" and "qvel" (walk), "target" [n, nq] (pose, reach), "env_prm" [n, 6] (hold), "fatigue" [n, 3, nu].

    m: the mjModel-like model; task: pose / walk / reach / stand / hold; init_qpos: [nq] ([2, nq] with init_qvel [2, nv] for walk's
    random reset); target_range [nq, 2]; joint_random: the stand range (lo, hi); ntip: reach sites; hold_d: cfg.task_d[0:12]."""
    env, episode = _u64(env).ravel(), _u64(episode).ravel()
    n, nq, njnt, nu = len(env), int(m.nq), int(m.njnt), int(m.nu)
    blocks = lambda k: -(-k // LANES)
    count = 1 + 2 * blocks(nq) + 2 * blocks(njnt) + blocks(njnt) + blocks(3 * ntip) + 1 + 2 * blocks(nu)     # more than any lane uses
    draw = _LaneDraws(seed, env, episode, count)
    init_qpos = np.asarray(init_qpos, dtype=np.float64)
    out = {"qpos": np.broadcast_to(init_qpos if init_qpos.ndim == 1 else init_qpos[0], (n, nq)).copy()}
    if task == "walk" and reset_random:
        # every lane draws one uniform, lane 0's picks the row; then (u1, u2) per coordinate, the height's draws consumed but unused
        key = (np.stack([draw(lane) for lane in range(LANES)])[0] >= 0.5).astype(np.int64)
        q = init_qpos[key]
        for i in range(nq):
            u1, u2 = draw(i % LANES), draw(i % LANES)
            z = np.sqrt(-2.0 * np.log(np.maximum(u1, 1e-300))) * np.cos(6.283185307179586 * u2)
            out["qpos"][:, i] = q[:, i] if i == 2 else q[:, i] + 0.02 * z
        out["key"], out["qvel"] = key, np.asarray(init_qvel, dtype=np.float64)[key]
    if task == "pose":
        # free joints draw nothing; every other joint draws u0 (target) and u1 (qpos), used or not
        target = np.zeros((n, nq))
        for j in range(njnt):
            if m.jnt_type[j] == 0:
                continue
            qa = int(m.jnt_qposadr[j])
            u0, u1 = draw(j % LANES), draw(j % LANES)
            if target_range is not None:
                target[:, qa] = target_range[qa, 0] + u0 * (target_range[qa, 1] - target_range[qa, 0])
            if reset_random:
                out["qpos"][:, qa] = m.jnt_range[j, 0] + u1 * (m.jnt_range[j, 1] - m.jnt_range[j, 0])
        out["target"] = target
    if task == "stand":
        u = np.stack([draw(j % LANES) for j in range(njnt)], axis=1)
        out["qpos"] = np.stack([stand_reset_qpos(m, init_qpos, u[e], tuple(joint_random)) for e in range(n)])
    if task in ("reach", "stand") and target_range is not None:
        target = np.zeros((n, nq))
        for k in range(3 * ntip):
            target[:, k] = target_range[k, 0] + draw(k % LANES) * (target_range[k, 1] - target_range[k, 0])
        out["target"] = target
    if task == "hold":
        # lanes 0-5 draw one uniform each, also when the Fixed variant ignores it: goal = object_init_pos + U(-3 cm, 3 cm), size ~ U(2 cm, 3 cm)
        prm = np.zeros((n, 6))
        for lane in range(6):
            u = draw(lane)
            if not reset_random:
                prm[:, lane] = hold_d[6 + lane]
            elif lane < 3:
                prm[:, lane] = hold_d[3 + lane] + (-0.030 + 0.060 * u)
            else:
                prm[:, lane] = 0.020 + 0.010 * u
        out["env_prm"] = prm
    if fatigue_random:
        # per muscle: nf then ap; MA = nf ap, MR = nf (1 - ap), MF = 1 - nf
        f = np.zeros((n, 3, nu))
        for i in range(nu):
            nf, ap = draw(i % LANES), draw(i % LANES)
            f[:, 0, i], f[:, 1, i], f[:, 2, i] = nf * ap, nf * (1 - ap), 1 - nf
        out["fatigue"] = f
    return out


# ------------------------------------------------------------------------------------------------ a batch's resets against the replay
EPS = np.finfo(np.float64).eps


def replay_env(env, seed, episode, envs=None):
    """replay_reset of the MyoVecEnv batch `env`'s envs `envs` (local indices, all by default) at episode counts `episode`."""
    from myosuite_b200 import abi
    cfg = env.cfg
    envs = np.arange(env.num_envs) if envs is None else np.asarray(envs)
    return replay_reset(env.mj_model, env.task, seed, env.env_offset + envs, episode, env.init_qpos, env.init_qvel,
                        target_range=env.t["target_range"].cpu().numpy(), reset_random=bool(cfg.reset_random),
                        joint_random=(cfg.joint_random[0], cfg.joint_random[1]), ntip=len(env.tip_names),
                        hold_d=list(cfg.task_d)[:12], fatigue_random=cfg.muscle_condition == abi.COND_FATIGUE and cfg.fatigue_reset == 1)


def _within(got, want, tol, label):
    excess = np.abs(got - want) - tol
    assert np.all(excess <= 0), "%s: %d entries off, worst by %.3g beyond %.3g at %s" % (
        label, int(np.sum(excess > 0)), excess.max(), np.broadcast_to(tol, excess.shape).flat[np.argmax(excess)], np.unravel_index(np.argmax(excess), excess.shape))


def _span_tol(lo, hi):
    """lo + u (hi - lo), with or without an FMA: within 4 eps max(|lo|, |hi|) of numpy's rounding."""
    return 4 * EPS * np.maximum(np.abs(lo), np.abs(hi))


def compare_reset(env, S, R, label, rows=slice(None)):
    """Device state S of the envs `rows` against replay R (already restricted to those envs): bit for bit where the kernel's expression
    admits no contraction (fatigue state, stand joint offsets, walk keyframe row, untouched init_qpos), else to a few ulps."""
    m, cfg, task = env.mj_model, env.cfg, env.task
    tr = env.t["target_range"].cpu().numpy()
    if "fatigue" in R:
        np.testing.assert_array_equal(S["fatigue"][rows], R["fatigue"], err_msg=label + ": fatigue state")
    if "key" in R:                                            # walk's random reset
        qv = S["qvel"][rows]
        key = np.where(np.all(qv == env.init_qvel[1], axis=1), 1, np.where(np.all(qv == env.init_qvel[0], axis=1), 0, -1))
        np.testing.assert_array_equal(key, R["key"], err_msg=label + ": walk keyframe row")
        _within(S["qpos"][rows], R["qpos"], 1e-15, label + ": walk qpos")
    elif task == "pose" and cfg.reset_random:
        free = m.jnt_type == 0
        adr = m.jnt_qposadr[~free]
        _within(S["qpos"][rows][:, adr], R["qpos"][:, adr], _span_tol(m.jnt_range[~free, 0], m.jnt_range[~free, 1]), label + ": pose qpos")
    else:                                                     # stand offsets (numpy's rounding, no contraction) or untouched init_qpos
        np.testing.assert_array_equal(S["qpos"][rows], R["qpos"], err_msg=label + ": qpos")
    if "target" in R:
        cols = m.jnt_qposadr[m.jnt_type != 0] if task == "pose" else np.arange(3 * int(cfg.task_i[0]))
        _within(S["target"][rows][:, cols], R["target"][:, cols], _span_tol(tr[cols, 0], tr[cols, 1]), label + ": target")
    if "env_prm" in R:
        got = S["env_prm"][rows][:, :6]
        if cfg.reset_random:
            obj = np.array(cfg.task_d[3:6])
            lo, hi = np.concatenate([obj - 0.03, [0.02] * 3]), np.concatenate([obj + 0.03, [0.03] * 3])
            _within(got, R["env_prm"], _span_tol(lo, hi), label + ": hold goal / size")
        else:
            np.testing.assert_array_equal(got, R["env_prm"], err_msg=label + ": hold fixed goal / size")
