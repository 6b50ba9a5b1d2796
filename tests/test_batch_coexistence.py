"""Batches that share one process: calls on one batch must never change another batch's results or whether its launches succeed.

Users keep a training batch and a make(id) evaluation env in one process, hold several models at once, and read, invert, roll out or
linearise one batch while another steps.  Every case here compares a batch with its twin (same id, size, seed and calls: bit-identical
results, as the determinism tests rely on) after other batches have been created and used in between, with torch.equal on every
output of the call and every bound tensor.

(a) Smaller batches leave larger ones launchable: twins A and B of a victim at a benchmarked launch shape; A runs an entry point, then
    smaller batches of the same library (the elbow, the victim's own id at one env and at 64 envs with a one-contact slice) and one of
    the other row storage are created and call every entry point; then B runs the entry point.  The dynamic shared-memory limit of a
    kernel belongs to the device context, not to a batch: a set-up that sets it to its own, smaller need makes the next launch of every
    larger batch fail with "invalid argument".
(b) A seeded random schedule of calls over a pool of batches of several models, sizes, contact capacities and both row storages
    (deleting and creating batches midway, and two batches on one device model) against each batch's calls replayed on a fresh twin.
(c) Streams and host threads: a batch built and driven on a side stream, two batches on two side streams with interleaved launches,
    and two host threads driving one batch each on its own stream, against default-stream twins."""
import gc
import threading

import numpy as np
import pytest

SEED = 23
HAND, HOLD, STAND, ELBOW = "myoHandPoseRandom-v0", "myoHandObjHoldRandom-v0", "myoLegStandRandom-v0", "myoElbowPose1D6MRandom-v0"
WALK, TORSO = "myoFatiLegWalk-v0", "myoTorsoPoseFixed-v0"
# victim -> (env id, n_env, constructor kwargs): the launch shapes of test_product_parity.py (hand: launch_bounds(448) kernel, 11 warps,
# load-sorted map; hold: launch_bounds(320) kernel, 8 warps; stand: 6 warps; the hand on f64 rows: the verification library)
VICTIMS = {"hand": (HAND, 4096, {}), "hold": (HOLD, 2048, {}), "stand": (STAND, 2048, {}), "hand_f64": (HAND, 4096, {"row_storage": "f64"})}
ENTRIES = ("reset", "step", "step_taps", "forward_debug", "refresh_obs", "data", "inverse", "rollout", "ik", "jac_site", "transition_fd")


# ----------------------------------------------------------------------------- entry points with inputs from a per-batch generator
def _sites(m):
    return [0, m.nsite // 2, m.nsite - 1]


def _call(env, entry, g):
    """Run one entry point of MyoVecEnv `env` with inputs drawn from the CPU generator g; returns clones of every output of the call."""
    import torch
    m, n, dev = env.mj_model, env.num_envs, env.device
    rand = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    if entry == "reset":
        obs, _ = env.reset(seed=int(torch.randint(0, 1 << 30, (1,), generator=g)))
        out = {"obs": obs}
    elif entry in ("step", "step_taps"):
        obs, rew, done, trunc, info = env.step((rand(n, m.nu) * 2 - 1).float().to(dev))
        out = dict(obs=obs, reward=rew, done=done, truncated=trunc, **{k: v for k, v in info.items() if v is not None})
    elif entry == "forward_debug":
        env.forward_debug(rand(n, m.nu).numpy(), 2)
        out = {}
    elif entry == "refresh_obs":
        out = dict(zip(("obs", "reward", "done"), env.refresh_obs()))
    elif entry == "data":
        out = env.data()
    elif entry == "inverse":
        out = env.inverse((rand(n, m.nv) * 2 - 1).to(dev), fields=env.INVERSE_FIELDS)
    elif entry == "rollout":
        out = env.rollout(rand(n, 3, m.nu).to(dev), substeps=2, fields=env.ROLLOUT_FIELDS)
    elif entry == "ik":
        s = _sites(m)
        target = (env.jac_site(s)[2] + 0.02 * (rand(n, len(s), 3) * 2 - 1).to(dev)).contiguous()
        out = env.ik(s, target, fields=env.IK_FIELDS)
    elif entry == "jac_site":
        out = dict(zip(("jacp", "jacr", "site_xpos", "site_xmat"), env.jac_site(_sites(m))))
    elif entry == "transition_fd":
        out = env.transition_fd(rand(n, m.nu).to(dev), fields=("A", "B", "overflow"))
    else:
        raise KeyError(entry)
    return {k: v.clone() for k, v in out.items()}


def _bits(t):
    import torch
    return t.view({torch.float64: torch.int64, torch.float32: torch.int32}[t.dtype]) if t.is_floating_point() else t


def _state(env):
    """Every bound tensor of the batch (state, task buffers, obs / reward / done, final_obs, returns, overflow, parity taps), cloned.
    Not the phase cycle counters of the debug kernel: clock readings, which no two runs share."""
    import torch
    return {k: v.clone() for k, v in env.t.items() if isinstance(v, torch.Tensor) and k != "tap_phase_cycles"}


def _assert_same(got, ref, what):
    """bit for bit (NaN rows of final_obs included)"""
    import torch
    assert set(got) == set(ref), (what, sorted(set(got) ^ set(ref)))
    for k in ref:
        assert got[k].shape == ref[k].shape and got[k].dtype == ref[k].dtype, (what, k)
        assert torch.equal(_bits(got[k]), _bits(ref[k])), "%s: %s differs from the twin's" % (what, k)


def _gen(seed):
    import torch
    return torch.Generator(device="cpu").manual_seed(seed)


def _new(eid, n, **kw):
    from myosuite_b200 import vec_env
    if n == 1:
        return vec_env.MyoEnv(eid, seed=SEED, **kw).vec          # the single-env facade's batch (its constructor resets)
    return vec_env.MyoVecEnv(eid, n, seed=SEED, **kw)


def _warm(env, entry=None, steps=3):
    """reset, a few steps, then (when given) one call of `entry`, so that its set-up happens here: identical for twins"""
    import torch
    g = _gen(SEED)
    env.reset(seed=SEED)
    for _ in range(steps):
        env.step((torch.rand(env.num_envs, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
    if entry is not None:
        _call(env, entry, _gen(SEED + 1))


# ----------------------------------------------------------------------------- (a) smaller batches leave larger ones launchable
def _intruders(eid, rows):
    """Smaller batches of the victim's library, the last one the smallest model, and one batch of the other row storage (a separate
    library: a control).  Returns [(name, env, same_library)]."""
    other = "p48" if rows == "f64" else "f64"
    return [("%s n 64 maxcon 1" % eid, lambda: _new(eid, 64, maxcon=1, row_storage=rows), True),
            ("%s single env" % eid, lambda: _new(eid, 1, row_storage=rows), True),
            ("elbow n 4096", lambda: _new(ELBOW, 4096, row_storage=rows), True),
            ("%s single env, %s rows" % (eid, other), lambda: _new(eid, 1, row_storage=other), False),
            ("elbow single env", lambda: _new(ELBOW, 1, row_storage=rows), True)]


@pytest.mark.gpu
@pytest.mark.parametrize("victim,entry", [(v, e) for v in VICTIMS for e in ENTRIES])
def test_smaller_batches_leave_larger_ones_launchable(victim, entry):
    import torch
    eid, n, kw = VICTIMS[victim]
    rows = kw.get("row_storage", "p48")
    taps = entry == "step_taps"
    A, B = _new(eid, n, taps=taps, **kw), _new(eid, n, taps=taps, **kw)
    _warm(A, entry); _warm(B, entry)
    smem = A.batch.launch_info()["smem_bytes"]
    out_a = _call(A, entry, _gen(SEED + 2))
    torch.cuda.synchronize()
    state_a = _state(A)
    lowered = []
    for name, make, same_lib in _intruders(eid, rows):
        env = make()
        for e in ENTRIES:
            if e != "step_taps":
                _call(env, e, _gen(SEED + 3))
        if same_lib:
            lowered.append((name, env.batch.launch_info()["smem_bytes"]))
        del env
    torch.cuda.synchronize()
    # the precondition of the case: at a limit set to each batch's own need, these set-ups leave it below what the victim launches with
    assert all(s < smem for _, s in lowered), (smem, lowered)
    out_b = _call(B, entry, _gen(SEED + 2))          # raised MyoError "cudaGetLastError(): invalid argument" where set-up lowered the limit
    torch.cuda.synchronize()
    _assert_same(out_b, out_a, "%s %s output" % (victim, entry))
    _assert_same(_state(B), state_a, "%s %s state" % (victim, entry))


# ----------------------------------------------------------------------------- (b) interleaved schedule against isolated twins
POOL = {"hand": (HAND, 4096, {}), "hold": (HOLD, 2048, {}), "elbow": (ELBOW, 4096, {}), "walk": (WALK, 2048, {}), "torso": (TORSO, 661, {}),
        "hand_f64": (HAND, 512, {"row_storage": "f64"}), "hand_maxcon1": (HAND, 256, {"maxcon": 1}),
        "single_hold": (HOLD, 1, {}), "single_elbow": (ELBOW, 1, {})}
LATE = {"stand": (STAND, 2048, {}), "single_hand_f64": (HAND, 1, {"row_storage": "f64"})}     # created midway
DROPPED = ("hold", "single_elbow")                                                              # deleted midway
SCHEDULE_ENTRIES = tuple(e for e in ENTRIES if e != "step_taps")
NCALL = 200


def _sibling(env):
    """A second batch on env's device model (same cfg), bound to fresh copies of env's tensors: a MyoVecEnv view of it."""
    import copy
    from myosuite_b200 import abi
    sib = copy.copy(env)
    sib.batch = abi.Batch(env.dev_model, env.device_index, env.num_envs, env.cfg)
    t = {k: v.clone() for k, v in env.t.items() if k not in ("obs_full", "final_obs_full")}
    sib.batch.bind(**t)
    t["obs_full"] = t["obs"]
    if "final_obs" in t:
        t["final_obs_full"] = t["final_obs"]
    sib.t, sib._data, sib._inv = t, {}, {}
    return sib


@pytest.mark.gpu
def test_interleaved_schedule_matches_isolated_twins():
    import torch
    rng = np.random.default_rng(SEED)
    spec = dict(POOL, **LATE)
    spec["hand_f64_sibling"] = spec["hand_f64"]           # a second batch on the hand_f64 batch's device model
    pool = {k: _new(eid, n, **kw) for k, (eid, n, kw) in POOL.items()}
    pool["hand_f64_sibling"] = _sibling(pool["hand_f64"])
    gens = {k: _gen(SEED + 100 + i) for i, k in enumerate(spec)}
    calls = {k: [] for k in spec}                                             # per batch: (entry, outputs) in call order
    final = {}                                                                # per batch: every bound tensor after its last call
    for i in range(NCALL):
        if i == NCALL // 2:
            for k in DROPPED + ("hand_f64",):          # (hand_f64's sibling keeps the device model alive and goes on)
                final[k] = _state(pool[k])
                del pool[k]
            gc.collect()
            pool.update({k: _new(eid, n, **kw) for k, (eid, n, kw) in LATE.items()})
        k = sorted(pool)[rng.integers(len(pool))]
        e = SCHEDULE_ENTRIES[rng.integers(len(SCHEDULE_ENTRIES))]
        calls[k].append((e, _call(pool[k], e, gens[k])))
    torch.cuda.synchronize()
    final.update({k: _state(v) for k, v in pool.items()})
    del pool
    gc.collect()
    used = 0
    for k, seq in calls.items():           # each batch's own calls on a fresh twin, one batch at a time
        eid, n, kw = spec[k]
        twin, g = _new(eid, n, **kw), _gen(SEED + 100 + list(spec).index(k))
        for j, (e, out) in enumerate(seq):
            _assert_same(_call(twin, e, g), out, "%s call %d (%s)" % (k, j, e))
        _assert_same(_state(twin), final[k], "%s final state" % k)
        used += bool(seq)
        del twin
        gc.collect()
    assert used >= len(spec) - 1, {k: len(v) for k, v in calls.items()}
    print("\ninterleaved schedule: %d calls over %d batches, %s" % (NCALL, len(spec), {k: len(v) for k, v in calls.items()}))


# ----------------------------------------------------------------------------- (c) streams and host threads
def _drive(env, seed, nstep=20):
    """Every entry point once, then nstep steps: the calls' outputs in order"""
    g, outs = _gen(seed), []
    for e in SCHEDULE_ENTRIES:
        outs.append(_call(env, e, g))
    for _ in range(nstep):
        outs.append(_call(env, "step", g))
    return outs


def _reference(eid, n, kw, seed, nstep=20):
    import torch
    env = _new(eid, n, **kw)
    outs = _drive(env, seed, nstep)
    torch.cuda.synchronize()
    return outs, _state(env)


def _assert_run(outs, state, ref, what):
    ref_outs, ref_state = ref
    assert len(outs) == len(ref_outs)
    for j, (o, r) in enumerate(zip(outs, ref_outs)):
        _assert_same(o, r, "%s call %d" % (what, j))
    _assert_same(state, ref_state, "%s final state" % what)


@pytest.mark.gpu
def test_batch_built_and_driven_on_a_side_stream():
    import torch
    ref = _reference(HAND, 4096, {}, SEED + 7)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        env = _new(HAND, 4096)               # set-up, the first call of every entry point (the readout's set-up too) on the side stream
        outs = _drive(env, SEED + 7)
    s.synchronize()
    _assert_run(outs, _state(env), ref, "side stream")


@pytest.mark.gpu
def test_two_batches_on_two_streams_interleaved():
    import torch
    cases = [(HAND, 4096, {}), (HOLD, 2048, {})]
    refs = [_reference(eid, n, kw, SEED + 8 + i) for i, (eid, n, kw) in enumerate(cases)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    envs, gens, outs = [], [_gen(SEED + 8), _gen(SEED + 9)], [[], []]
    for (eid, n, kw), s in zip(cases, streams):
        with torch.cuda.stream(s):
            envs.append(_new(eid, n, **kw))
    plan = list(SCHEDULE_ENTRIES) + ["step"] * 20            # the order of _drive; launches alternate between the streams, unsynchronised
    for e in plan:
        for i in range(2):
            with torch.cuda.stream(streams[i]):
                outs[i].append(_call(envs[i], e, gens[i]))
    torch.cuda.synchronize()
    for i in range(2):
        _assert_run(outs[i], _state(envs[i]), refs[i], "stream %d" % i)


@pytest.mark.gpu
def test_two_host_threads_each_driving_a_batch():
    import torch
    cases = [(HAND, 4096, {}), (STAND, 2048, {})]
    refs = [_reference(eid, n, kw, SEED + 10 + i) for i, (eid, n, kw) in enumerate(cases)]
    results, errors = [None, None], []
    start = threading.Barrier(2)

    def worker(i):
        try:
            eid, n, kw = cases[i]
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                env = _new(eid, n, **kw)
                start.wait()                   # the two threads' calls overlap (ctypes releases the GIL inside the library)
                outs = _drive(env, SEED + 10 + i)
            s.synchronize()
            results[i] = (outs, _state(env))
        except BaseException as ex:           # re-raised in the main thread
            errors.append(ex)
            start.abort()

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    for i in range(2):
        _assert_run(results[i][0], results[i][1], refs[i], "thread %d" % i)
