"""GPU parity tests proper: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Tolerances: north_star asks <= 1e-5 relative on qacc and muscle force; the two f64 implementations agree to
~1e-10, so the tests assert 1e-7 (headroom for FMA / summation-order differences).  Contact pair lists are
compared bit-exactly (integer indexing)."""
import os

import numpy as np
import pytest

from parity_helpers import _in_regime, _oracle_for, _states, relerr

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "pylogic.npz"))
RTOL = 1e-7
# qacc passes through the constraint solve.  The product library STORES the contact Jacobian rows as the upper 48 bits of the f64 value
# (36 mantissa bits, 1.5e-11 relative; all arithmetic stays f64; DESIGN.md section 3) -- plain f32 storage was measured to move qacc by up
# to 9e-5 on stiff multi-contact states and was rejected.  The verification build of the same source (row_storage="f64",
# abi.lib("f64rows")) stores plain doubles.  Every physics parity test below runs on BOTH with the SAME tolerances: 1e-7 on one forward
# pass from sampled states, 1e-6 on states reached mid-episode (bounded by the oracle's own 1e-6 inverse-wrap tolerance).
ROWS = ["p48", "f64"]
QACC_TOL = {r: {"fwd": 1e-7, "mid": 1e-6, "legs": 1e-6} for r in ROWS}
WORST = {}


def _note(test, rows, v):
    k = (test, rows); WORST[k] = max(WORST.get(k, 0.0), float(v)); return v


@pytest.fixture(scope="module")
def envs():
    from myosuite_b200 import vec_env
    yield {(eid, rows): vec_env.MyoVecEnv(eid, 64, taps=True, maxcon=48, row_storage=rows) for eid in ("myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0") for rows in ROWS}
    print("\nworst qacc deviation per test / row storage: " + "; ".join("%s[%s] %.1e" % (k[0], k[1], v) for k, v in sorted(WORST.items())))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("eid", ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0"])
def test_forward_parity(envs, eid, rows):
    """qacc, actuator_force, tendon length, mass matrix, smooth force and the contact list of one mj_forward."""
    import torch
    from oracle.oracle_py import Oracle
    env = envs[eid, rows]; m = env.mj_model; n = env.num_envs
    qpos, qvel, act, ctrl = _states(m, n, np.random.default_rng(11))
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy() for k, v in env.t.items() if k.startswith("tap_")}
    o = Oracle(env.I, env.D)
    pmi = env.prog_info["pair_model_index"]
    total_con = checked = 0
    for e in range(n):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        if not _in_regime(o, m):
            continue
        checked += 1
        assert _note("forward/" + eid[3:8], rows, relerr(t["tap_qacc"][e], o.f("qacc"))) < QACC_TOL[rows]["fwd"]
        assert relerr(t["tap_actuator_force"][e], o.f("actuator_force")) < RTOL
        assert relerr(t["tap_ten_length"][e], o.f("actuator_length")) < 1e-10
        assert relerr(t["tap_qM"][e], o.f("qM")) < 1e-8
        assert relerr(t["tap_qfrc_smooth"][e], o.f("qfrc_smooth")) < RTOL
        nc = int(t["tap_ncon"][e, 0])
        got = [pmi[p] for p in t["tap_contact_pair"][e][:nc]]
        exp = [int(p) for p in o.i("con_pair") if int(p) in set(pmi)]
        # integer contact-pair indexing, bit-exact AND in order: the kernel merges its two collider passes into model pair order
        # (the order MuJoCo reports contacts in); the oracle lists plain pair order
        assert got == exp
        od = [d for p, d in zip(o.i("con_pair"), o.f("con_dist")) if int(p) in set(pmi)]
        np.testing.assert_allclose(t["tap_contact_dist"][e][:nc], od, rtol=1e-7, atol=1e-11)
        assert t["tap_ncon"][e, 3] == 0                      # no contact-capacity overflow
        total_con += nc
    assert checked >= n // 2      # (random joint configurations incl. 2 % beyond the limits: many deep finger-pad overlaps; see test_regime_rate_on_rollouts)
    if m.nv > 1:
        assert total_con > 0                                 # the hand batch really exercised contacts


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("eid", ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0"])
def test_rollout_parity(envs, eid, rows):
    """10 chained mj_step's with a fixed ctrl (one control step of robot.py:901-905)."""
    import torch
    from oracle.oracle_py import Oracle
    env = envs[eid, rows]; m = env.mj_model; n = env.num_envs
    qpos, qvel, act, ctrl = _states(m, n, np.random.default_rng(12), overshoot=0.0)
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 10); torch.cuda.synchronize()
    gq, gv, ga = env.t["qpos"].cpu().numpy(), env.t["qvel"].cpu().numpy(), env.t["act"].cpu().numpy()
    o = Oracle(env.I, env.D)
    checked = 0
    for e in range(16):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e])
        ok = True
        for _ in range(10):
            o.step(1); ok = ok and _in_regime(o, m)
        if not ok:
            continue
        checked += 1
        # substeps 2..10 warm-start the inverse-wrap root (converged to 1e-10) while the oracle keeps MuJoCo's cold start with its
        # 1e-6 residual tolerance: agreement is bounded by that tolerance, still far inside the north-star's 1e-5
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=1e-7)
        assert relerr(gv[e], o.f("qvel")) < 1e-5
        np.testing.assert_allclose(ga[e, :m.na], o.f("act"), rtol=0, atol=1e-12)
    assert checked >= 8
    assert int(env.t["tap_ncon"][:, 3].sum().item()) == 0          # no contact-capacity overflow in this batch (maxcon=48)


@pytest.mark.parametrize("rows", ROWS)
def test_elbow_joint_limit_rows(envs, rows):
    """Edge cases of the one-sided limit row: exactly at, just inside, beyond both ends of the range."""
    import torch
    from oracle.oracle_py import Oracle
    env = envs["myoElbowPose1D6MRandom-v0", rows]; m = env.mj_model; n = env.num_envs
    lo, hi = m.jnt_range[0]
    q = np.linspace(lo - 0.1, hi + 0.1, n)[:, None]
    q[0], q[1], q[2], q[3] = lo, hi, lo - 1e-9, hi + 1e-9
    rng = np.random.default_rng(5)
    qvel, act, ctrl = rng.normal(0, 3, (n, 1)), rng.uniform(0, 1, (n, 6)), rng.uniform(0, 1, (n, 6))
    env.set_state(qpos=q, qvel=qvel, act=act); env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy() for k, v in env.t.items() if k.startswith("tap_")}
    o = Oracle(env.I, env.D)
    for e in range(n):
        o.reset(); o.set(qpos=q[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        assert int(t["tap_ncon"][e, 1]) == o.nefc
        assert _note("limit_rows", rows, relerr(t["tap_qacc"][e], o.f("qacc"))) < QACC_TOL[rows]["fwd"]
    assert t["tap_ncon"][:, 1].max() == 1 and t["tap_ncon"][0, 1] == 0 and t["tap_ncon"][2, 1] == 1


@pytest.mark.parametrize("eid,tag,thd", [("myoElbowPose1D6MRandom-v0", "elbow", 0.175), ("myoHandPoseRandom-v0", "hand", 0.7)])
def test_env_step_obs_reward_vs_oracle(eid, tag, thd):
    """Full env.step through the public batched API vs (env_oracle + physics oracle), auto-reset off."""
    import torch
    from myosuite_b200 import vec_env
    from oracle import env_oracle
    from oracle.oracle_py import Oracle
    n = 32
    env = vec_env.MyoVecEnv(eid, n, auto_reset=False, maxcon=48)
    m = env.mj_model
    rng = np.random.default_rng(21)
    qpos, qvel, act, _ = _states(m, n, rng, overshoot=0.0, vel=0.5)
    target = np.stack([rng.uniform(env.t["target_range"][:, 0].cpu().numpy(), env.t["target_range"][:, 1].cpu().numpy()) for _ in range(n)])
    env.set_state(qpos=qpos, qvel=qvel, act=act, target=target)
    oracles = []
    for e in range(n):
        o = Oracle(env.I, env.D); o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e]); oracles.append(o)
    good = [True] * n
    for step in range(3):
        a = rng.uniform(-1, 1, (n, m.nu)).astype(np.float32)
        obs, rew, done, trunc, info = env.step(torch.as_tensor(a, device=env.device)); torch.cuda.synchronize()
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for e in range(n):
            o = oracles[e]
            ctrl_e = env_oracle.action_to_ctrl(a[e].astype(np.float64)); o.set(ctrl=ctrl_e)
            for _ in range(env.n_frames):
                o.step(1); good[e] = good[e] and _in_regime(o, m)
            if not good[e]:
                continue
            exp_obs = env_oracle.pose_obs(o.f("qpos"), o.f("qvel"), o.f("act"), target[e], env.dt)
            np.testing.assert_allclose(obs[e], exp_obs, rtol=2e-6, atol=2e-6)
            r = env_oracle.pose_reward(o.f("qpos"), o.f("act"), target[e], thd)
            assert rew[e] == pytest.approx(r["dense"], rel=1e-5, abs=1e-5) and bool(done[e]) == bool(r["done"])
    assert sum(good) >= n // 2
    assert np.all(env.t["step_count"].cpu().numpy() == 3)
    assert np.allclose(env.t["time"].cpu().numpy(), 3 * env.dt)


def test_pose_obs_reward_golden_from_reference():
    """obs / reward / done produced by the kernel epilogue on states whose expected values were computed by the
    reference's own PoseEnvV0.get_obs_dict / get_reward_dict / obsdict2obsvec (tests/golden/make_golden.py)."""
    import torch
    from myosuite_b200 import vec_env
    for eid, tag in (("myoElbowPose1D6MRandom-v0", "elbow"), ("myoHandPoseRandom-v0", "hand")):
        q, v, a, tg = (G["pose_%s_%s" % (tag, k)] for k in ("qpos", "qvel", "act", "target"))
        env = vec_env.MyoVecEnv(eid, len(q), auto_reset=False)
        env.set_state(qpos=q, qvel=v, act=a, target=tg)
        env.refresh_obs(); torch.cuda.synchronize()
        np.testing.assert_array_equal(env.t["obs"].cpu().numpy(), G["pose_%s_obs" % tag])      # float32, bit-exact
        np.testing.assert_allclose(env.t["reward"].cpu().numpy(), G["pose_%s_rwd_dense" % tag], rtol=2e-6, atol=2e-6)
        np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), G["pose_%s_rwd_done" % tag].astype(bool))


def test_fatigue_variant_vs_reference_golden():
    """myoFati*: the device-side 3CC-r update against the golden MA/MR/MF produced by the reference's fatigue.py
    (same actions as tests/golden/make_golden.py BaseV0.step run: 39 muscles, dt=0.02)."""
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv("myoFatiHandPoseRandom-v0", 2, auto_reset=False)
    A = G["step_action_fatigue"].astype(np.float32)   # float32 is what crosses the ABI
    from oracle import env_oracle
    f = env_oracle.Fatigue(39, dt=0.02)
    for k in range(len(A)):
        a = torch.as_tensor(np.stack([A[k], A[k]]), device=env.device)
        env.step(a)
        exp = f.compute_act(env_oracle.action_to_ctrl(A[k].astype(np.float64)))
        torch.cuda.synchronize()
        got = env.t["fatigue"][0].cpu().numpy()
        np.testing.assert_allclose(got, np.stack(exp), rtol=1e-12, atol=1e-15)
    # and the chain agrees with the reference golden to float32-action round-off
    np.testing.assert_allclose(env.t["fatigue"][0, 0].cpu().numpy(), G["step_ctrl_fatigue"][-1], rtol=0, atol=5e-6)


@pytest.mark.parametrize("rows", ROWS)
def test_legs_physics_parity(rows):
    """myolegs (config 4 model): free joint + quaternion integration, 14 polynomial joint equalities, foot/floor plane contacts
    (capsule and ellipsoid), 80 muscles; physics only (the Walk task logic is not on the device yet)."""
    import torch
    from myosuite_b200 import vec_env
    from oracle.oracle_py import Oracle
    n = 16
    env = vec_env.MyoVecEnv.from_model("myolegs", n, taps=True, maxcon=48, row_storage=rows)
    m = env.mj_model
    rng = np.random.default_rng(4)
    qpos = np.tile(m.key_qpos[0], (n, 1)); qpos[:, 2] -= rng.uniform(0.0, 0.03, n)        # standing keyframe, feet pressed into the floor a little
    qpos[:, 7:] += rng.normal(0, 0.02, (n, m.nq - 7))
    qvel = rng.normal(0, 0.3, (n, m.nv)); act = rng.uniform(0, 1, (n, m.na)); ctrl = rng.uniform(0, 1, (n, m.nu))
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy() for k, v in env.t.items() if k.startswith("tap_")}
    o = Oracle(env.I, env.D)
    ncon = 0
    for e in range(n):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        assert int(t["tap_ncon"][e, 1]) == o.nefc and o.nefc >= 14
        assert _note("legs", rows, relerr(t["tap_qacc"][e], o.f("qacc"))) < QACC_TOL[rows]["legs"]
        assert relerr(t["tap_actuator_force"][e], o.f("actuator_force")) < RTOL
        assert relerr(t["tap_qM"][e], o.f("qM")) < 1e-8
        ncon += o.ncon
    assert ncon > 0
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.forward_debug(ctrl, 10); torch.cuda.synchronize()
    gq, gv = env.t["qpos"].cpu().numpy(), env.t["qvel"].cpu().numpy()
    for e in range(4):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.step(10)
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=1e-8)
        assert relerr(gv[e], o.f("qvel")) < 1e-5
        assert abs(np.linalg.norm(gq[e, 3:7]) - 1) < 1e-12                                   # quaternion stays normalised


TG = np.load(os.path.join(os.path.dirname(__file__), "golden", "tasks.npz"))


def test_walk_task_golden_from_reference():
    """myoLegWalk-v0 obs (403) / reward / done produced by the kernel on states whose expected values come from the reference's own
    WalkEnvV0 methods (tests/golden/make_golden_tasks.py)."""
    import torch
    from myosuite_b200 import vec_env
    n = len(TG["walk_qpos"])
    env = vec_env.MyoVecEnv("myoLegWalk-v0", n, auto_reset=False)
    assert env.obs_dim == 403 and env.act_dim == 80 and env.dt == pytest.approx(0.01) and env.max_episode_steps == 1000
    env.set_state(qpos=TG["walk_qpos"], qvel=TG["walk_qvel"], act=TG["walk_act"])
    env.t["step_count"][:] = torch.as_tensor(TG["walk_steps"].astype(np.int32), device=env.device)
    env.refresh_obs(); torch.cuda.synchronize()
    np.testing.assert_allclose(env.t["obs"].cpu().numpy(), TG["walk_obs"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(env.t["reward"].cpu().numpy(), TG["walk_dense"], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), TG["walk_done"].astype(bool))


def test_walk_env_step_and_reset_vs_oracle():
    """Full myoFatiLegWalk-v0 control steps (fatigue + 10 substeps with equality/contact constraints + Walk obs) vs the oracles."""
    import torch
    from myosuite_b200 import vec_env
    from oracle import env_oracle
    from oracle.oracle_py import Oracle
    n = 4
    env = vec_env.MyoVecEnv("myoFatiLegWalk-v0", n, auto_reset=False, maxcon=48)
    m = env.mj_model
    obs0, _ = env.reset(seed=3); torch.cuda.synchronize()
    np.testing.assert_allclose(env.t["qpos"].cpu().numpy(), np.tile(m.key_qpos[2], (n, 1)), atol=1e-12)      # reset_type "init": keyframe 2 (walk_v0.py:348-349)
    np.testing.assert_allclose(env.t["qvel"].cpu().numpy(), np.tile(m.key_qvel[2], (n, 1)), atol=1e-12)
    ids = env_oracle.walk_ids(m)
    cfg = dict(hip_period=100, min_height=0.8, max_rot=0.8, target_x_vel=0.0, target_y_vel=1.2, target_rot=m.key_qpos[0][3:7])
    oracles, fats = [], []
    for e in range(n):
        o = Oracle(env.I, env.D); o.reset(); o.set(qpos=m.key_qpos[2], qvel=m.key_qvel[2]); oracles.append(o); fats.append(env_oracle.Fatigue(m.nu, dt=env.dt))
    rng = np.random.default_rng(8)
    for step in range(3):
        a = rng.uniform(-1, 1, (n, m.nu)).astype(np.float32)
        obs, rew, done, trunc, _ = env.step(torch.as_tensor(a, device=env.device)); torch.cuda.synchronize()
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for e in range(n):
            o = oracles[e]
            env_oracle.env_step(o, a[e].astype(np.float64), env.n_frames, fatigue=fats[e])
            state = (o.f("qpos").copy(), o.f("qvel").copy(), o.f("act").copy(), o.f("ctrl").copy())
            o.set(ctrl=np.zeros(m.nu)); o.forward()                       # the reference's observed data: forward with ctrl = 0
            exp_obs, r = env_oracle.walk_obs_reward(m, o, step, env.dt, ids, cfg)
            o.set(qpos=state[0], qvel=state[1], act=state[2], ctrl=state[3])
            np.testing.assert_allclose(obs[e], exp_obs, rtol=1e-4, atol=2e-5)
            assert rew[e] == pytest.approx(r["dense"], rel=1e-4, abs=1e-4) and bool(done[e]) == bool(r["done"])


def test_hold_task_golden_and_reset():
    import torch
    from myosuite_b200 import vec_env
    n = len(TG["hold_qpos"])
    env = vec_env.MyoVecEnv("myoHandObjHoldRandom-v0", n, auto_reset=False)
    assert env.obs_dim == 91 and env.max_episode_steps == 75
    env.set_state(qpos=TG["hold_qpos"], qvel=TG["hold_qvel"], act=TG["hold_act"])
    env.t["env_prm"][:, :3] = torch.as_tensor(TG["hold_goal"], device=env.device)
    env.refresh_obs(); torch.cuda.synchronize()
    np.testing.assert_allclose(env.t["obs"].cpu().numpy(), TG["hold_obs"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(env.t["reward"].cpu().numpy(), TG["hold_dense"], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), TG["hold_done"].astype(bool))
    # ObjHoldRandomEnvV0.reset: goal within +-3 cm of the object's initial position, object radii in [2, 3] cm, hand open with qpos[0] = -1.5
    env.reset(seed=5); torch.cuda.synchronize()
    prm = env.t["env_prm"].cpu().numpy(); q = env.t["qpos"].cpu().numpy()
    obj0 = np.array([-.235, -.51, 1.450])
    assert np.all(np.abs(prm[:, :3] - obj0) <= 0.03 + 1e-12) and np.all(prm[:, 3:6] >= 0.02) and np.all(prm[:, 3:6] <= 0.03)
    assert np.std(prm[:, 3]) > 0 and np.allclose(q[:, 0], -1.5) and np.allclose(q[:, 1:23], 0) and np.allclose(q[:, 23:26], obj0)
    # the object rests in the palm for a few control steps: finite, contacts active, not dropped immediately
    a = torch.zeros(n, env.act_dim, device=env.device)
    for _ in range(5):
        obs, rew, done, trunc, _ = env.step(a)
    torch.cuda.synchronize()
    assert torch.isfinite(obs).all() and not bool(done.any())


def test_reach_task_golden_reset_and_time_switch():
    """myoHandReachRandom-v0 on the device: obs / reward / done against the reference's own ReachEnvV0 outputs (tests/golden/tasks.npz),
    target sampling inside the registered spans, and far_th arming at the 2nd control step (mjData.time accumulates per substep)."""
    import torch
    from myosuite_b200 import vec_env
    n = len(TG["reach_qpos"])
    env = vec_env.MyoVecEnv("myoHandReachRandom-v0", n, auto_reset=False)
    assert env.obs_dim == 115 and env.max_episode_steps == 100 and env.tip_names == ["THtip", "IFtip", "MFtip", "RFtip", "LFtip"]
    env.set_state(qpos=TG["reach_qpos"], qvel=TG["reach_qvel"], act=TG["reach_act"])
    env.t["target"][:, :15] = torch.as_tensor(TG["reach_targets"].reshape(n, 15), device=env.device)
    env.t["time"][:] = torch.as_tensor(TG["reach_time"], device=env.device)
    env.refresh_obs(); torch.cuda.synchronize()
    np.testing.assert_allclose(env.t["obs"].cpu().numpy(), TG["reach_obs"], rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(env.t["reward"].cpu().numpy(), TG["reach_dense"], rtol=1e-5, atol=1e-5)
    np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), TG["reach_done"].astype(bool))
    # reset: targets ~ U(span) per coordinate, initial pose = init_qpos, obs consistent with them
    env.reset(seed=3); torch.cuda.synchronize()
    tg = env.t["target"][:, :15].cpu().numpy(); lo, hi = env.t["target_range"][:15, 0].cpu().numpy(), env.t["target_range"][:15, 1].cpu().numpy()
    assert np.all(tg >= lo - 1e-15) and np.all(tg <= hi + 1e-15) and np.all(np.std(tg, axis=0)[hi > lo] > 0)
    obs = env.t["obs"].cpu().numpy()
    np.testing.assert_allclose(obs[:, 46:61] + obs[:, 61:76], tg, rtol=0, atol=1e-6)          # tip_pos + reach_err = target
    # zero action: far from the targets, done must stay off at step 1 and switch on at step 2 (time = 0.04000000000000002 > 2 dt)
    a = torch.full((n, env.act_dim), -1.0, device=env.device)
    for k in range(1, 4):
        obs, rew, done, trunc, info = env.step(a); torch.cuda.synchronize()
        dist = np.linalg.norm(obs[:, 61:76].cpu().numpy().astype(np.float64), axis=1); dn = done.cpu().numpy().astype(bool)
        clear = np.abs(dist - 5 * 0.034) > 1e-5                                            # (f32 obs: skip envs sitting on the threshold)
        if k == 1:
            assert not dn.any()
        else:
            assert np.array_equal(dn[clear], (dist > 5 * 0.034)[clear])
    assert info["time"].cpu().numpy()[0] == pytest.approx(0.06)


def test_dense_solver_all_sizes():
    """The dense SPD solver of the Newton / integrator phases against numpy for every n it dispatches on: register Cholesky (n <= 32,
    four unrolled sizes), bordered register Cholesky (33..36) and shared-memory rows fallback (> 36)."""
    from myosuite_b200 import abi
    rng = np.random.default_rng(5)
    for n in list(range(1, 41)) + [48]:
        count = 6
        A = rng.normal(size=(count, n, n)); H = A @ np.transpose(A, (0, 2, 1)) + n * np.eye(n)[None] * rng.uniform(0.01, 1.0, (count, 1, 1))
        b = rng.normal(size=(count, n))
        il = np.tril_indices(n)
        Hp = np.stack([H[k][il] for k in range(count)])
        ref = np.stack([np.linalg.solve(H[k], b[k]) for k in range(count)])
        x = abi.debug_chol_solve(Hp, b)
        np.testing.assert_allclose(x, ref, rtol=1e-9, atol=1e-11 * np.abs(ref).max(), err_msg="n=%d" % n)


# ----------------------------------------------------------------------------- mid-episode states, the hold model, regime and overflow rates
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("eid,warm", [("myoHandObjHoldRandom-v0", 8), ("myoHandObjHoldRandom-v0", 14), ("myoHandPoseRandom-v0", 30)])
def test_mid_episode_forward_and_rollout_parity(eid, warm, rows):
    """States REACHED by the simulator (reset + `warm` control steps of random actions), not random joint configurations: the object
    resting in / slipping through the curling fingers (per-env random object sizes), the hand mid-curl.  One forward pass (qacc, muscle
    force, contact list in order, distances) and 10 chained substeps against the oracle; every env must be checked."""
    import torch
    from myosuite_b200 import vec_env
    n = 192
    env = vec_env.MyoVecEnv(eid, n, taps=True, maxcon=48, auto_reset=False, seed=5, row_storage=rows)
    m = env.mj_model
    env.reset(seed=5)
    g = torch.Generator(device="cpu").manual_seed(warm)
    for _ in range(warm):
        env.step((torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device))
    torch.cuda.synchronize()
    assert int(env.t["overflow"].sum().item()) == 0
    qpos, qvel, act = (env.t[k].cpu().numpy().copy() for k in ("qpos", "qvel", "act"))
    alive = ~env.t["done"].cpu().numpy().astype(bool)
    ctrl = np.random.default_rng(warm).uniform(0, 1, (n, m.nu))
    env.t["qacc_warmstart"].zero_()
    env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_")}
    pmi = env.prog_info["pair_model_index"]
    ncon_total = checked = deep_n = deep_ok = 0; worst = 0.0
    oracles = [_oracle_for(env, e) for e in range(n)]
    for e in range(n):
        o = oracles[e]; o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e, :m.na], ctrl=ctrl[e]); o.forward()
        if not alive[e]:
            continue
        if not _in_regime(o, m):          # deep finger-pad overlap (6 % of env-steps of a random-action rollout, see the regime test): checked like every other env
            deep_n += 1; deep_ok += relerr(t["tap_qacc"][e], o.f("qacc")) < QACC_TOL[rows]["mid"]
        checked += 1
        worst = max(worst, relerr(t["tap_qacc"][e], o.f("qacc")))
        assert _note("mid/%s/%d" % (eid[3:11], warm), rows, relerr(t["tap_qacc"][e], o.f("qacc"))) < QACC_TOL[rows]["mid"]          # (stiff object / finger contacts; north star: 1e-5)
        assert relerr(t["tap_actuator_force"][e], o.f("actuator_force")) < RTOL
        nc = int(t["tap_ncon"][e, 0])
        got = [pmi[p] for p in t["tap_contact_pair"][e][:nc]]
        exp = [int(p) for p in o.i("con_pair") if int(p) in set(pmi)]
        assert got == exp
        np.testing.assert_allclose(t["tap_contact_dist"][e][:nc], [d for p, d in zip(o.i("con_pair"), o.f("con_dist")) if int(p) in set(pmi)], rtol=1e-7, atol=1e-11)
        ncon_total += nc
    print("%s after %d steps: %d/%d envs checked, %d contacts, worst qacc deviation %.2e; deep-overlap envs: %d, of which %d agree within tolerance" % (eid + "[" + rows + "]", warm, checked, n, ncon_total, worst, deep_n, deep_ok))
    assert checked == int(alive.sum()) and checked >= n // 4 and deep_ok == deep_n          # EVERY live env is checked: states the simulator reaches are inside the parity claim
    assert ncon_total > 0
    if env.task == "hold":      # the object really is in contact with the hand in this batch
        obj = m.name2id("geom", "object")
        assert any(obj in (int(a), int(b)) for o in oracles[:8] for a, b in zip(o.i("con_geom1"), o.i("con_geom2")))
    # 10 chained substeps from the same states
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 10); torch.cuda.synchronize()
    gq, gv = env.t["qpos"].cpu().numpy(), env.t["qvel"].cpu().numpy()
    for e in range(0, n, 3):
        if not alive[e]:
            continue
        o = oracles[e]; o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e, :m.na], ctrl=ctrl[e]); o.step(10)
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=2e-7)
        assert relerr(gv[e], o.f("qvel")) < 1e-5


@pytest.mark.parametrize("eid,n", [("myoHandPoseRandom-v0", 4096), ("myoHandObjHoldRandom-v0", 2048)])
def test_regime_and_overflow_rate_on_rollouts(eid, n):
    """How often does a real rollout (BASELINE sizes, random actions, 100 control steps, auto-reset) leave the regime the parity claim
    covers (ellipsoid contacts deeper than half a capsule radius) or exceed the contact capacity?  Both must be rare: < 1e-3 of env-steps
    (measured round 2: see DESIGN.md)."""
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv(eid, n, taps=True, seed=9)
    m = env.mj_model
    env.reset(seed=9)
    pmi = np.asarray(env.prog_info["pair_model_index"])
    g1, g2 = m.pair_geom1[pmi], m.pair_geom2[pmi]
    ell = torch.as_tensor(m.geom_type[g2] == 4, device=env.device)
    rad = torch.as_tensor(np.where(m.geom_type[g1] == 3, m.geom_size[g1][:, 0], m.geom_size[g1].min(1)), device=env.device)
    g = torch.Generator(device=env.device).manual_seed(1)
    deep = over = 0
    steps = 100
    for _ in range(steps):
        env.step(torch.rand(n, m.nu, device=env.device, generator=g) * 2 - 1)
        pair = env.t["tap_contact_pair"].long(); dist = env.t["tap_contact_dist"]
        valid = pair >= 0
        p = pair.clamp(min=0)
        bad = valid & ell[p] & (dist < -0.5 * rad[p])
        deep += int(bad.any(1).sum().item())
        over += int((env.t["tap_ncon"][:, 3] != 0).sum().item())
    rate_deep, rate_over = deep / (n * steps), over / (n * steps)
    print("regime: deep ellipsoid penetration %.2e of env-steps, contact overflow %.2e (last substep of each step)" % (rate_deep, rate_over))
    assert rate_over < 1e-3
    # the product-path flag: sticky per env until its next reset
    assert int((env.t["overflow"] != 0).sum().item()) <= n * 0.05


# ----------------------------------------------------------------------------- torso model / TorsoEnvV0 (myoTorsoPoseFixed-v0: 18 dof, 210 muscles, 15 joint couplings)
def test_torso_task_golden_physics_parity_and_env_step():
    import torch
    from myosuite_b200 import vec_env
    from oracle import env_oracle
    from oracle.oracle_py import Oracle
    T = np.load(os.path.join(os.path.dirname(__file__), "golden", "torso.npz"))
    n = len(T["qpos"])
    env = vec_env.MyoVecEnv("myoTorsoPoseFixed-v0", n, taps=True, auto_reset=False)
    m = env.mj_model
    assert (m.nq, m.nv, m.nu, env.obs_dim, env.max_episode_steps, env.n_frames) == (18, 18, 210, 264, 200, 5)
    env.reset(seed=0)
    np.testing.assert_allclose(env.t["target"][0].cpu().numpy(), T["target"], atol=0)           # target = mean of the registered ranges, never resampled
    # (1) task logic on the device vs the reference's own TorsoEnvV0 outputs
    env.set_state(qpos=T["qpos"], qvel=T["qvel"], act=T["act"])
    env.refresh_obs(); torch.cuda.synchronize()
    np.testing.assert_array_equal(env.t["obs"].cpu().numpy(), T["obs"])                       # float32, bit-exact
    np.testing.assert_allclose(env.t["reward"].cpu().numpy(), T["dense"], rtol=3e-6, atol=3e-6)
    np.testing.assert_array_equal(env.t["done"].cpu().numpy().astype(bool), T["done"].astype(bool))
    # (2) physics: one forward pass and 5 chained substeps vs the oracle, on states inside the joint ranges
    rng = np.random.default_rng(3)
    qpos, qvel, act, ctrl = _states(m, n, rng, overshoot=0.02, vel=0.5)
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 0); torch.cuda.synchronize()
    t = {k: v.cpu().numpy().copy() for k, v in env.t.items() if k.startswith("tap_")}
    o = Oracle(env.I, env.D)
    for e in range(0, n, 3):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        assert relerr(t["tap_qacc"][e], o.f("qacc")) < 1e-6
        assert relerr(t["tap_actuator_force"][e], o.f("actuator_force")) < RTOL
        assert relerr(t["tap_ten_length"][e], o.f("actuator_length")) < 1e-10
        assert int(t["tap_ncon"][e, 1]) == o.nefc
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 5); torch.cuda.synchronize()
    gq = env.t["qpos"].cpu().numpy()
    for e in range(0, n, 6):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.step(5)
        np.testing.assert_allclose(gq[e], o.f("qpos"), rtol=0, atol=1e-8)
    # (3) one full env step (sigmoid remap, 5 substeps, obs / reward) vs env_oracle
    env.set_state(qpos=qpos, qvel=qvel, act=act); env.t["time"].zero_(); env.t["step_count"].zero_()
    a = rng.uniform(-1, 1, (n, m.nu)).astype(np.float32)
    obs, rew, done, trunc, _ = env.step(torch.as_tensor(a, device=env.device)); torch.cuda.synchronize()
    obs, rew = obs.cpu().numpy(), rew.cpu().numpy()
    for e in range(0, n, 6):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e])
        env_oracle.env_step(o, a[e].astype(np.float64), env.n_frames)
        np.testing.assert_allclose(obs[e], env_oracle.pose_obs(o.f("qpos"), o.f("qvel"), o.f("act"), T["target"], env.dt), rtol=2e-6, atol=2e-6)
        r = env_oracle.pose_reward(o.f("qpos"), o.f("act"), T["target"], 0.25, far_th=np.pi)
        assert rew[e] == pytest.approx(r["dense"], rel=1e-5, abs=1e-5)
