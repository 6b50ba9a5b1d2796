"""CPU reference of the leg stand task, myoLegStandRandom-v0 (the ReachEnvV0 of myosuite/envs/myo/myobase/walk_v0.py): obs / reward
terms of a state held by the physics oracle, and the randomised joint reset.  Test infrastructure, pinned against tests/golden/stand.npz,
which the reference's own unmodified methods produced (tests/golden/make_golden_stand.py)."""
import numpy as np

from oracle import env_oracle

STAND_WEIGHTS = {"reach": 1.0, "bonus": 4.0, "penalty": 50, "act_reg": 1}        # walk_v0.py:18-24


def stand_obs_reward(m, o, dt, tips, targets, time, far_th=0.44, weights=None):
    """walk_v0.py:80-140: obs = [qpos, qvel*dt, tip_pos, target - tip_pos, act] (f32, the reach layout); reward terms with
    reach = 10 - d - 10 |qvel dt|, act_reg = -100 |act|/na, near_th = 0.05 ntip, far_th armed once time > 2 dt."""
    weights = weights or STAND_WEIGHTS
    obs, _ = env_oracle.reach_obs_reward(m, o, dt, tips, targets, time, far_th=far_th)
    qvel, act = o.f("qvel"), o.f("act")
    sx = o.f("site_xpos").reshape(-1, 3)
    tip = np.concatenate([sx[m.name2id("site", t)] for t in tips])
    d = np.linalg.norm(np.asarray(targets, dtype=np.float64).ravel() - tip)
    v = np.linalg.norm(qvel * dt)
    act_mag = np.linalg.norm(act) / m.na if m.na else 0.0
    far = far_th * len(tips) if time > 2 * dt else np.inf
    near = len(tips) * 0.050
    r = dict(reach=10.0 - 1.0 * d - 10.0 * v, bonus=1.0 * (d < 2 * near) + 1.0 * (d < near), act_reg=-100.0 * act_mag, penalty=-1.0 * (d > far),
             sparse=-1.0 * d, solved=bool(d < near), done=bool(d > far))
    r["dense"] = sum(wt * r[k] for k, wt in weights.items())
    return obs, r


def stand_reset_qpos(m, init_qpos, u, joint_random_range=(-0.2, 0.2)):
    """ReachEnvV0.generate_qpos (walk_v0.py:152-167) on given uniforms u ~ U[0, 1), one per joint in joint order: the first qpos
    coordinate of every joint += U(lo, hi) (numpy's low + (high - low) u), clipped to jnt_range whether or not the joint is limited."""
    lo, hi = joint_random_range
    adr = m.jnt_qposadr
    q = np.array(init_qpos, dtype=np.float64, copy=True)
    q[adr] += lo + (hi - lo) * np.asarray(u, dtype=np.float64)
    q[adr] = np.clip(q[adr], m.jnt_range[:, 0], m.jnt_range[:, 1])
    return q
