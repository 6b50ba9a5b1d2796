"""CPU ORACLE for the Python-side part of the hot path (TEST INFRASTRUCTURE, not product code).

numpy restatement of what the reference does around mj_step each control step; every function cites
the reference lines it follows.  Pinned against tests/golden/pylogic.npz, which was produced by running
the reference's own unmodified code (tests/golden/make_golden.py).
"""
import numpy as np


def action_to_ctrl(a, normalize_act=True):
    """myosuite/envs/myo/base_v0.py:83-96 (all actuators of the hot-path models are muscles)."""
    a = np.array(a, dtype=np.float64, copy=True)
    if normalize_act:
        a = 1.0 / (1.0 + np.exp(-5.0 * (a - 0.5)))
    return a


class Fatigue:
    """3CC-r cumulative fatigue, myosuite/envs/myo/fatigue.py:8-99."""

    def __init__(self, n, dt, tauact=0.01, taudeact=0.04):
        self.r, self.F, self.R = 10 * 15, 0.00912, 0.1 * 0.00094      # fatigue.py:9-11
        self.dt = dt                                                 # fatigue.py:12 (timestep * frame_skip)
        self.tauact, self.taudeact = np.broadcast_to(tauact, (n,)).astype(float), np.broadcast_to(taudeact, (n,)).astype(float)
        self.MA, self.MR, self.MF = np.zeros(n), np.ones(n), np.zeros(n)   # fatigue.py:18-20

    def compute_act(self, act):
        """fatigue.py:38-76 (order of the masked assignments matters; returns the updated MA as the muscle ctrl)."""
        TL = np.array(act, dtype=np.float64)
        MA, MR, MF = self.MA, self.MR, self.MF
        LD = 1 / self.tauact * (0.5 + 1.5 * MA)
        LR = (0.5 + 1.5 * MA) / self.taudeact
        C = np.zeros_like(MA)
        i = (MA < TL) & (MR > (TL - MA)); C[i] = LD[i] * (TL[i] - MA[i])
        i = (MA < TL) & (MR <= (TL - MA)); C[i] = LD[i] * MR[i]
        i = MA >= TL; C[i] = LR[i] * (TL[i] - MA[i])
        rR = np.where(MA >= TL, self.r * self.R, self.R)
        C = np.clip(C, np.maximum(-MA / self.dt + self.F * MA, (MR - 1) / self.dt + rR * MF),
                    np.minimum((1 - MA) / self.dt + self.F * MA, MR / self.dt + rR * MF))
        dMA, dMR, dMF = (C - self.F * MA) * self.dt, (-C + rR * MF) * self.dt, (self.F * MA - rR * MF) * self.dt
        self.MA, self.MR, self.MF = MA + dMA, MR + dMR, MF + dMF
        return self.MA, self.MR, self.MF


def pose_obs(qpos, qvel, act, target, dt):
    """myosuite/envs/myo/myobase/pose_v0.py:100-111 + envs/obs_vec_dict.py:76-88
    (keys qpos, qvel, pose_err, act in that order; float32)."""
    return np.concatenate([qpos, np.asarray(qvel) * dt, np.asarray(target) - qpos, act]).astype(np.float32)


def pose_reward(qpos, act, target, pose_thd, weights=(1.0, 4.0, 1.0, 50.0), far_th=4 * np.pi / 2):
    """myosuite/envs/myo/myobase/pose_v0.py:113-140 -> dict(dense, solved, done, pose, bonus, penalty, act_reg).
    TorsoEnvV0 (torso_v0.py:98-125) is the same rule with far_th = pi."""
    pose_dist = np.linalg.norm(np.asarray(target) - qpos)
    act_mag = np.linalg.norm(act) / (len(act) if len(act) else 1)
    r = dict(pose=-pose_dist, bonus=1.0 * (pose_dist < pose_thd) + 1.0 * (pose_dist < 1.5 * pose_thd), penalty=-1.0 * (pose_dist > far_th),
             act_reg=-act_mag, sparse=-pose_dist, solved=pose_dist < pose_thd, done=pose_dist > far_th)
    r["dense"] = weights[0] * r["pose"] + weights[1] * r["bonus"] + weights[2] * r["act_reg"] + weights[3] * r["penalty"]
    return r


def env_step(oracle, action, frame_skip, normalize_act=True, fatigue=None):
    """One control step on the physics oracle: base_v0.py:82-118 + robot.py:901-905 (same ctrl for all substeps)."""
    ctrl = action_to_ctrl(action, normalize_act)
    if fatigue is not None:
        ctrl = fatigue.compute_act(ctrl)[0].copy()
    oracle.set(ctrl=ctrl)
    oracle.step(frame_skip)
    return ctrl


# ----------------------------------------------------------------------------- WalkEnvV0 (walk_v0.py)
def quat2mat00(q):
    """[0,0] entry of myosuite.utils.quat_math.quat2mat (used by WalkEnvV0._get_rot_condition, walk_v0.py:463-473)."""
    w, x, y, z = q
    n = w * w + x * x + y * y + z * z
    return 1.0 - 2.0 / n * (y * y + z * z)


def walk_obs_reward(m, o, steps, dt, ids, cfg):
    """obs vector (f32[403]) and reward terms of WalkEnvV0 from the oracle's forward quantities of the observed state.
    Follows walk_v0.py:268-319 (obs / reward), :358-494 (helpers).  `ids`: dict of model ids; `cfg`: registry kwargs.
    `steps` is WalkEnvV0.steps at the time _forward runs, i.e. BEFORE the increment in step() (walk_v0.py:339-342)."""
    qpos, qvel, act = o.f("qpos"), o.f("qvel"), o.f("act")
    xpos, xquat, xipos, cvel = o.f("xpos").reshape(-1, 3), o.f("xquat").reshape(-1, 4), o.f("xipos").reshape(-1, 3), o.f("cvel").reshape(-1, 6)
    mass = m.body_mass[:, None]
    com_vel = (np.sum(mass * (-cvel), 0) / np.sum(mass))[3:5]                  # _get_com_velocity :449-455
    com = np.sum(mass * xipos, 0) / np.sum(mass)                              # _get_com :475-481
    phase = (steps / cfg["hip_period"]) % 1
    fl, fr, pel = xpos[ids["talus_l"]], xpos[ids["talus_r"]], xpos[ids["pelvis"]]
    obs = np.concatenate([qpos[2:], qvel * dt, com_vel, xquat[ids["torso"]], [fl[2], fr[2]], [com[2]], fl - pel, fr - pel, [phase],
                          o.f("actuator_length"), np.clip(o.f("actuator_velocity"), -100, 100), np.clip(o.f("actuator_force") / 1000, -100, 100), act]).astype(np.float32)
    vel_reward = np.exp(-np.square(cfg["target_y_vel"] - com_vel[1])) + np.exp(-np.square(cfg["target_x_vel"] - com_vel[0]))
    des = np.array([0.8 * np.cos(phase * 2 * np.pi + np.pi), 0.8 * np.cos(phase * 2 * np.pi)], dtype=np.float32)
    ang = np.array([qpos[ids["q_hip_flexion_l"]], qpos[ids["q_hip_flexion_r"]]])
    cyclic = np.linalg.norm(des - ang)
    ref_rot = np.exp(-np.linalg.norm(5.0 * (qpos[3:7] - cfg["target_rot"])))
    jrew = np.exp(-5 * np.mean(np.abs([qpos[ids[k]] for k in ("q_hip_adduction_l", "q_hip_adduction_r", "q_hip_rotation_l", "q_hip_rotation_r")])))
    done = bool(com[2] < cfg["min_height"] or abs(quat2mat00(qpos[3:7])) > cfg["max_rot"])
    dense = 5.0 * vel_reward - 100 * done - 10 * cyclic + 10.0 * ref_rot + 5.0 * jrew      # DEFAULT_RWD_KEYS_AND_WEIGHTS :205-211
    return obs, dict(vel_reward=vel_reward, cyclic_hip=cyclic, ref_rot=ref_rot, joint_angle_rew=jrew, done=done, dense=dense)


def walk_ids(m):
    ids = {k: m.name2id("body", k) for k in ("talus_l", "talus_r", "pelvis", "torso")}
    for j in ("hip_flexion_l", "hip_flexion_r", "hip_adduction_l", "hip_adduction_r", "hip_rotation_l", "hip_rotation_r"):
        ids["q_" + j] = int(m.jnt_qposadr[m.name2id("joint", j)])
    return ids


# ----------------------------------------------------------------------------- ObjHold (obj_hold_v0.py)
def hold_obs_reward(m, o, dt, goal_pos):
    """obj_hold_v0.py:79-121: obs = [qpos[:-7], qvel[:-6]*dt, obj_pos, goal - obj_pos, act] (f32[91]); reward terms."""
    qpos, qvel, act = o.f("qpos"), o.f("qvel"), o.f("act")
    obj = o.f("site_xpos").reshape(-1, 3)[m.name2id("site", "object")]
    err = np.asarray(goal_pos) - obj
    obs = np.concatenate([qpos[:-7], qvel[:-6] * dt, obj, err, act]).astype(np.float32)
    d = np.abs(np.linalg.norm(err))
    drop = bool(d > 0.300)
    dense = 100.0 * (-d) + 4.0 * (1.0 * (d < 0.020) + 1.0 * (d < 0.010)) + 10 * (-1.0 * drop)
    return obs, dict(goal_dist=-d, done=drop, dense=dense)


def reach_obs_reward(m, o, dt, tips, targets, time, far_th=0.35, weights=None):
    """reach_v0.py:98-160: obs = [qpos, qvel*dt, tip_pos, target - tip_pos, act] (f32); reach / bonus / penalty terms.
    tips: site names; targets: [ntip, 3] world positions of the target sites; time: mjData.time of the observed state."""
    weights = weights or {"reach": 1.0, "bonus": 4.0, "penalty": 50}
    qpos, qvel, act = o.f("qpos"), o.f("qvel"), o.f("act")
    sx = o.f("site_xpos").reshape(-1, 3)
    tip = np.concatenate([sx[m.name2id("site", t)] for t in tips])
    err = np.asarray(targets, dtype=np.float64).ravel() - tip
    obs = np.concatenate([qpos, qvel * dt, tip, err, act]).astype(np.float32)
    d = np.linalg.norm(err)
    act_mag = np.linalg.norm(act) / m.na if m.na else 0.0
    far = far_th * len(tips) if time > 2 * dt else np.inf
    near = len(tips) * 0.0125
    terms = dict(reach=-d, bonus=1.0 * (d < 2 * near) + 1.0 * (d < near), act_reg=-act_mag, penalty=-1.0 * (d > far))
    dense = sum(wt * terms[k] for k, wt in weights.items())
    return obs, dict(reach=-d, done=bool(d > far), solved=bool(d < near), dense=dense)
