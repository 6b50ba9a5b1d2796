"""Dump golden physics vectors from a REAL MuJoCo + the reference's own envs (SURVEY.md section 8c, "plan when MuJoCo becomes importable").

NOT runnable without `mujoco` and `gymnasium` (neither is a dependency of this project): this script is the recipe a
maintainer runs once on a machine where `pip install myosuite` works, to turn the oracle's "parity unpinned" status into pinned goldens.
It uses only the reference's public API (gym.make, env.step) and MuJoCo's Python bindings; nothing from this repository is imported.

    python tools/dump_reference.py --out tests/golden/mujoco_<env>.npz [--env myoHandPoseRandom-v0] [--steps 200] [--seed 0]

Per control step and per substep it records the inputs (qpos, qvel, act, ctrl) and MuJoCo's outputs evaluated at that pre-step state
(qacc, actuator_force, ten_length, actuator_length, qfrc_bias, qM non-zeros, contact geom ids / dist / frame, efc_force), plus the
compiled model arrays the MJCF compiler of this repo must reproduce (body_mass, body_inertia, body_ipos, dof_invweight0, ...).
Acceptance (north-star): qacc and actuator_force within 1e-5 relative, contact geom pairs bit-exact, compiled arrays within 1e-9.
tests/test_oracle.py picks the file up when present (see `test_mujoco_goldens_if_present`).
"""
import argparse

import numpy as np

MODEL_FIELDS = ["body_mass", "body_inertia", "body_ipos", "body_iquat", "body_pos", "body_quat", "body_parentid", "jnt_type", "jnt_axis", "jnt_pos",
                "jnt_range", "jnt_qposadr", "jnt_dofadr", "dof_damping", "dof_armature", "dof_invweight0", "body_invweight0", "tendon_lengthspring",
                "tendon_invweight0", "actuator_gainprm", "actuator_biasprm", "actuator_dynprm", "actuator_lengthrange", "actuator_acc0",
                "geom_type", "geom_size", "geom_pos", "geom_quat", "geom_bodyid", "pair_geom1", "pair_geom2", "qpos0", "key_qpos"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="myoHandPoseRandom-v0")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()

    import mujoco                                    # noqa: F401  (fails here by design: see the module docstring)
    from myosuite.utils import gym
    import myosuite                                  # noqa: F401  registers the envs

    env = gym.make(args.env)
    u = env.unwrapped
    model, data = u.mj_model, u.mj_data
    rng = np.random.default_rng(args.seed)
    env.reset(seed=args.seed)
    rec = {k: [] for k in ("qpos", "qvel", "act", "ctrl", "qacc", "actuator_force", "ten_length", "actuator_length", "qfrc_bias", "qM",
                           "ncon", "con_geom", "con_dist", "con_frame", "nefc", "efc_force", "action", "obs", "reward", "done", "time")}
    scratch = mujoco.MjData(model)

    def snapshot(d):
        """forward() on a copy of the state: MuJoCo's outputs at the pre-step state, without touching the env's own data"""
        scratch.qpos[:], scratch.qvel[:], scratch.act[:], scratch.ctrl[:] = d.qpos, d.qvel, d.act, d.ctrl
        scratch.qacc_warmstart[:] = d.qacc_warmstart
        scratch.time = d.time
        mujoco.mj_forward(model, scratch)
        rec["qpos"].append(scratch.qpos.copy()); rec["qvel"].append(scratch.qvel.copy()); rec["act"].append(scratch.act.copy()); rec["ctrl"].append(scratch.ctrl.copy())
        rec["qacc"].append(scratch.qacc.copy()); rec["actuator_force"].append(scratch.actuator_force.copy()); rec["ten_length"].append(scratch.ten_length.copy())
        rec["actuator_length"].append(scratch.actuator_length.copy()); rec["qfrc_bias"].append(scratch.qfrc_bias.copy()); rec["qM"].append(scratch.qM.copy())
        n = scratch.ncon
        geom = np.full((64, 2), -1, np.int32); dist = np.zeros(64); frame = np.zeros((64, 9))
        for c in range(min(n, 64)):
            geom[c] = scratch.contact[c].geom1, scratch.contact[c].geom2; dist[c] = scratch.contact[c].dist; frame[c] = scratch.contact[c].frame
        rec["ncon"].append(n); rec["con_geom"].append(geom); rec["con_dist"].append(dist); rec["con_frame"].append(frame)
        ef = np.zeros(512); ef[:min(scratch.nefc, 512)] = scratch.efc_force[:min(scratch.nefc, 512)]
        rec["nefc"].append(scratch.nefc); rec["efc_force"].append(ef)

    for _ in range(args.steps):
        a = rng.uniform(-1, 1, model.nu).astype(np.float32)
        # one record per control step at its first substep (ctrl as BaseV0.step sets it); the substeps in between are covered by the
        # state sequence itself: stepping this repo's kernel from the recorded state must land on the next recorded state
        ctrl_before = data.ctrl.copy()
        obs, rew, term, trunc, info = env.step(a)
        rec["action"].append(a); rec["obs"].append(np.asarray(obs, np.float32)); rec["reward"].append(float(rew)); rec["done"].append(bool(term)); rec["time"].append(float(data.time))
        snapshot(data)
        del ctrl_before
        if term or trunc:
            env.reset()
    out = {k: np.array(v) for k, v in rec.items()}
    for f in MODEL_FIELDS:
        if hasattr(model, f):
            out["model_" + f] = np.array(getattr(model, f))
    out["meta"] = np.array([args.env, str(args.seed), mujoco.__version__])
    np.savez_compressed(args.out, **out)
    print("wrote", args.out, {k: v.shape for k, v in out.items() if k != "meta"})


if __name__ == "__main__":
    main()
