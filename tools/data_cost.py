"""Cost of the mjData readout (MyoVecEnv.data, myo_batch_data), of the inverse dynamics (MyoVecEnv.inverse, myo_batch_inverse) and of
mj_step rollouts (MyoVecEnv.rollout, myo_batch_rollout) next to one env step, at the benchmarked launch shapes.

    python tools/data_cost.py [--reps 50] [--warmup 10] [--out FILE.json]

For each case: warm-up steps from a reset, then `reps` rounds that each time one env step, one readout of every group (pose, actuation,
dynamics, all fields), the inverse of the readout's qacc (with constraints, without them, with every output) and two rollouts from the
current state with CUDA events on the batch's stream, in alternating order.  The rollouts: "rollout", 8 intervals of frame_skip substeps,
reported per interval (the physics of one env step); "rollout_1", frame_skip intervals of one substep, reported per call (the same physics).  Prints medians (and min / max) in microseconds and the
GPU name, power limit and SM clock read through nvidia-smi's query interface (read-only).  Writes nothing unless --out is given."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [("hand_pose", "myoHandPoseRandom-v0", 4096), ("hold", "myoHandObjHoldRandom-v0", 2048),
         ("walk_fatigue", "myoFatiLegWalk-v0", 2048), ("elbow", "myoElbowPose1D6MRandom-v0", 4096)]
GROUPS = {"pose": ("xpos", "xquat", "xmat", "site_xpos"),
          "actuation": ("actuator_length", "actuator_velocity", "actuator_force", "qfrc_actuator"),
          "dynamics": ("qacc", "ncon", "contact_geom", "contact_dist", "contact_pos", "contact_frame", "contact_force"),
          "all": ()}
INVERSE = {"inverse": dict(fields=("qfrc_inverse",)), "inverse_free": dict(constraints=False, fields=("qfrc_inverse",)),
           "inverse_all": dict(fields=("qfrc_inverse", "qfrc_constraint", "contact_force", "actuator_moment"))}
ROLLOUT_NSTEP = 8           # intervals of the "rollout" row


def gpu_info():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                                     "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:          # (the numbers still print; the machine line says why it is missing)
        return ["unknown (%s)" % e]


def main():
    import numpy as np
    import torch
    from myosuite_b200 import vec_env
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"gpu_before": gpu_info(), "cases": {}}
    for name, eid, n in CASES:
        env = vec_env.MyoVecEnv(eid, n, seed=0)
        m = env.mj_model
        env.reset(seed=0)
        stream = torch.cuda.current_stream(env.device)
        g = torch.Generator(device="cpu").manual_seed(0)
        acts = [(torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device) for _ in range(8)]
        for k in range(args.warmup):
            env.step(acts[k % 8])
            for fields in GROUPS.values():
                env.data(*fields)
        qacc = env.data("qacc")["qacc"].clone()
        for kw in INVERSE.values():
            env.inverse(qacc, **kw)
        fs = env.frame_skip
        roll = {"rollout": (torch.rand(n, ROLLOUT_NSTEP, m.nu, generator=g, dtype=torch.float64).to(env.device), fs, ROLLOUT_NSTEP),
                "rollout_1": (torch.rand(n, fs, m.nu, generator=g, dtype=torch.float64).to(env.device), 1, 1)}      # (ctrl, substeps, divisor)
        for ctrl, sub, _ in roll.values():
            env.rollout(ctrl, substeps=sub)
        torch.cuda.synchronize()
        order = ["step"] + list(GROUPS) + list(INVERSE) + list(roll)
        t = {k: [] for k in order}
        for r in range(args.reps):
            seq = order if r % 2 == 0 else order[::-1]
            for k in seq:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                if k == "step":
                    env.step(acts[r % 8])
                elif k in INVERSE:
                    env.inverse(qacc, **INVERSE[k])
                elif k in roll:
                    env.rollout(roll[k][0], substeps=roll[k][1])
                else:
                    env.data(*GROUPS[k])
                e1.record(stream)
                e1.synchronize()
                t[k].append(e0.elapsed_time(e1) * 1e3 / (roll[k][2] if k in roll else 1))
        s = {k: dict(median_us=float(np.median(v)), min_us=float(np.min(v)), max_us=float(np.max(v))) for k, v in t.items()}
        for k in order[1:]:
            s[k]["per_step"] = s[k]["median_us"] / s["step"]["median_us"]
        res["cases"][name] = dict(env_id=eid, n_env=n, frame_skip=env.frame_skip, **s)
        print("%-13s n %4d  step %8.1f us | " % (name, n, s["step"]["median_us"])
              + "  ".join("%s %7.1f us (%.3f step)" % (k, s[k]["median_us"], s[k]["per_step"]) for k in order[1:]), flush=True)
        del env
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print("GPU [name, power limit, SM clock, max SM clock, throttle reasons] before: %s after: %s" % (res["gpu_before"], res["gpu_after"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
