"""Time MyoVecEnv.static_opt (muscle static optimisation, one launch) with CUDA events at the benchmarked shapes, 4096 hand envs, 2048 legs
envs and the torso, and the CPU reference of tests/static_opt_ref.py (the problem from the oracle, solved by bounded least squares) on one
host core per env.  Prints Newton step counts and the GPU's name and power limit read in the same run; what was not measured is printed as
"not measured".  Writes nothing into the tree.

    python tools/static_opt_bench.py [--reps 20] [--cpu-envs 16]
"""
import argparse
import json
import os
import subprocess
import sys
import time

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(_v, "1")        # the CPU reference on one core
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

# (label, env id, envs, reserve strength): the tests' reserve scales (tests/test_static_opt.py)
SHAPES = [("hand", "myoHandPoseRandom-v0", 4096, 1.0), ("legs", "myoLegStandRandom-v0", 2048, 100.0), ("torso", "myoTorsoPoseFixed-v0", 661, 100.0)]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split("\n")[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception:
        import torch
        return dict(gpu=torch.cuda.get_device_name(0), power_limit="not measured", max_sm_clock="not measured")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warm", type=int, default=6, help="random-action env steps before the timed calls")
    ap.add_argument("--cpu-envs", type=int, default=16, help="envs of each shape solved by the CPU reference (0: not measured)")
    args = ap.parse_args()
    import torch
    from myosuite_b200 import vec_env
    try:
        os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
    except (AttributeError, OSError):
        pass
    torch.set_num_threads(1)
    info = gpu_info()
    print("%s, power limit %s, max SM clock %s" % (info["gpu"], info["power_limit"], info["max_sm_clock"]))
    rows = []
    for label, eid, n, rho in SHAPES:
        env = vec_env.MyoVecEnv(eid, n, seed=0)
        env.reset(seed=0)
        g = torch.Generator(device="cpu").manual_seed(0)
        for _ in range(args.warm):
            env.step((torch.rand(n, env.mj_model.nu, generator=g) * 2 - 1).to(env.device))
        Q = env.data("qacc")["qacc"].clone()
        S = env.static_opt(Q, rho, fields=("act", "niter", "converged"))      # first call: launch set-up
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.reps):
            env.static_opt(Q, rho, fields=("act", "niter", "converged"))
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.reps
        it = S["niter"].double()
        row = dict(shape=label, env_id=eid, n_env=n, reserve=rho, gpu_ms=round(ms, 3), gpu_us_per_env=round(1e3 * ms / n, 3),
                   niter_mean=round(it.mean().item(), 2), niter_max=int(it.max().item()), converged=float((S["converged"] == 1).double().mean().item()))
        if args.cpu_envs > 0:
            import static_opt_ref as R
            from inverse_oracle import InvOracle
            st = env.get_env_state(); m = env.mj_model; QH = Q.cpu().numpy()
            o = InvOracle(env.I, env.D)
            k = min(args.cpu_envs, n)
            t, G, _, _, _, _ = R.problem(o, m, st["qpos"][0], st["qvel"][0], st["act"][0, :m.na], QH[0])
            R.solve_lsq(t, G, np.ones(m.nu), np.full(m.nv, rho))      # (untimed: imports and first-call set-up)
            t0 = time.perf_counter()
            for e in range(k):
                t, G, _, _, _, _ = R.problem(o, m, st["qpos"][e], st["qvel"][e], st["act"][e, :m.na], QH[e])
                R.solve_lsq(t, G, np.ones(m.nu), np.full(m.nv, rho))
            row["cpu_ms_per_env"] = round(1e3 * (time.perf_counter() - t0) / k, 3)
            row["cpu_envs"] = k
        else:
            row["cpu_ms_per_env"] = "not measured"
        rows.append(row)
        print("%-6s %5d envs  reserve %g: %.3f ms per call (%.3f us per env), Newton steps mean %.2f max %d, converged %.4f; CPU reference %s ms per env"
              % (label, n, rho, ms, 1e3 * ms / n, row["niter_mean"], row["niter_max"], row["converged"], row["cpu_ms_per_env"]))
        del env
        torch.cuda.empty_cache()
    print(json.dumps(dict(info, shapes=rows)))


if __name__ == "__main__":
    main()
