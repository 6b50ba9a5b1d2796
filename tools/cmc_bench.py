"""Time computed muscle control as one call (MyoVecEnv.cmc) against the same loop written with the public per-frame calls (the loop of
tests/test_static_opt.py::test_cmc_tracks_hand_trajectory without its bookkeeping: desired acceleration in torch, static_opt(), rollout(),
the state copied back into the bound tensors).  Alternating runs of the two on each case, host clock around work that ends in a device
synchronise.  Cases: the hand pose (4096 envs), the elbow (4096) and the legs (2048), 200 frames each, at substeps 1 and frame_skip (the loop
then holds static_opt's one-step ctrl over the interval: the same work, not the same excitation).  The reference of each case is a rollout
of smooth random excitations from the reset state.  Prints ms per frame, mean Newton steps, and the GPU's name and power limit read in the
same run.  Writes nothing into the tree.

    python tools/cmc_bench.py [--frames 200] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KP, KV = 100.0, 20.0
# (label, env id, envs, reserve strength): tests/test_static_opt.py's reserve scales
CASES = [("hand", "myoHandPoseRandom-v0", 4096, 1.0), ("elbow", "myoElbowPose1D6MRandom-v0", 4096, 1.0), ("legs", "myoLegStandRandom-v0", 2048, 100.0)]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split("\n")[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception:
        import torch
        return dict(gpu=torch.cuda.get_device_name(0), power_limit="not measured", max_sm_clock="not measured")


def tangent_diff(m, dev):
    """mj_differentiatePos(q1, q2) (dt = 1) over a batch in torch: hinge and slide joints subtract, free and ball joints take the rotation
    vector of conj(q1) q2"""
    import torch
    lin_q, lin_d, rot = [], [], []
    for j in range(m.njnt):
        qa, da, jt = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j]), int(m.jnt_type[j])
        if jt == 0:
            lin_q += [qa, qa + 1, qa + 2]; lin_d += [da, da + 1, da + 2]; rot.append((qa + 3, da + 3))
        elif jt == 1:
            rot.append((qa, da))
        else:
            lin_q.append(qa); lin_d.append(da)
    lq, ld = torch.tensor(lin_q, device=dev), torch.tensor(lin_d, device=dev)

    def diff(q1, q2):
        v = torch.empty(q1.shape[0], m.nv, dtype=q1.dtype, device=dev)
        v[:, ld] = q2[:, lq] - q1[:, lq]
        for qa, da in rot:
            a, b = q1[:, qa:qa + 4], q2[:, qa:qa + 4]
            w = (a * b).sum(1)
            x = torch.stack([a[:, 0] * b[:, 1] - b[:, 0] * a[:, 1] - (a[:, 2] * b[:, 3] - a[:, 3] * b[:, 2]),
                             a[:, 0] * b[:, 2] - b[:, 0] * a[:, 2] - (a[:, 3] * b[:, 1] - a[:, 1] * b[:, 3]),
                             a[:, 0] * b[:, 3] - b[:, 0] * a[:, 3] - (a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1])], 1)
            s = x.norm(dim=1)
            ang = 2 * torch.atan2(s, w)
            ang = torch.where(ang > torch.pi, ang - 2 * torch.pi, ang)
            v[:, da:da + 3] = torch.where(s[:, None] < 1e-15, torch.zeros_like(x), x / s.clamp_min(1e-300)[:, None] * ang[:, None])
        return v
    return diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3, help="alternating timed runs of each variant per case")
    args = ap.parse_args()
    import torch
    from myosuite_b200 import vec_env
    info = gpu_info()
    print("%s, power limit %s, max SM clock %s" % (info["gpu"], info["power_limit"], info["max_sm_clock"]))
    T, rows = args.frames, []
    for label, eid, n, rho in CASES:
        env = vec_env.MyoVecEnv(eid, n, seed=0)
        env.reset(seed=0)
        m, dev = env.mj_model, env.device
        diff = tangent_diff(m, dev)
        start = {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart", "time")}
        for k in (1, env.n_frames):
            g = torch.Generator(device="cpu").manual_seed(0)
            phase, freq = torch.rand(n, 1, m.nu, generator=g) * 6.283, 0.5 + 2 * torch.rand(n, 1, m.nu, generator=g)
            tt = torch.arange(T, dtype=torch.float64)[None, :, None] * m.opt_timestep * k
            gen = env.rollout((0.4 + 0.3 * torch.sin(6.283 * freq * tt + phase)).to(dev).contiguous(), substeps=k, initial_state=start)
            P = torch.cat([start["qpos"][:, None], gen["qpos"][:, :-1]], 1).contiguous()
            V = torch.cat([start["qvel"][:, None], gen["qvel"][:, :-1]], 1).contiguous()
            A = gen["qacc"].contiguous()
            del gen

            def fused():
                return env.cmc(P, V, A, KP, KV, rho, substeps=k, initial_state=start, fields=("qpos", "qvel", "act", "ctrl", "reserve_force", "niter"))

            def loop():
                for key, x in start.items():
                    env.t[key].copy_(x)
                its = []
                for f in range(T):
                    q, v = env.t["qpos"], env.t["qvel"]
                    qd = (A[:, f] + KV * (V[:, f] - v) + KP * diff(q, P[:, f])).contiguous()
                    S = env.static_opt(qd, rho, fields=("ctrl", "reserve_force", "niter"))
                    its.append(S["niter"])
                    r = env.rollout(S["ctrl"][:, None].contiguous(), qfrc_applied=S["reserve_force"][:, None].contiguous(), substeps=k)
                    for key in ("qpos", "qvel", "act", "time"):
                        env.t[key].copy_(r[key][:, 0])
                    env.t["qacc_warmstart"].copy_(r["qacc"][:, 0])
                return torch.stack(its, 1)

            out, its = fused(), loop()          # (untimed: first-call set-up of both paths)
            torch.cuda.synchronize()
            t_f, t_l = [], []
            for _ in range(args.reps):
                for fn, acc in ((fused, t_f), (loop, t_l)):
                    torch.cuda.synchronize(); t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize(); acc.append(1e3 * (time.perf_counter() - t0) / T)
            row = dict(case=label, env_id=eid, n_env=n, frames=T, substeps=k, reserve=rho, fused_ms_per_frame=sorted(t_f)[len(t_f) // 2],
                       loop_ms_per_frame=sorted(t_l)[len(t_l) // 2], fused_runs=[round(x, 3) for x in t_f], loop_runs=[round(x, 3) for x in t_l],
                       fused_newton_mean=round(out["niter"].double().mean().item(), 2), loop_newton_mean=round(its.double().mean().item(), 2))
            row["speedup"] = round(row["loop_ms_per_frame"] / row["fused_ms_per_frame"], 2)
            rows.append(row)
            print("%-5s %5d envs substeps %2d: cmc() %.3f ms per frame, loop %.3f ms per frame (x%.2f); Newton steps cmc %.2f, loop %.2f"
                  % (label, n, k, row["fused_ms_per_frame"], row["loop_ms_per_frame"], row["speedup"], row["fused_newton_mean"], row["loop_newton_mean"]))
            del out, its, P, V, A
            torch.cuda.empty_cache()
        del env
        torch.cuda.empty_cache()
    print(json.dumps(dict(info, cases=rows)))


if __name__ == "__main__":
    main()
