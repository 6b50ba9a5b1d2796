"""Cost of the mjData readout (MyoVecEnv.data, myo_batch_data), of the inverse dynamics (MyoVecEnv.inverse, myo_batch_inverse) and of
mj_step rollouts (MyoVecEnv.rollout, myo_batch_rollout) next to one env step, at the benchmarked launch shapes.

    python tools/data_cost.py [--reps 50] [--warmup 10] [--out FILE.json]

For each case: warm-up steps from a reset, then `reps` rounds that each time one env step, one readout of every group (pose, actuation,
dynamics, all fields), the inverse of the readout's qacc (with constraints, without them, with every output) and two rollouts from the
current state with CUDA events on the batch's stream, in alternating order.  The rollouts: "rollout", 8 intervals of frame_skip substeps,
reported per interval (the physics of one env step); "rollout_1", frame_skip intervals of one substep, reported per call (the same physics).  Prints medians (and min / max) in microseconds and the
GPU name, power limit and SM clock read through nvidia-smi's query interface (read-only).  Writes nothing unless --out is given.

The "ik" case (MyoVecEnv.ik, myo_batch_ik): the hand, 4096 envs, the five fingertip sites, targets from forward kinematics of random
in-range configurations, start at qpos0, in alternating order with one env step: "ik" at the default parameters (per call, with the mean
and largest number of iterations), "ik_10" (tol = 0, max_iter = 10: every env runs 10 iterations) and "jac_site" (max_iter = 0).  Per
iteration = (ik_10 - jac_site) / 10.  Beside them, the C reference (tests/ik_oracle.c, oracle_ik) at the same defaults on one host core
for the first --ref-envs targets.

The "fd" case (MyoVecEnv.transition_fd, myo_batch_transition_fd): the hand, 4096 envs, in alternating order with one env step: forward
and centred A and B at substeps 1 and frame_skip, and the host loop of rollout calls (one per column) that the rollout API alone allows
for the same forward A and B at substeps 1; then the single env (MyoEnv.mjd_transitionFD, the device call alone, the host loop) on the
hand and the legs, beside the C reference (tests/fd_oracle.c) on one host core.  --fd-reps rounds (x4 for the single env).

The "inverse_fd" case (MyoVecEnv.inverse_fd, myo_batch_inverse_fd): the hand pose at 4096 envs, the hold and the legs (walk) at 2048, the
elbow at 4096 and the torso at 661, at the readout's qacc, in alternating order with one env step: all three blocks with constraints,
without them and with actuation, and the host loop that inverse() alone allows for the same Jacobians: 3 nv + 1 inverse() calls (hinge and
slide qpos columns only; a free joint's rotation would need its quaternion update on the host as well), each after setting the bound state
or qacc of its column, with the bound state restored at the end.  --fd-reps rounds.
--cases selects cases by name (the fd and inverse_fd cases run only when named)."""
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
IK_ENV, IK_N, IK_SITES = "myoHandPoseRandom-v0", 4096, ("THtip", "IFtip", "MFtip", "RFtip", "LFtip")


def gpu_info():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                                     "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception as e:          # (the numbers still print; the machine line says why it is missing)
        return ["unknown (%s)" % e]


def _timed(stream, fn):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3


def ik_case(args):
    """one IK call, one iteration and jac_site beside one env step on the hand; the C reference on one host core"""
    import time
    import numpy as np
    import torch
    from myosuite_b200 import blob, program, vec_env
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ik_oracle import IkOracle
    env = vec_env.MyoVecEnv(IK_ENV, IK_N, seed=0)
    m, n = env.mj_model, IK_N
    env.reset(seed=0)
    stream = torch.cuda.current_stream(env.device)
    g = torch.Generator(device="cpu").manual_seed(0)
    acts = [(torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device) for _ in range(8)]
    sites = [m.name2id("site", x) for x in IK_SITES]
    rng = np.random.default_rng(0)
    qt = np.tile(m.qpos0, (n, 1))
    for j in range(m.njnt):
        if m.jnt_type[j] in (2, 3) and m.jnt_limited[j]:
            qt[:, m.jnt_qposadr[j]] = rng.uniform(*m.jnt_range[j], n)
    dev = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=env.device)
    q0 = dev(np.tile(m.qpos0, (n, 1)))
    tp = env.jac_site(sites, qpos=dev(qt))[2].contiguous()
    calls = {"step": lambda k: env.step(acts[k % 8]), "ik": lambda k: env.ik(sites, tp, qpos_init=q0),
             "ik_10": lambda k: env.ik(sites, tp, qpos_init=q0, max_iter=10, tol=0.0), "jac_site": lambda k: env.jac_site(sites, qpos=q0)}
    for k in range(args.warmup):
        for f in calls.values():
            f(k)
    torch.cuda.synchronize()
    order = list(calls)
    t = {k: [] for k in order}
    for r in range(args.reps):
        for k in (order if r % 2 == 0 else order[::-1]):
            t[k].append(_timed(stream, lambda: calls[k](r)))
    s = {k: dict(median_us=float(np.median(v)), min_us=float(np.min(v)), max_us=float(np.max(v))) for k, v in t.items()}
    it = env.ik(sites, tp, qpos_init=q0, fields=("niter", "converged"))
    niter = it["niter"].cpu().numpy()
    s["ik"].update(mean_iter=float(niter.mean()), max_iter=int(niter.max()), converged=float(it["converged"].float().mean()))
    s["per_iteration_us"] = (s["ik_10"]["median_us"] - s["jac_site"]["median_us"]) / 10
    for k in order[1:]:
        s[k]["per_step"] = s[k]["median_us"] / s["step"]["median_us"]
    # the C reference on one host core, same targets and defaults
    prog, _ = program.build_program(m)
    I, D = blob.pack(m, prog)
    o = IkOracle(I, D, m.site_quat)
    TP = tp.cpu().numpy()
    t0, iters = time.perf_counter(), 0
    for e in range(args.ref_envs):
        iters += o.ik(sites, TP[e], m.qpos0)["niter"]
    dt = time.perf_counter() - t0
    s["c_reference"] = dict(envs=args.ref_envs, us_per_call=dt / args.ref_envs * 1e6, us_per_iteration=dt / max(iters, 1) * 1e6)
    print("ik            n %4d  step %8.1f us | ik %8.1f us (%.3f step; iterations mean %.1f, max %d, converged %.4f) | ik_10 %8.1f us | "
          "jac_site %7.1f us (%.3f step) | per iteration %6.1f us | C reference, one core: %.0f us per env call, %.1f us per iteration"
          % (n, s["step"]["median_us"], s["ik"]["median_us"], s["ik"]["per_step"], s["ik"]["mean_iter"], s["ik"]["max_iter"], s["ik"]["converged"],
             s["ik_10"]["median_us"], s["jac_site"]["median_us"], s["jac_site"]["per_step"], s["per_iteration_us"],
             s["c_reference"]["us_per_call"], s["c_reference"]["us_per_iteration"]), flush=True)
    return dict(env_id=IK_ENV, n_env=n, sites=list(IK_SITES), **s)


FD_ENV, FD_N, FD_SINGLE = "myoHandPoseRandom-v0", 4096, (("hand", "myoHandPoseRandom-v0"), ("legs", "myoLegWalk-v0"))


def _fd_host_loop(env, ctrl, substeps):
    """forward-difference A and B the way the rollout API alone allows: one rollout per column from a host-built perturbed start (hinge /
    slide qpos, qvel, act and ctrl columns; a free joint's rotation would need its quaternion update on the host as well)"""
    import numpy as np
    import torch
    m, eps = env.mj_model, 1e-6
    nv, na = m.nv, m.na
    S = {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart")}
    roll = lambda st, c: env.rollout(c[:, None].contiguous(), substeps=substeps, initial_state=st, fields=("qpos", "qvel", "act"))
    R0 = roll(S, ctrl)
    x0 = torch.cat([R0["qpos"][:, 0], R0["qvel"][:, 0], R0["act"][:, 0]], 1)
    cols = []
    for j in range(2 * nv + na + m.nu):
        st, c = dict(S), ctrl
        if j < nv:
            q = S["qpos"].clone(); st["qpos"] = q
            jn = int(np.nonzero(m.jnt_dofadr <= j)[0][-1]); qa, k = m.jnt_qposadr[jn], j - m.jnt_dofadr[jn]
            if m.jnt_type[jn] != 0 or k < 3:
                q[:, qa + k] += eps
            else:           # a free joint's rotation: q <- q (cos eps/2, e_k sin eps/2), normalised (mj_integratePos)
                w = q[:, qa + 3:qa + 7].clone(); r = torch.zeros(4, dtype=q.dtype, device=q.device)
                r[0], r[k - 2] = np.cos(eps / 2), np.sin(eps / 2)
                prod = torch.stack([w[:, 0] * r[0] - (w[:, 1:] * r[1:]).sum(1)] + [w[:, 0] * r[1 + i] + r[0] * w[:, 1 + i] for i in range(3)], 1)
                prod[:, 1:] += torch.cross(w[:, 1:], r[1:].expand(len(w), 3), dim=1)
                q[:, qa + 3:qa + 7] = prod / prod.norm(dim=1, keepdim=True)
        elif j < 2 * nv:
            v = S["qvel"].clone(); v[:, j - nv] += eps; st["qvel"] = v
        elif j < 2 * nv + na:
            a = S["act"].clone(); a[:, j - 2 * nv] += eps; st["act"] = a
        else:
            c = ctrl.clone(); c[:, j - 2 * nv - na] += eps
        R = roll(st, c)
        cols.append((torch.cat([R["qpos"][:, 0], R["qvel"][:, 0], R["act"][:, 0]], 1) - x0) * (1 / eps))
    return torch.stack(cols, 2)


def fd_case(args):
    """transition_fd beside one env step: the hand batch (forward and centred, substeps 1 and frame_skip), the host loop of rollouts over
    the columns, the single env on the hand and the legs, and the C reference (tests/fd_oracle.c) on one host core"""
    import time
    import numpy as np
    import torch
    from myosuite_b200 import vec_env
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from fd_oracle import FdOracle
    out = {}
    env = vec_env.MyoVecEnv(FD_ENV, FD_N, seed=0)
    m, n, fs = env.mj_model, FD_N, env.frame_skip
    env.reset(seed=0)
    stream = torch.cuda.current_stream(env.device)
    g = torch.Generator(device="cpu").manual_seed(0)
    acts = [(torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device) for _ in range(8)]
    for k in range(4):
        env.step(acts[k])
    ctrl = torch.rand(n, m.nu, generator=g, dtype=torch.float64).to(env.device)
    calls = {"step": lambda k: env.step(acts[k % 8]),
             "fd_fwd_1": lambda k: env.transition_fd(ctrl), "fd_ctr_1": lambda k: env.transition_fd(ctrl, centered=True),
             "fd_fwd_fs": lambda k: env.transition_fd(ctrl, substeps=fs), "fd_ctr_fs": lambda k: env.transition_fd(ctrl, centered=True, substeps=fs),
             "host_loop_fwd_1": lambda k: _fd_host_loop(env, ctrl, 1)}
    for k in range(2):
        for f in calls.values():
            f(k)
    torch.cuda.synchronize()
    order = list(calls)
    t = {k: [] for k in order}
    for r in range(args.fd_reps):
        for k in (order if r % 2 == 0 else order[::-1]):
            t[k].append(_timed(stream, lambda: calls[k](r)))
    s = {k: dict(median_us=float(np.median(v)), min_us=float(np.min(v)), max_us=float(np.max(v))) for k, v in t.items()}
    for k in order[1:]:
        s[k]["per_step"] = s[k]["median_us"] / s["step"]["median_us"]
    out["batch"] = dict(env_id=FD_ENV, n_env=n, frame_skip=fs, columns=2 * m.nv + m.na + m.nu, **s)
    print("fd batch      n %4d  step %8.1f us | " % (n, s["step"]["median_us"]) + "  ".join("%s %9.1f us (%.2f step)" % (k, s[k]["median_us"], s[k]["per_step"]) for k in order[1:]), flush=True)
    del env, calls
    torch.cuda.empty_cache()
    for name, eid in FD_SINGLE:
        one = vec_env.MyoEnv(eid, seed=0)
        one.reset()
        v = one.vec
        c1 = torch.rand(1, v.mj_model.nu, generator=g, dtype=torch.float64).to(v.device)
        st = torch.cuda.current_stream(v.device)
        calls = {"mjd_transitionFD": lambda k: one.mjd_transitionFD(c1[0].cpu().numpy()), "fd_device": lambda k: v.transition_fd(c1),
                 "host_loop": lambda k: _fd_host_loop(v, c1, 1)}
        for k in range(2):
            for f in calls.values():
                f(k)
        torch.cuda.synchronize()
        t = {k: [] for k in calls}
        for r in range(args.fd_reps * 4):
            for k in (list(calls) if r % 2 == 0 else list(calls)[::-1]):
                t[k].append(_timed(st, lambda: calls[k](r)))
        s = {k: dict(median_us=float(np.median(x)), min_us=float(np.min(x)), max_us=float(np.max(x))) for k, x in t.items()}
        o = FdOracle(v.I, v.D)
        o.reset(); o.set(qpos=v.t["qpos"][0].cpu().numpy(), qvel=v.t["qvel"][0].cpu().numpy(), act=v.t["act"][0].cpu().numpy())
        t0 = time.perf_counter()
        for _ in range(3):
            o.transition_fd(c1[0].cpu().numpy())
        s["c_reference_us"] = (time.perf_counter() - t0) / 3 * 1e6
        out["single_" + name] = dict(env_id=eid, **s)
        print("fd single %-4s  mjd_transitionFD %8.1f us | device call %8.1f us | host loop of rollouts %9.1f us | C reference, one core %10.1f us"
              % (name, s["mjd_transitionFD"]["median_us"], s["fd_device"]["median_us"], s["host_loop"]["median_us"], s["c_reference_us"]), flush=True)
        del one, v
    return out


IFD_CASES = (("hand_pose", "myoHandPoseRandom-v0", 4096), ("hold", "myoHandObjHoldRandom-v0", 2048), ("walk", "myoLegWalk-v0", 2048),
             ("elbow", "myoElbowPose1D6MRandom-v0", 4096), ("torso", "myoTorsoPoseFixed-v0", 661))


def _ifd_host_loop(env, qacc):
    """DfDq (hinge / slide columns), DfDv and DfDa the way inverse() alone allows: one call per column after setting the bound qpos, qvel
    or the qacc of that column, then the bound state restored"""
    import torch
    m, eps = env.mj_model, 1e-6
    keep = {k: env.t[k].clone() for k in ("qpos", "qvel")}
    f0 = env.inverse(qacc)["qfrc_inverse"].clone()
    cols = []
    for j in range(m.njnt):
        if m.jnt_type[j] in (2, 3):
            env.t["qpos"][:, m.jnt_qposadr[j]] += eps
            cols.append((env.inverse(qacc)["qfrc_inverse"] - f0) * (1 / eps))
            env.t["qpos"].copy_(keep["qpos"])
    for i in range(m.nv):
        env.t["qvel"][:, i] += eps
        cols.append((env.inverse(qacc)["qfrc_inverse"] - f0) * (1 / eps))
        env.t["qvel"].copy_(keep["qvel"])
    for i in range(m.nv):
        a = qacc.clone(); a[:, i] += eps
        cols.append((env.inverse(a)["qfrc_inverse"] - f0) * (1 / eps))
    return torch.stack(cols, 1)


def inverse_fd_case(args):
    """inverse_fd beside one env step and beside the host loop of inverse() calls, on every IFD_CASES batch"""
    import numpy as np
    import torch
    from myosuite_b200 import vec_env
    out = {}
    for name, eid, n in IFD_CASES:
        env = vec_env.MyoVecEnv(eid, n, seed=0)
        m = env.mj_model
        env.reset(seed=0)
        stream = torch.cuda.current_stream(env.device)
        g = torch.Generator(device="cpu").manual_seed(0)
        acts = [(torch.rand(n, m.nu, generator=g) * 2 - 1).to(env.device) for _ in range(8)]
        for k in range(4):
            env.step(acts[k])
        qacc = env.data("qacc")["qacc"].clone()
        hinge = sum(1 for j in range(m.njnt) if m.jnt_type[j] in (2, 3))
        calls = {"step": lambda k: env.step(acts[k % 8]),
                 "inverse_fd": lambda k: env.inverse_fd(qacc), "inverse_fd_free": lambda k: env.inverse_fd(qacc, constraints=False),
                 "inverse_fd_actuation": lambda k: env.inverse_fd(qacc, actuation=True), "host_loop": lambda k: _ifd_host_loop(env, qacc)}
        for k in range(2):
            for f in calls.values():
                f(k)
        torch.cuda.synchronize()
        order = list(calls)
        t = {k: [] for k in order}
        for r in range(args.fd_reps):
            for k in (order if r % 2 == 0 else order[::-1]):
                t[k].append(_timed(stream, lambda: calls[k](r)))
        s = {k: dict(median_us=float(np.median(v)), min_us=float(np.min(v)), max_us=float(np.max(v))) for k, v in t.items()}
        for k in order[1:]:
            s[k]["per_step"] = s[k]["median_us"] / s["step"]["median_us"]
        s["host_loop_calls"] = 1 + hinge + 2 * m.nv
        out[name] = dict(env_id=eid, n_env=n, nv=m.nv, **s)
        print("inverse_fd %-9s n %4d nv %2d  step %8.1f us | " % (name, n, m.nv, s["step"]["median_us"])
              + "  ".join("%s %9.1f us (%.2f step)" % (k, s[k]["median_us"], s[k]["per_step"]) for k in order[1:])
              + " | host loop: %d calls, %.1fx the device call" % (s["host_loop_calls"], s["host_loop"]["median_us"] / s["inverse_fd"]["median_us"]), flush=True)
        del env, calls
        torch.cuda.empty_cache()
    return out


def main():
    import numpy as np
    import torch
    from myosuite_b200 import vec_env
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default=",".join([c[0] for c in CASES] + ["ik"]))
    ap.add_argument("--ref-envs", type=int, default=64)
    ap.add_argument("--fd-reps", type=int, default=5)
    args = ap.parse_args()
    want = set(args.cases.split(","))
    res = {"gpu_before": gpu_info(), "cases": {}}
    for name, eid, n in CASES:
        if name not in want:
            continue
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
    if "ik" in want:
        res["cases"]["ik"] = ik_case(args)
    if "fd" in want:
        res["cases"]["fd"] = fd_case(args)
    if "inverse_fd" in want:
        res["cases"]["inverse_fd"] = inverse_fd_case(args)
    res["gpu_after"] = gpu_info()
    print("GPU [name, power limit, SM clock, max SM clock, throttle reasons] before: %s after: %s" % (res["gpu_before"], res["gpu_after"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
