"""GPU parity + timing probe (developer tool; needs a GPU).  Compares the CUDA path with the CPU oracle."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np, torch
from myosuite_b200 import vec_env, blob
from oracle.oracle_py import Oracle

def relerr(a, b):
    return float(np.max(np.abs(a - b) / (np.abs(b) + 1e-6 * max(1.0, np.abs(b).max()))))

def probe(env_id, n=64, seed=0, substeps=10):
    env = vec_env.MyoVecEnv(env_id, n, taps=True)
    m = env.mj_model
    rng = np.random.default_rng(seed)
    lo, hi = m.jnt_range[:, 0], m.jnt_range[:, 1]
    qpos = np.tile(m.qpos0, (n, 1))
    for j in range(m.njnt):
        if m.jnt_type[j] != 0:
            span = hi[j] - lo[j]
            qpos[:, m.jnt_qposadr[j]] = rng.uniform(lo[j] - 0.02 * span, hi[j] + 0.02 * span, n)
    qvel = rng.normal(0, 1.0, (n, m.nv)); act = rng.uniform(0, 1, (n, m.na)); ctrl = rng.uniform(0, 1, (n, m.nu))
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, 0)
    torch.cuda.synchronize()
    t = {k: v.cpu().numpy() for k, v in env.t.items() if k.startswith("tap_")}
    o = Oracle(env.I, env.D)
    errs = dict(qacc=0, force=0, len=0, qM=0, fsm=0); ncon_mis = 0; maxcon = 0; maxit = 0
    for e in range(n):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.forward()
        errs["qacc"] = max(errs["qacc"], relerr(t["tap_qacc"][e], o.f("qacc")))
        errs["force"] = max(errs["force"], relerr(t["tap_actuator_force"][e], o.f("actuator_force")))
        errs["len"] = max(errs["len"], relerr(t["tap_ten_length"][e], o.f("actuator_length")))
        errs["qM"] = max(errs["qM"], relerr(t["tap_qM"][e], o.f("qM")))
        errs["fsm"] = max(errs["fsm"], relerr(t["tap_qfrc_smooth"][e], o.f("qfrc_smooth")))
        sup = set(env.prog_info["pair_model_index"])
        ocon = [p for p in o.i("con_pair") if p in sup]
        gcon = [env.prog_info["pair_model_index"][p] for p in t["tap_contact_pair"][e][:t["tap_ncon"][e, 0]]]
        if list(ocon) != list(gcon): ncon_mis += 1
        maxcon = max(maxcon, t["tap_ncon"][e, 0]); maxit = max(maxit, t["tap_ncon"][e, 2])
    print(env_id, "forward parity (max rel err over %d envs):" % n, {k: "%.2e" % v for k, v in errs.items()}, "contact-list mismatches", ncon_mis, "max ncon", maxcon, "max newton it", maxit, flush=True)
    # multi-substep rollout parity
    env.set_state(qpos=qpos, qvel=qvel, act=act)
    env.forward_debug(ctrl, substeps); torch.cuda.synchronize()
    gq, gv, ga = env.t["qpos"].cpu().numpy(), env.t["qvel"].cpu().numpy(), env.t["act"].cpu().numpy()
    eq = ev = ea = 0
    for e in range(min(n, 16)):
        o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=act[e], ctrl=ctrl[e]); o.step(substeps)
        eq = max(eq, float(np.abs(gq[e] - o.f("qpos")).max())); ev = max(ev, relerr(gv[e], o.f("qvel"))); ea = max(ea, float(np.abs(ga[e, :m.na] - o.f("act")).max()))
    print("   %d-substep rollout: |dqpos| %.2e  rel dqvel %.2e  |dact| %.2e" % (substeps, eq, ev, ea), flush=True)
    return env

def timing(env_id, n=4096, steps=50):
    env = vec_env.MyoVecEnv(env_id, n)
    env.reset(seed=1)
    a = torch.rand(n, env.act_dim, device=env.device) * 2 - 1
    for _ in range(5): env.step(a)
    torch.cuda.synchronize(); t0 = time.time()
    for _ in range(steps): env.step(a)
    torch.cuda.synchronize(); dt = time.time() - t0
    print(env_id, "n=%d: %.1f ms/step, %.0f env-steps/s; smem/env %d B, warps/cta %s" % (n, dt / steps * 1e3, n * steps / dt, env.dims.smem_bytes_per_env, "?"),
          "mean reward %.3f done %.3f" % (env.t["reward"].mean().item(), env.t["done"].float().mean().item()), flush=True)

if __name__ == "__main__":
    for eid in ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0"]:
        probe(eid)
    for eid in ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0"]:
        timing(eid)
