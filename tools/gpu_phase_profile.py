"""Per-phase SM-cycle breakdown + contact-count histogram over a rollout (developer tool; needs a GPU)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from myosuite_b200 import vec_env
eid = sys.argv[1] if len(sys.argv) > 1 else "myoHandPoseRandom-v0"
n, steps = int(os.environ.get("N", 4096)), int(os.environ.get("STEPS", 60))
env = vec_env.MyoVecEnv(eid, n, taps=True, maxcon=int(os.environ.get("MAXCON", 0)), profile_waits=bool(int(os.environ.get("WAITS", 0))), solver_tolerance=float(os.environ.get("TOL", 0))); env.reset(seed=0); print("maxcon", env.dims.maxcon, "smem/env", env.dims.smem_bytes_per_env, "const", env.dims.reserved[1])
names = ["kinematics", "tendon", "actuation", "crb+bias", "collision", "constraints", "solve", "taps+integrate"]
tot = np.zeros(8); sub = np.zeros(8); extra = np.zeros(4); hist = np.zeros(64, dtype=np.int64); hefc = []; iters = []
g = torch.Generator(device=env.device).manual_seed(0)
for s in range(steps):
    env.step(torch.rand(n, env.act_dim, device=env.device, generator=g) * 2 - 1)
    pc = env.t["tap_phase_cycles"].cpu().numpy()
    tot += pc[:, :8].sum(0); sub += pc[:, 8:16].sum(0); extra += pc[:, 16:20].sum(0); hist += np.bincount(np.minimum(pc[:, 12], 63), minlength=64); hefc.append(pc[:, 13].copy()); iters.append(env.t["tap_ncon"][:, 2].cpu().numpy().copy())
print(eid, "phase share of cycles:", {k: "%.1f%%" % (100 * v / tot.sum()) for k, v in zip(names, tot)})
print("cycles per substep per env-warp: %.0f ; cooperative collision section %.0f ; whole substep loop %.0f ; integrate: M.a + matrix %.0f, LDL factor+solve %.0f" % tuple(x / (n * steps * env.n_frames) for x in (tot.sum(), extra[0], extra[1], extra[2], extra[3])))
print("solve sub-phases (share of solve):", {k: "%.1f%%" % (100 * v / max(sub[:4].sum(), 1)) for k, v in zip(["gradient", "H assembly", "factor+solve", "linesearch+update"], sub[:4])},
      "newton iters/substep %.2f, dense share %.2f" % (sub[6] / (n * steps * env.n_frames), sub[7] / max(sub[6], 1)))
c = np.cumsum(hist) / hist.sum()
print("max-ncon-in-step histogram (count):", {i: int(h) for i, h in enumerate(hist) if h})
print("P(max ncon <= k): ", {k: "%.4f" % c[k] for k in (0, 2, 4, 6, 8, 10, 12, 16, 20, 24, 31)})
he = np.concatenate(hefc); print("nefc: mean %.1f p50 %d p99 %d max %d" % (he.mean(), np.percentile(he, 50), np.percentile(he, 99), he.max()))
it = np.concatenate(iters); print("newton iterations (last substep): mean %.2f max %d" % (it.mean(), it.max()))
