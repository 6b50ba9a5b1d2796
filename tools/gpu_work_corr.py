"""How predictable is an env's solver work from its previous step?  (developer probe for work-sorted env placement; needs a GPU)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from myosuite_b200 import vec_env
n, steps = 4096, 40
env = vec_env.MyoVecEnv("myoHandPoseRandom-v0", n, taps=True); env.reset(seed=0)
g = torch.Generator(device=env.device).manual_seed(0)
W = []
for s in range(steps):
    env.step(torch.rand(n, env.act_dim, device=env.device, generator=g) * 2 - 1)
    pc = env.t["tap_phase_cycles"].cpu().numpy()
    W.append(np.stack([pc[:, 6], pc[:, 14], pc[:, 4], pc[:, 12]], 1).astype(np.float64))   # solve cycles, newton iterations, collision cycles, max ncon
W = np.stack(W)   # steps, n, 4
for k, name in enumerate(["solve cycles", "newton iterations", "collision cycles", "max ncon"]):
    a, b = W[10:-1, :, k].ravel(), W[11:, :, k].ravel()
    print(name, "mean %.1f std %.1f  lag-1 corr %.3f" % (a.mean(), a.std(), np.corrcoef(a, b)[0, 1]))
# simulated lockstep cost of the solve: groups of 10 envs, cost = max over the group (per step; a proxy for per substep)
def cost(order, x): 
    m = (len(order) // 10) * 10
    return x[order[:m]].reshape(-1, 10).max(1).sum()
tot_id = tot_sorted = tot_ideal = 0
for s in range(11, steps):
    x = W[s, :, 0]; tot_id += cost(np.arange(n), x); tot_sorted += cost(np.argsort(W[s - 1, :, 0]), x); tot_ideal += cost(np.argsort(x), x)
print("sum over groups of max solve cycles: identity %.3g  sorted-by-previous-step %.3g (%.1f%%)  oracle sort %.3g (%.1f%%)  mean*10 %.3g" %
      (tot_id, tot_sorted, 100 * tot_sorted / tot_id, tot_ideal, 100 * tot_ideal / tot_id, W[11:, :, 0].sum()))
