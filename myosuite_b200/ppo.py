"""On-device PPO over MyoVecEnv (SURVEY.md section 8f-2): the zero-copy policy path.

What the reference does: SB3 PPO over `make_vec_env` on host processes (agents/sb3_job_script.py:49-70, hydra_myo_sb3_ppo_config.yaml), and brax
PPO over the MJX envs in its training benchmark (benchmarks/mjx_benchmark_PPO.py:17-62 with myosuite/envs/myo/mjx/__init__.py:43-67: lr 3e-4,
discount 0.97, GAE lambda 0.95, entropy 1e-3, clip 0.3, grad-norm 1.0, unroll 10, 8 updates x 32 minibatches per batch, normalised
observations, 3 x 64 tanh... networks).  Here the rollout is the fused env kernel, observations / actions / rewards / advantages are torch CUDA
tensors that never leave HBM, and the networks are plain torch modules trained with autograd (library code: the network is not the hot path
of this repository, the simulator is).  Defaults follow the reference's MJX PPO configuration.

Time-limit truncation: MyoVecEnv auto-resets inside the step, so the observation after a `done | truncated` step already belongs to the next
episode, and both end the GAE recursion.  By default that is all (like SB3 without terminal-observation bootstrapping): a truncated episode
is valued as if its last state were terminal.  With PPO(..., bootstrap_truncated=True) (`--bootstrap_truncated`) a step that is truncated
but not terminated adds gamma V(s_T) to its TD target, V evaluated on the state the episode ended in (the step's info["final_obs"]).
"""
import math
import time


def gae(rewards, values, dones, last_value, gamma, lam, boot=None):
    """Generalised advantage estimate.  rewards / values / dones: [T, n] (dones[t] = episode ended BY step t); last_value: [n] = V(obs after
    the last step).  boot: None, or (boot_mask [T, n], final_values [T, n]) to bootstrap episodes cut by the time limit: where boot_mask[t]
    is set (truncated and not terminated), the TD target of step t gains gamma final_values[t] = gamma V(the state the episode ended in);
    final_values must be finite (zero, say) where the mask is clear.  The recursion still stops at dones[t].  Returns (advantages [T, n],
    returns [T, n])."""
    import torch
    T = rewards.shape[0]
    adv = torch.zeros_like(rewards)
    nxt, run = last_value, torch.zeros_like(last_value)
    for t in range(T - 1, -1, -1):
        live = 1.0 - dones[t].to(rewards.dtype)
        delta = rewards[t] + gamma * nxt * live - values[t]
        if boot is not None:
            delta = delta + gamma * (boot[0][t].to(rewards.dtype) * boot[1][t])
        run = delta + gamma * lam * live * run
        adv[t] = run
        nxt = values[t]
    return adv, adv + values


class RunningNorm:
    """Running mean / variance of the observations (Welford over batches), on the device."""

    def __init__(self, dim, device):
        import torch
        self.torch = torch
        self.mean, self.var, self.count = torch.zeros(dim, device=device), torch.ones(dim, device=device), 1e-4

    def update(self, x):
        x = x.reshape(-1, x.shape[-1])
        bm, bv, bc = x.mean(0), x.var(0, unbiased=False), x.shape[0]
        d, tot = bm - self.mean, self.count + bc
        self.mean = self.mean + d * (bc / tot)
        self.var = (self.var * self.count + bv * bc + d * d * (self.count * bc / tot)) / tot
        self.count = tot

    def __call__(self, x):
        return ((x - self.mean) / (self.var + 1e-8).sqrt()).clamp(-10.0, 10.0)


def _mlp(torch, sizes, out_gain):
    layers = []
    for i in range(len(sizes) - 1):
        lin = torch.nn.Linear(sizes[i], sizes[i + 1])
        torch.nn.init.orthogonal_(lin.weight, gain=out_gain if i == len(sizes) - 2 else math.sqrt(2.0))
        torch.nn.init.zeros_(lin.bias)
        layers.append(lin)
        if i < len(sizes) - 2:
            layers.append(torch.nn.Tanh())
    return torch.nn.Sequential(*layers)


class PPO:
    def __init__(self, env, hidden=(64, 64, 64), lr=3e-4, gamma=0.97, lam=0.95, clip=0.3, entropy=1e-3, vf_coef=0.5, max_grad_norm=1.0,
                 unroll=10, epochs=8, minibatches=32, init_log_std=-0.5, normalize_obs=True, seed=0, bootstrap_truncated=False):
        import torch
        if not env.cfg.auto_reset:
            raise ValueError("PPO needs MyoVecEnv(..., auto_reset=True)")
        self.torch, self.env, self.dev = torch, env, env.device
        torch.manual_seed(seed)
        self.gen = torch.Generator(device=self.dev).manual_seed(seed)
        self.gamma, self.lam, self.clip, self.entropy, self.vf_coef, self.max_grad_norm = gamma, lam, clip, entropy, vf_coef, max_grad_norm
        self.unroll, self.epochs, self.minibatches = int(unroll), int(epochs), int(minibatches)
        self.bootstrap_truncated = bool(bootstrap_truncated)
        od, ad = env.obs_dim, env.act_dim
        self.pi = _mlp(torch, (od, *hidden, ad), 0.01).to(self.dev)
        self.vf = _mlp(torch, (od, *hidden, 1), 1.0).to(self.dev)
        self.log_std = torch.nn.Parameter(torch.full((ad,), float(init_log_std), device=self.dev))
        self.opt = torch.optim.Adam(list(self.pi.parameters()) + list(self.vf.parameters()) + [self.log_std], lr=lr, eps=1e-5)
        self.norm = RunningNorm(od, self.dev) if normalize_obs else None
        self.obs, _ = env.reset(seed=seed)
        self.total_steps, self.ep_ret = 0, torch.zeros(env.num_envs, device=self.dev)
        self.finished_returns = []

    # ---------------------------------------------------------------- policy
    def _n(self, obs):
        return self.norm(obs) if self.norm is not None else obs

    def _logp(self, mean, a):
        std = self.log_std.exp()
        return (-0.5 * ((a - mean) / std) ** 2 - self.log_std - 0.5 * math.log(2 * math.pi)).sum(-1)

    def act(self, obs, mode="evaluation", generator=None, clip=True):
        """rollout.examine_policy-compatible: batched action on the device."""
        torch = self.torch
        with torch.no_grad():
            a = self.pi(self._n(obs))
            if mode == "exploration":
                a = a + self.log_std.exp() * torch.randn(a.shape, device=a.device, generator=generator or self.gen)
        return a.clamp(-1.0, 1.0) if clip else a

    # ---------------------------------------------------------------- one iteration: unroll, GAE, clipped-surrogate updates
    def collect(self):
        torch, env, T, n = self.torch, self.env, self.unroll, self.env.num_envs
        O = torch.zeros(T, n, env.obs_dim, device=self.dev); A = torch.zeros(T, n, env.act_dim, device=self.dev)
        R = torch.zeros(T, n, device=self.dev); D = torch.zeros(T, n, dtype=torch.bool, device=self.dev)
        if self.bootstrap_truncated:          # truncated-not-terminated mask and the observations those episodes ended in
            B = torch.zeros(T, n, dtype=torch.bool, device=self.dev); FO = torch.zeros(T, n, env.obs_dim, device=self.dev)
        with torch.no_grad():
            for t in range(T):
                O[t] = self.obs
                mean = self.pi(self._n(self.obs))
                A[t] = mean + self.log_std.exp() * torch.randn(mean.shape, device=self.dev, generator=self.gen)
                obs, rew, done, trunc, info = env.step(A[t].clamp(-1.0, 1.0))          # the env clips like the reference's action space does
                R[t], D[t] = rew, done.bool() | trunc.bool()
                if self.bootstrap_truncated:
                    B[t] = trunc.bool() & ~done.bool()
                    FO[t] = info["final_obs"]          # (rows outside done | truncated are stale or NaN; masked out below)
                self.obs = obs
                self.ep_ret += rew
                if bool(D[t].any()):
                    self.finished_returns.append(self.ep_ret[D[t]].clone())
                    self.ep_ret[D[t]] = 0.0
            if self.norm is not None:
                self.norm.update(O)
            No = self._n(O)
            V = self.vf(No).squeeze(-1)
            logp = self._logp(self.pi(No), A)
            last_v = self.vf(self._n(self.obs)).squeeze(-1)
            boot = None
            if self.bootstrap_truncated:          # V of the final states, normalised like the unroll's observations
                boot = (B, torch.where(B, self.vf(self._n(FO)).squeeze(-1), 0.0))
            adv, ret = gae(R, V, D, last_v, self.gamma, self.lam, boot)
        self.total_steps += T * n
        return dict(obs=No.reshape(T * n, -1), act=A.reshape(T * n, -1), logp=logp.reshape(-1), adv=adv.reshape(-1), ret=ret.reshape(-1), rew=R)

    def update(self, batch):
        torch = self.torch
        N = batch["adv"].shape[0]; mb = max(N // self.minibatches, 1)
        stats = {}
        for _ in range(self.epochs):
            perm = torch.randperm(N, device=self.dev, generator=self.gen)
            for k in range(0, N - mb + 1, mb):
                i = perm[k:k + mb]
                adv = batch["adv"][i]; adv = (adv - adv.mean()) / (adv.std() + 1e-8)
                logp = self._logp(self.pi(batch["obs"][i]), batch["act"][i])
                ratio = (logp - batch["logp"][i]).exp()
                pg = -torch.min(ratio * adv, ratio.clamp(1 - self.clip, 1 + self.clip) * adv).mean()
                v = self.vf(batch["obs"][i]).squeeze(-1)
                vl = 0.5 * (v - batch["ret"][i]).pow(2).mean()
                ent = (self.log_std + 0.5 * math.log(2 * math.pi * math.e)).sum()
                loss = pg + self.vf_coef * vl - self.entropy * ent
                self.opt.zero_grad(set_to_none=True)
                loss.backward()
                torch.nn.utils.clip_grad_norm_(list(self.pi.parameters()) + list(self.vf.parameters()) + [self.log_std], self.max_grad_norm)
                self.opt.step()
        stats.update(policy_loss=float(pg.detach()), value_loss=float(vl.detach()), entropy=float(ent.detach()))
        return stats

    def train(self, total_timesteps, log=None):
        """Train for >= total_timesteps env-steps.  Returns a list of per-iteration dicts (steps, mean reward per step of the unroll, mean return
        of the episodes that finished, wall-clock env-steps/s including the updates)."""
        torch, hist, t0 = self.torch, [], time.perf_counter()
        while self.total_steps < total_timesteps:
            batch = self.collect()
            st = self.update(batch)
            torch.cuda.current_stream(self.dev).synchronize()
            fin = torch.cat(self.finished_returns) if self.finished_returns else None
            self.finished_returns = []
            row = dict(steps=self.total_steps, reward_per_step=float(batch["rew"].mean()), episode_return=float(fin.mean()) if fin is not None and fin.numel() else None,
                       steps_per_s=self.total_steps / (time.perf_counter() - t0), **st)
            hist.append(row)
            if log:
                log(row)
        return hist


if __name__ == "__main__":      # python -m myosuite_b200.ppo --env myoElbowPose1D6MRandom-v0 --num_envs 8192 --num_timesteps 5000000
    # (the measurement of the reference's benchmarks/mjx_benchmark_PPO.py:17-62: wall-clock of PPO training for a fixed number of env-steps)
    import argparse
    from myosuite_b200 import vec_env
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="myoElbowPose1D6MRandom-v0"); ap.add_argument("--num_envs", type=int, default=8192)
    ap.add_argument("--num_timesteps", type=int, default=5_000_000); ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--bootstrap_truncated", action="store_true", help="bootstrap time-limit truncations with V(final observation)")
    a = ap.parse_args()
    agent = PPO(vec_env.MyoVecEnv(a.env, a.num_envs, seed=a.seed), seed=a.seed, bootstrap_truncated=a.bootstrap_truncated)
    t0 = time.perf_counter()
    h = agent.train(a.num_timesteps, log=lambda r: print({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))
    print("PPO training for %d total steps on %d envs took %.2f s (%.0f env-steps/s incl. updates)" % (h[-1]["steps"], a.num_envs, time.perf_counter() - t0, h[-1]["steps_per_s"]))
