"""N>1 host logic on CPU (gloo, world_size 2): env-sharding rule and the end-of-rollout gather of episode returns."""
import os
import socket

import numpy as np
import pytest


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, n, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # rank r owns global env ids [r*n, (r+1)*n): the Philox key is (seed, env_offset + local_env, episode) with env_offset = r*n
    env_offset = rank * n
    ids = torch.arange(n) + env_offset
    last_return = ids.float() * 0.5 + 1.0              # stands in for env.t["last_return"] (one value per env)
    gathered = torch.empty(world * n)
    dist.all_gather_into_tensor(gathered, last_return)  # the single collective of the path (SURVEY 8e)
    t = torch.tensor([float(rank + 1)])
    dist.all_reduce(t, op=dist.ReduceOp.MAX)            # bench.py takes the MAX over ranks of the device time
    q.put((rank, gathered.numpy().copy(), float(t[0])))
    dist.destroy_process_group()


def test_env_sharding_and_return_gather_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, n, port = 2, 8, _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    exp = np.arange(world * n) * 0.5 + 1.0
    for rank, g, tmax in res:
        np.testing.assert_array_equal(g, exp)           # every rank sees all returns in global env order, no overlap / gap
        assert tmax == world


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm run beside the GPU arm) prints one JSON line with the contract's keys;
    under torchrun only rank 0 prints.  Runs on the host cores (oracle port), no GPU needed."""
    import json, os, subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MYO_BENCH_CPU_BUDGET_S="0.5")
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "3", "--warmup", "3"], capture_output=True, text=True, env=env, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in line, k
    assert line["impl"] == "reference" and line["value"] > 0 and line["cpu_baseline"]["kind"] == "port" and line["e2e"]["h2d_bytes_per_step"] == 0
    env2 = dict(env, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out2 = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "2"], capture_output=True, text=True, env=env2, timeout=120)
    assert out2.returncode == 0 and out2.stdout.strip() == ""
