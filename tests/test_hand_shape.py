"""The step kernel compiled for the hand's shape (myo_env_kernel_w14_hand): its shape header is the model's, batches of that shape run
it and no others do, and it computes bit for bit what the generic launch_bounds(448) kernel computes."""
import os

import numpy as np
import pytest

from myosuite_b200 import shape

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAND = "myoHandPoseRandom-v0"
ROWS = ["p48", "f64"]
KEYS = ("qpos", "qvel", "act", "qacc_warmstart", "time", "obs", "reward", "done", "truncated", "last_return", "episode_count")


def test_hand_shape_header_in_sync():
    assert open(shape.HEADER).read() == shape.emit_header()


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("task", [HAND, "myoHandReachRandom-v0"])
def test_hand_shape_kernel_chosen(task, rows):
    from myosuite_b200 import vec_env
    info = vec_env.MyoVecEnv(task, 4096, row_storage=rows).batch.launch_info()
    assert info["use_w14"] == 1 and info["hand_shape"] == 1, info


@pytest.mark.gpu
@pytest.mark.parametrize("task, n, kw", [(HAND, 4096, {"maxcon": 33}), (HAND, 4096, {"maxcon": 24}), ("myoHandObjHoldRandom-v0", 2048, {})])
def test_hand_shape_kernel_not_chosen(task, n, kw):
    from myosuite_b200 import vec_env
    info = vec_env.MyoVecEnv(task, n, **kw).batch.launch_info()
    assert info["hand_shape"] == 0, info


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
def test_hand_shape_kernel_matches_generic(rows):
    """4096 hand envs at maxcon 32 (the hand's kernel) and at maxcon 33 (the generic launch_bounds(448) kernel), same seed and 10 steps of
    the same actions: every output bit for bit on each env whose contacts never overflowed the smaller capacity."""
    import torch
    from myosuite_b200 import vec_env
    n, nstep = 4096, 10
    envs = {mc: vec_env.MyoVecEnv(HAND, n, seed=5, row_storage=rows, maxcon=mc) for mc in (32, 33)}
    assert envs[32].batch.launch_info()["hand_shape"] == 1 and envs[33].batch.launch_info()["hand_shape"] == 0
    rng = np.random.default_rng(3)
    actions = [torch.as_tensor(rng.uniform(-1, 1, (n, envs[32].mj_model.nu)).astype(np.float32), device=envs[32].device) for _ in range(nstep)]
    out, ov = {}, {}
    for mc, env in envs.items():
        env.reset(seed=5)
        ov[mc] = np.zeros(n, bool)
        for a in actions:
            env.step(a)
            ov[mc] |= env.t["overflow"].cpu().numpy() != 0
        torch.cuda.synchronize()
        out[mc] = {k: env.t[k].cpu().numpy().copy() for k in KEYS}
    ok = np.nonzero(~ov[32] & ~ov[33])[0]
    assert len(ok) >= n // 2, len(ok)
    differ = {k: int((out[32][k][ok] != out[33][k][ok]).sum()) for k in KEYS}
    print("\nhand shape [%s]: %d / %d envs compared over %d steps, differing values %s" % (rows, len(ok), n, nstep, differ))
    assert not any(differ.values()), differ
