"""The product step kernels against the CPU oracle at the launch shapes that are benchmarked.

Every other oracle comparison of a full env step runs either the debug kernel (bound parity taps select it) or a product kernel in a
single round of one small launch.  Here no tap is bound: each case builds a batch at a benchmark size, lets launch_info() confirm which
kernel, how many warps per CTA and how many rounds per CTA the step runs with, steps it from reset with random actions (auto-reset on),
forces a quarter of the envs to hit the TimeLimit on the checked step, and replays the checked step of selected envs on the oracle from
a snapshot of the full env state (warm start, time, fatigue and per-env object sizes included).

The envs are chosen from the slot -> env map the step ran with (the load-sorted permutation, or the fixed map of env_kernel_body) so
that every (round, warp slot) pair is checked in at least two CTAs, together with the last slot, the neighbours of idle slots, the
most contact-heavy envs of a pre-sample, envs that auto-reset on this step and a random sample.  The leg stand cases also reset some
envs right before the checked step: their step starts from the randomised reset state, whose joint couplings are broken, and is held to
the mid-episode bounds too."""
import time

import pytest

from parity_helpers import LAUNCH_ENV, Oracles, replay_product_step  # noqa: F401  (Oracles: imported from here by other modules)

pytestmark = pytest.mark.gpu

HAND = "myoHandPoseRandom-v0"
# case -> (env id, n_env, environment of the library, env kwargs, expected launch_info subset).  The expected shapes are those of the
# launch heuristic of myo_batch_create on an H100 SXM (132 SMs, 227 KB of shared memory per CTA); a change there fails the case.
CASES = {
    "headline": (HAND, 4096, {}, {}, dict(use_w14=1, warps_per_cta=11, rounds=3, regroup=1)),
    "no_regroup": (HAND, 4096, {"MYO_B200_REGROUP": "0"}, {}, dict(use_w14=1, warps_per_cta=11, rounds=3, regroup=0, balanced=1)),
    "kernel320": (HAND, 4096, {"MYO_B200_W14": "0"}, {}, dict(use_w14=0, warps_per_cta=8, rounds=4, regroup=1)),
    "w14_14warps": (HAND, 4096, {"MYO_B200_WARPS_PER_CTA": "14"}, {}, dict(use_w14=1, warps_per_cta=14, rounds=3, regroup=1)),
    "f64rows": (HAND, 4096, {}, {"row_storage": "f64"}, dict(use_w14=1, warps_per_cta=11, rounds=3, regroup=1)),
    "idle_slots": (HAND, 2954, {}, {}, dict(use_w14=1, warps_per_cta=12, rounds=2, regroup=1)),      # 246 groups of 12 + one of 2
    "hold": ("myoHandObjHoldRandom-v0", 2048, {}, {}, dict(use_w14=0, warps_per_cta=8, rounds=2, regroup=1)),
    "walk": ("myoFatiLegWalk-v0", 2048, {}, {}, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1)),
    "reach": ("myoHandReachRandom-v0", 4096, {}, {}, dict(use_w14=1, warps_per_cta=11, rounds=3, regroup=1)),
    "elbow": ("myoElbowPose1D6MRandom-v0", 4096, {}, {}, dict(use_w14=1, warps_per_cta=14, rounds=3, regroup=0, balanced=0)),
    "torso": ("myoTorsoPoseFixed-v0", 661, {}, {}, dict(use_w14=0, warps_per_cta=3, rounds=2, regroup=1)),   # smallest n with 2 rounds
    "stand": ("myoLegStandRandom-v0", 2048, {}, {}, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1)),
    "stand_fatigue": ("myoFatiLegStandRandom-v0", 2048, {}, {}, dict(use_w14=0, warps_per_cta=6, rounds=3, regroup=1)),
}
N_FIRST = {"stand": 48, "stand_fatigue": 48}      # envs reset right before the checked step (0 for the other cases)
REPORT = []


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    print("\nproduct kernels vs oracle (%.0f s for the module):" % (time.time() - t0))
    for line in REPORT:
        print("  " + line)


@pytest.mark.parametrize("case", list(CASES))
def test_product_step_vs_oracle(case, monkeypatch):
    eid, n, lib_env, kw, expect = CASES[case]
    for k in LAUNCH_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in lib_env.items():
        monkeypatch.setenv(k, v)
    replay_product_step(case, eid, n, kw, expect, n_first=N_FIRST.get(case, 0), report=REPORT)
