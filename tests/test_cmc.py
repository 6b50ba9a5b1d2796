"""Computed muscle control on the device (myo_batch_cmc, MyoVecEnv.cmc, MyoEnv.cmc).

CPU: the C ABI's buffer and parameter structs against the binding, and the k-step excitation (bisection over the k-step map of the
activation dynamics) against the oracle's own activation dynamics stepped k times.
GPU, on both row storages where the pattern exists: every row of the call bit-identical to static_opt() and rollout() run from the call's
previous row, at substeps 1 and frame_skip; qacc_des against a numpy restatement; act at the end of a frame_skip interval against a*;
tracking of the hand trajectory fixture and of references the simulator generated itself; batch independence, side effects, launch count
and input checks; the single env.  (tests/test_cmc_reference.py holds the call to a CPU reference of the whole frame.)
"""
import ctypes
import os

import numpy as np
import pytest

import static_opt_ref as R
from parity_helpers import _states
from test_mj_data import CASES, ROWS, SEED, _header_struct, _same
from test_static_opt import CASE_RESERVE, CMC_ENVS, CMC_RESERVE, CMC_STEPS, EXCITE_TOL, KP, KV, RESERVE, SHIPPED, _reference, _zoo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAME_SKIP = 10            # the registered tasks' frame_skip (tasks.configure's default)
QDES_REL, QDES_REL_FREE = 1e-13, 1e-12     # qacc_des against numpy, relative to the row's largest term (free joints: the quaternion log)
CHAIN_ENVS, CHAIN_FRAMES = 64, 8
TRACK_RATIO = 10.0         # pooled RMS tracking error: passive / CMC
SOLVE = ("act_opt", "reserve_force", "lambda", "niter", "converged", "residual")
STATE = ("qpos", "qvel", "act", "qacc", "time")
ALL = ("qacc_des", "ctrl") + SOLVE + STATE
REPORT = {}


# ----------------------------------------------------------------------------- CPU
def test_cmc_buffer_fields_match_header():
    from myosuite_b200 import abi
    fields, decls = _header_struct("myo_cmc_buffers")
    assert len(fields) == decls and abi.CMC_FIELDS == fields
    assert [n for n, _ in abi.MyoCmcBuffers._fields_] == fields and ctypes.sizeof(abi.MyoCmcBuffers) == 8 * len(fields)
    assert set(abi.CMC_SHAPES) == set(fields) - {"ref_qpos", "ref_qvel", "ref_qacc", "kp", "kv", "weight", "reserve", "lambda0", "qpos0", "qvel0",
                                                 "act0", "qacc_warmstart0", "time0", "overflow"}
    src = open(os.path.join(ROOT, "include", "myo_b200.h")).read()
    p = src[src.index("} myo_cmc_buffers;"):]
    assert "typedef struct { int32_t max_iter, substeps; double tol; } myo_cmc_params;" in p
    assert [n for n, _ in abi.MyoCmcParams._fields_] == ["max_iter", "substeps", "tol"]
    assert "myo_batch_cmc" in abi.EXPORTS and "int myo_batch_cmc(" in src


def act_after(m, i, ctrl, act, k):
    for _ in range(k):
        act = R.act_next(m, i, ctrl, act)
    return act


def excitation_k(m, i, act, a, k):
    """the ctrl of muscle i that, held for k steps, takes act to a: bisection over the k-step map, clipped to the control range"""
    lo, hi = R.ctrl_range(m, i)
    if act_after(m, i, hi, act, k) <= a:
        return hi
    if act_after(m, i, lo, act, k) >= a:
        return lo
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if not lo < mid < hi:
            break
        lo, hi = (mid, hi) if act_after(m, i, mid, act, k) < a else (lo, mid)
    return lo if abs(act_after(m, i, lo, act, k) - a) <= abs(act_after(m, i, hi, act, k) - a) else hi


def test_k_step_excitation_reaches_target(models, tmp_path):
    """The k-step excitation, then k oracle steps with ctrl held: act = a* where ctrl is inside the range, and at a range end a* is out of
    reach on that side; k = 1, 5 and frame_skip on every shipped model and on the zoo's MUSCLE model (tausmooth > 0, ctrllimited false)."""
    from myosuite_b200 import blob
    from oracle.oracle_py import Oracle
    rng = np.random.default_rng(SEED)
    z = _zoo(tmp_path)["MUSCLE"]
    cases = [(name, models[name]) + tuple(_states(models[name], 2, rng, overshoot=0.0, vel=0.3)[:3]) for name in SHIPPED]
    cases.append(("zoo/MUSCLE", z["m"], z["qpos"][:2], z["qvel"][:2], z["act"][:2]))
    worst, clipped, inside, smooth = 0.0, 0, 0, 0
    for name, m, qpos, qvel, act in cases:
        o = Oracle(*blob.pack(m))
        for k in (1, 5, FRAME_SKIP):
            for e in range(len(qpos)):
                a0 = np.clip(act[e], 0, 1)
                target = np.clip(a0 + rng.normal(0, 0.1, m.nu), 0, 1)
                target[::4] = rng.uniform(0, 1, len(target[::4]))      # some out of reach within the interval
                ctrl = np.array([excitation_k(m, i, a0[i], target[i], k) for i in range(m.nu)])
                o.reset(); o.set(qpos=qpos[e], qvel=qvel[e], act=a0, ctrl=ctrl); o.step(k)
                got = o.f("act")
                for i in range(m.nu):
                    lo, hi = R.ctrl_range(m, i)
                    smooth += int(m.actuator_dynprm[i, 2] > 0)
                    if lo < ctrl[i] < hi:
                        inside += 1
                        worst = max(worst, abs(got[i] - target[i]))
                        assert abs(got[i] - target[i]) <= EXCITE_TOL, (name, k, i, got[i], target[i])
                    else:
                        clipped += 1
                        assert (ctrl[i] == hi and got[i] <= target[i] + EXCITE_TOL) or (ctrl[i] == lo and got[i] >= target[i] - EXCITE_TOL), \
                            (name, k, i, ctrl[i], got[i], target[i])
    assert clipped > 0 and inside > 0 and smooth > 0
    print("\nk-step excitation: worst |act_k - a*| %.1e on %d unclipped muscles; %d clipped" % (worst, inside, clipped))


# ----------------------------------------------------------------------------- GPU helpers
def _host(D):
    return {k: v.cpu().numpy().copy() for k, v in D.items()}


def _env(case, n, rows="p48", **kw):
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv(CASES[case][0], n, seed=SEED, row_storage=rows, **kw)
    env.reset(seed=SEED)
    return env


def _self_reference(env, T, substeps, seed=SEED):
    """A reference the simulator generated itself: a rollout of smooth random excitations from the env's state x_0.  Row t of the
    reference is the state at the start of frame t (x_0, then the rollout's rows) and the acceleration of that interval.  Returns
    (ref_qpos, ref_qvel, ref_qacc, start, goal): start is x_0 with its velocity perturbed; goal [n, T, nq] the states the frames end at."""
    import torch
    m, n, dev = env.mj_model, env.num_envs, env.device
    g = torch.Generator(device="cpu").manual_seed(seed)
    phase, freq = torch.rand(n, 1, m.nu, generator=g) * 6.283, 0.5 + 2 * torch.rand(n, 1, m.nu, generator=g)
    tt = torch.arange(T, dtype=torch.float64)[None, :, None] * env.mj_model.opt_timestep * substeps
    ctrl = (0.4 + 0.3 * torch.sin(6.283 * freq * tt + phase)).to(torch.float64).to(dev).contiguous()
    x0 = {k: env.t[k].clone() for k in ("qpos", "qvel", "act", "qacc_warmstart", "time")}
    gen = env.rollout(ctrl, substeps=substeps, initial_state=x0)
    ref_qpos = torch.cat([x0["qpos"][:, None], gen["qpos"][:, :-1]], 1).contiguous()
    ref_qvel = torch.cat([x0["qvel"][:, None], gen["qvel"][:, :-1]], 1).contiguous()
    start = dict(x0)
    start["qvel"] = (x0["qvel"] + 0.1 * torch.randn(n, m.nv, generator=g).to(torch.float64).to(dev)).contiguous()
    return ref_qpos, ref_qvel, gen["qacc"].contiguous(), start, gen["qpos"]


def _row_state(out, start, t):
    """the state frame t starts from: the call's row t - 1 (start for t = 0), as rollout()'s initial_state"""
    if t == 0:
        return {k: v.clone() for k, v in start.items()}
    return {"qpos": out["qpos"][:, t - 1].contiguous(), "qvel": out["qvel"][:, t - 1].contiguous(), "act": out["act"][:, t - 1].contiguous(),
            "qacc_warmstart": out["qacc"][:, t - 1].contiguous(), "time": out["time"][:, t - 1].contiguous()}


# ----------------------------------------------------------------------------- GPU: the chain of public calls
def _chain(case, rows, frame_skip):
    """the chain of public calls at one substep per frame or at the task's frame_skip; there the call's ctrl is the k-step excitation, which
    static_opt()'s one-step ctrl is not, so ctrl is left to test_excitation_over_interval"""
    import torch
    from fd_oracle import FdOracle
    env = _env(case, CHAIN_ENVS, rows)
    m, T = env.mj_model, CHAIN_FRAMES
    k = env.n_frames if frame_skip else 1
    rho = CASE_RESERVE.get(case, RESERVE)
    ref_qpos, ref_qvel, ref_qacc, start, _ = _self_reference(env, T, k)
    free = bool(np.any(np.asarray(m.jnt_type) == 0))
    fo = FdOracle(env.I, env.D)
    worst_q = 0.0
    for con, disc in ((True, False), (False, False), (False, True)):
        out = env.cmc(ref_qpos, ref_qvel, ref_qacc, KP, KV, rho, substeps=k, constraints=con, discrete=disc, initial_state=start, fields=ALL)
        torch.cuda.synchronize()
        assert torch.all(out["niter"] >= 0) and (torch.isfinite(out["qpos"]).all() or (k > 1 and case in DIVERGING))
        for t in range(T):
            s = _row_state(out, start, t)
            for key in ("qpos", "qvel", "act"):
                env.t[key].copy_(s[key])
            S = env.static_opt(out["qacc_des"][:, t].contiguous(), rho, constraints=con, discrete=disc,
                               warmstart=None if t == 0 else out["lambda"][:, t - 1].contiguous(),
                               fields=("act", "reserve_force", "ctrl", "lambda", "niter", "converged", "residual"))
            for a, b in (("act", "act_opt"), ("reserve_force", "reserve_force"), ("ctrl", "ctrl"), ("lambda", "lambda"), ("niter", "niter"),
                         ("converged", "converged"), ("residual", "residual")):
                assert (a == "ctrl" and k > 1) or _same(S[a], out[b][:, t]), (con, disc, t, b)
            r = env.rollout(out["ctrl"][:, t:t + 1].contiguous(), qfrc_applied=out["reserve_force"][:, t:t + 1].contiguous(), substeps=k,
                            initial_state=s)
            for key in STATE:
                assert _same(r[key][:, 0], out[key][:, t]), (con, disc, t, key)
        # qacc_des = ref_qacc + kv (ref_qvel - qvel) + kp (ref_qpos (-) qpos) at each frame's start state
        H = _host(out)
        S0 = _host(start)
        RQ, RV, RA = (x.cpu().numpy() for x in (ref_qpos, ref_qvel, ref_qacc))
        for e in range(CHAIN_ENVS):
            for t in range(T):
                q = S0["qpos"][e] if t == 0 else H["qpos"][e, t - 1]
                v = S0["qvel"][e] if t == 0 else H["qvel"][e, t - 1]
                if not (np.isfinite(q).all() and np.isfinite(v).all()):        # a diverged row (bit-identical above all the same)
                    continue
                terms = np.stack([RA[e, t], KV * (RV[e, t] - v), KP * fo.differentiate_pos(q, RQ[e, t])])
                err = np.abs(H["qacc_des"][e, t] - terms.sum(0)).max() / max(np.abs(terms).max(), 1e-300)
                worst_q = max(worst_q, err)
                assert err <= (QDES_REL_FREE if free else QDES_REL), (con, disc, e, t, err)
    key = "chain %s[%s]%s" % (case, rows, "" if k == 1 else " k=%d" % k)
    REPORT[key] = "bit-identical over %d frames x 3 flag sets; qacc_des worst %.1e relative" % (T, worst_q)
    print("\n" + REPORT[key])


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_chain_identity_and_qacc_des(case, rows):
    """64 envs, 8 frames, substeps 1, on a self-generated reference, with constraints, with constraints=False and with discrete=True: every
    row bit-identical to static_opt(qacc_des[:, t], warmstart=lambda[:, t - 1]) and rollout(ctrl[:, t], qfrc_applied=reserve_force[:, t]),
    both from the call's row t - 1; and qacc_des against its numpy restatement with FdOracle.differentiate_pos."""
    _chain(case, rows, False)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_chain_identity_at_frame_skip(case, rows):
    """The same at substeps = frame_skip: act_opt, reserve_force, lambda, niter, converged and residual bit-identical to static_opt(), and
    the state to rollout(ctrl[:, t], qfrc_applied=reserve_force[:, t], substeps=frame_skip), both from the call's row t - 1."""
    _chain(case, rows, True)


# ----------------------------------------------------------------------------- GPU: the excitation over a control interval
@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("case", list(CASES))
def test_excitation_over_interval(case, rows):
    """substeps = frame_skip: the returned ctrl rolled out from each frame's start state (act := act_t) brings act to act_opt at the end of
    the interval where ctrl is not clipped; where it is clipped, a* is out of reach on that side."""
    import torch
    env = _env(case, CHAIN_ENVS, rows)
    m, T, k = env.mj_model, CHAIN_FRAMES, env.n_frames
    ref_qpos, ref_qvel, ref_qacc, start, _ = _self_reference(env, T, k)
    out = env.cmc(ref_qpos, ref_qvel, ref_qacc, KP, KV, CASE_RESERVE.get(case, RESERVE), substeps=k, initial_state=start, fields=ALL)
    lo = np.array([R.ctrl_range(m, i)[0] for i in range(m.nu)]); hi = np.array([R.ctrl_range(m, i)[1] for i in range(m.nu)])
    worst, clipped, checked = 0.0, 0, 0
    for t in range(T):
        r = env.rollout(out["ctrl"][:, t:t + 1].contiguous(), qfrc_applied=out["reserve_force"][:, t:t + 1].contiguous(), substeps=k,
                        initial_state=_row_state(out, start, t))
        got, tgt, c = r["act"][:, 0].cpu().numpy(), out["act_opt"][:, t].cpu().numpy(), out["ctrl"][:, t].cpu().numpy()
        assert _same(r["act"][:, 0], out["act"][:, t])
        live = np.isfinite(tgt).all(1) & np.isfinite(c).all(1)             # the envs whose frame starts from a finite row
        got, tgt, c = got[live], tgt[live], c[live]
        free = (c > lo) & (c < hi)
        worst = max(worst, float(np.abs(got - tgt)[free].max()) if free.any() else 0.0)
        assert np.all(np.abs(got - tgt)[free] <= EXCITE_TOL), float(np.abs(got - tgt)[free].max())
        at_hi, at_lo = (c >= hi) & ~free, (c <= lo) & ~free
        assert np.all(got[at_hi] <= tgt[at_hi] + EXCITE_TOL) and np.all(got[at_lo] >= tgt[at_lo] - EXCITE_TOL)
        clipped += int((~free).sum())
        checked += int(live.sum())
    assert torch.isfinite(out["ctrl"]).all() or case in DIVERGING
    REPORT["excite %s[%s]" % (case, rows)] = "k %d: worst |act - a*| %.1e where not clipped, %d clipped, %d of %d env-frames from finite rows" % (
        k, worst, clipped, checked, CHAIN_ENVS * T)
    print("\n" + REPORT["excite %s[%s]" % (case, rows)])


# ----------------------------------------------------------------------------- GPU: tracking
def _pooled(err_sq_a, err_sq_b):
    return float(np.sqrt(err_sq_a.mean()) / max(np.sqrt(err_sq_b.mean()), 1e-300))


@pytest.mark.gpu
def test_cmc_call_tracks_hand_trajectory():
    """test_static_opt.py's hand trajectory criteria through the one call: 256 envs, 200 frames, kp 100, kv 20, rho 10, one mj_step per
    frame; pooled RMS error at least 10x below the passive hand's, and at least 8x on every joint that moves by more than 0.1 rad."""
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoVecEnv.from_model("myohand_pose", CMC_ENVS)
    m, n, dev = env.mj_model, CMC_ENVS, env.device
    pos, vel, acc = _reference(m.opt_timestep)
    starts = np.random.default_rng(SEED).integers(0, len(pos) - CMC_STEPS - 1, n)
    idx = starts[:, None] + np.arange(CMC_STEPS)[None, :]
    d = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=dev)
    start = {"qpos": d(pos[starts]), "qvel": d(vel[starts]), "act": torch.zeros(n, m.na, dtype=torch.float64, device=dev),
             "qacc_warmstart": torch.zeros(n, m.nv, dtype=torch.float64, device=dev), "time": torch.zeros(n, dtype=torch.float64, device=dev)}
    out = env.cmc(d(pos[idx]), d(vel[idx]), d(acc[idx]), KP, KV, CMC_RESERVE, initial_state=start,
                  fields=("qpos", "reserve_force", "act_opt", "niter", "converged", "qacc_des"))
    passive = env.rollout(torch.zeros(n, CMC_STEPS, m.nu, dtype=torch.float64, device=dev), initial_state=start, fields=("qpos",))
    goal = pos[idx + 1]
    e_cmc = (out["qpos"].cpu().numpy() - goal) ** 2
    e_pas = (passive["qpos"].cpu().numpy() - goal) ** 2
    rms_c, rms_p = np.sqrt(e_cmc.mean((0, 1))), np.sqrt(e_pas.mean((0, 1)))
    ratio = rms_p / np.maximum(rms_c, 1e-300)
    moving = np.array([np.ptp(pos[s:s + CMC_STEPS + 1, j]) for s in starts for j in range(m.nq)]).reshape(n, m.nq).mean(0) > 0.1
    pooled = _pooled(e_pas, e_cmc)
    REPORT["track hand trajectory"] = ("pooled ratio %.1f, worst on the %d moving joints %.1f, Newton steps %.2f, unconverged %.4f"
                                       % (pooled, int(moving.sum()), ratio[moving].min(), out["niter"].double().mean().item(),
                                          (out["converged"] != 1).double().mean().item()))
    print("\n" + REPORT["track hand trajectory"] + "; per joint %s" % np.round(ratio, 1).tolist())
    assert pooled >= TRACK_RATIO and moving.sum() >= 8 and np.all(ratio[moving] >= 8), (pooled, ratio)


# Pooled ratios below the 10x bound on an NVIDIA H100 80GB HBM3 (700 W), and the floor each case is held to (0.8x the measured ratio, so
# that a regression fails).  With the per-model reserves the muscles carry most of the force on the hands, and their activation lag
# limits the tracking; on the legs the reserves carry the unactuated pelvis through changing ground contacts.
BELOW_BOUND = {("hand_pose", "1"): 4.9, ("hand_pose", "frame_skip"): 4.7, ("reach", "1"): 2.8, ("reach", "frame_skip"): 4.7,
               ("hold", "1"): 4.0, ("walk_fatigue", "1"): 0.7, ("stand", "1"): 1.0, ("torso", "1"): 1.6}
FLOOR = 0.8
# Held over frame_skip substeps, the reserve forces and a* solved at the frame's start state diverge on the held object and the legs:
# the CPU reference of the same loop diverges as well (tests/test_cmc_reference.py, DESIGN.md section 4).
DIVERGING = ("hold", "walk_fatigue", "stand")


@pytest.mark.gpu
@pytest.mark.parametrize("case,substeps", [(c, k) for c in CASES for k in ("1", "frame_skip")])
def test_cmc_tracks_self_generated_reference(case, substeps):
    """On every base task, along a self-generated reference from a perturbed start, with the per-model reserves of test_static_opt.py: the
    pooled RMS position error at least 10x below that of the same start with zero ctrl and no reserves; FLOOR x the measured ratio for
    the cases BELOW_BOUND lists; and at frame_skip on the DIVERGING tasks, the divergence itself (a non-finite row or |qvel| > 1e3)."""
    import torch
    n, T = 256, 100
    env = _env(case, n)
    m, k = env.mj_model, (1 if substeps == "1" else env.n_frames)
    ref_qpos, ref_qvel, ref_qacc, start, goal = _self_reference(env, T, k)
    out = env.cmc(ref_qpos, ref_qvel, ref_qacc, KP, KV, CASE_RESERVE.get(case, RESERVE), substeps=k, initial_state=start,
                  fields=("qpos", "qvel", "reserve_force", "niter", "converged"))
    passive = env.rollout(torch.zeros(n, T, m.nu, dtype=torch.float64, device=env.device), substeps=k, initial_state=start, fields=("qpos",))
    g = goal.cpu().numpy()
    # errors in the tangent space (free joints: position and rotation vector)
    from fd_oracle import FdOracle
    fo = FdOracle(env.I, env.D)
    Q, P = out["qpos"].cpu().numpy(), passive["qpos"].cpu().numpy()
    e_c = np.array([[fo.differentiate_pos(g[e, t], Q[e, t]) for t in range(T)] for e in range(n)]) ** 2
    e_p = np.array([[fo.differentiate_pos(g[e, t], P[e, t]) for t in range(T)] for e in range(n)]) ** 2
    pooled = _pooled(e_p, e_c)
    V = out["qvel"].cpu().numpy()
    gone = ~(np.isfinite(Q).all(2) & (np.abs(np.nan_to_num(V, nan=np.inf)) <= 1e3).all(2))          # [n, T]
    diverged = gone.any(1)
    REPORT["track %s k=%d" % (case, k)] = ("pooled ratio %.1f (RMS CMC %.2e, passive %.2e), Newton steps %.2f, unconverged %.4f, RMS reserve force %.3g; "
                                           "%d of %d envs diverge (first at frame %d)"
                                           % (pooled, np.sqrt(e_c.mean()), np.sqrt(e_p.mean()), out["niter"].double().mean().item(),
                                              (out["converged"] != 1).double().mean().item(), out["reserve_force"].pow(2).mean().sqrt().item(),
                                              int(diverged.sum()), n, int(gone.any(0).argmax()) if diverged.any() else T))
    print("\n" + REPORT["track %s k=%d" % (case, k)])
    if substeps == "frame_skip" and case in DIVERGING:
        assert diverged.any(), "the run no longer diverges: re-measure it and move the case to BELOW_BOUND or the 10x bound"
    elif (case, substeps) in BELOW_BOUND:
        assert not diverged.any() and pooled >= FLOOR * BELOW_BOUND[(case, substeps)], (pooled, BELOW_BOUND[(case, substeps)])
    else:
        assert not diverged.any() and pooled >= TRACK_RATIO, pooled


# ----------------------------------------------------------------------------- GPU: batches, side effects, launches, checks
def _hand_inputs(n, T, rng, dev):
    import torch
    from myosuite_b200 import assets
    m = assets.load("myohand_pose")
    qpos, qvel, act, _ = _states(m, n, rng, overshoot=0.0, vel=0.5)
    d = lambda x: torch.as_tensor(np.ascontiguousarray(x), dtype=torch.float64, device=dev)
    ref_qpos = d(qpos[:, None] + rng.normal(0, 0.05, (n, T, m.nq)))
    return m, qpos, qvel, act, ref_qpos, d(rng.normal(0, 0.5, (n, T, m.nv))), d(rng.normal(0, 5, (n, T, m.nv)))


@pytest.mark.gpu
def test_batch_independence():
    """4096 hand envs against the same states and references at other slots of a 64-env batch, and against a batch at another contact
    capacity: every output bit-identical, at substeps 1 and frame_skip (at the other capacity, on the envs that dropped no contacts in
    either batch)."""
    import torch
    from myosuite_b200 import vec_env
    N, T = 4096, 4
    rng = np.random.default_rng(SEED)
    big = vec_env.MyoVecEnv.from_model("myohand_pose", N)
    m, qpos, qvel, act, RQ, RV, RA = _hand_inputs(N, T, rng, big.device)
    big.set_state(qpos=qpos, qvel=qvel, act=act)
    idx = rng.choice(N, 64, replace=False); it = torch.as_tensor(idx, device=big.device)
    for k in (1, FRAME_SKIP):
        out = big.cmc(RQ, RV, RA, KP, KV, RESERVE, substeps=k, fields=ALL + ("overflow",))
        for maxcon in (None, 24):
            small = vec_env.MyoVecEnv.from_model("myohand_pose", 64, **({} if maxcon is None else dict(maxcon=maxcon)))
            small.set_state(qpos=qpos[idx], qvel=qvel[idx], act=act[idx])
            small.t["qacc_warmstart"].copy_(big.t["qacc_warmstart"][it]); small.t["time"].copy_(big.t["time"][it])
            got = small.cmc(RQ[it].contiguous(), RV[it].contiguous(), RA[it].contiguous(), KP, KV, RESERVE, substeps=k, fields=ALL + ("overflow",))
            torch.cuda.synchronize()
            # envs that dropped contacts at either capacity ran different physics; every other env matches bit for bit
            ok = (got["overflow"] == 0) & (out["overflow"][it] == 0)
            assert int(ok.sum()) >= 48, (k, maxcon, int(ok.sum()))
            for f in ALL:
                assert _same(got[f][ok], out[f][it][ok]), (k, maxcon, f)
            if maxcon is None:
                assert torch.equal(got["overflow"], out["overflow"][it])
            print("\nsubsteps %d, maxcon %s: %d of 64 envs without dropped contacts" % (k, maxcon, int(ok.sum())))
        assert torch.isfinite(out["qpos"]).all()


@pytest.mark.gpu
def test_no_side_effects_and_unrequested_outputs():
    """Twin batches with and without cmc calls between their 50 steps stay bit-identical, every bound tensor is untouched by a call, and
    outputs that are not requested are not written."""
    import torch
    from myosuite_b200 import abi, vec_env
    from test_mj_data import BOUND
    eid, n, T = "myoHandObjHoldRandom-v0", 517, 3
    a_env, b_env = (vec_env.MyoVecEnv(eid, n, seed=SEED) for _ in range(2))
    m = a_env.mj_model
    for env in (a_env, b_env):
        env.reset(seed=SEED)
    g = torch.Generator(device="cpu").manual_seed(SEED)
    dev = a_env.device
    for step in range(50):
        action = (torch.rand(n, m.nu, generator=g) * 2 - 1).to(dev)
        RQ = a_env.t["qpos"][:, None].repeat(1, T, 1).contiguous()
        RV = torch.zeros(n, T, m.nv, dtype=torch.float64, device=dev)
        before = {k: a_env.t[k].clone() for k in BOUND if k in a_env.t}
        a_env.cmc(RQ, RV, RV, KP, KV, RESERVE, fields=ALL)
        if step % 10 == 0:
            a_env.cmc(RQ, RV, RV, KP, KV, RESERVE, substeps=3, constraints=False, discrete=True)
        torch.cuda.synchronize()
        for k, v in before.items():
            assert _same(v, a_env.t[k]), (step, k)
        a_env.step(action); b_env.step(action.clone())
        torch.cuda.synchronize()
        for k in BOUND:
            if k in a_env.t:
                assert _same(a_env.t[k], b_env.t[k]), (step, k)
    RQ = a_env.t["qpos"][:, None].repeat(1, T, 1).contiguous()
    RV = torch.zeros(n, T, m.nv, dtype=torch.float64, device=dev)
    full = {k: v.clone() for k, v in a_env.cmc(RQ, RV, RV, KP, KV, RESERVE, fields=ALL).items()}
    vec = lambda x, w: torch.full((w,), x, dtype=torch.float64, device=dev)
    params = abi.MyoCmcParams(max_iter=50, substeps=1, tol=1e-12)
    for ask in (("qpos",), ("ctrl", "lambda", "time"), ("act_opt", "niter", "residual", "qacc_des")):
        sent = {k: torch.full_like(v, -7 if v.dtype == torch.int32 else float("nan")) for k, v in full.items()}
        n0 = a_env.batch.launches
        a_env.batch.cmc(params, T, stream=a_env._stream(), ref_qpos=RQ, ref_qvel=RV, ref_qacc=RV, kp=vec(KP, m.nv), kv=vec(KV, m.nv),
                        reserve=vec(RESERVE, m.nv), **{k: sent[k] for k in ask})
        torch.cuda.synchronize()
        assert a_env.batch.launches > n0
        for k, v in sent.items():
            untouched = (v == -7).all() if v.dtype == torch.int32 else v.isnan().all()
            assert torch.equal(v, full[k]) if k in ask else untouched, (ask, k)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["elbow", "hand_pose"])
def test_launch_count(case):
    """Launches per call = T (3 + (substeps > 1) + R) + 1, R the regroup launch of a rollout interval (include/myo_b200.h)."""
    import torch
    env = _env(case, CASES[case][1])
    m, n, dev = env.mj_model, env.num_envs, env.device
    n0 = env.batch.launches
    env.rollout(torch.zeros(n, 1, m.nu, dtype=torch.float64, device=dev))
    R_ = env.batch.launches - n0 - 1
    assert R_ in (0, 1)
    for T in (1, 5):
        RQ = env.t["qpos"][:, None].repeat(1, T, 1).contiguous()
        RV = torch.zeros(n, T, m.nv, dtype=torch.float64, device=dev)
        for k in (1, env.n_frames):
            n0 = env.batch.launches
            env.cmc(RQ, RV, RV, KP, KV, CASE_RESERVE.get(case, RESERVE), substeps=k)
            assert env.batch.launches - n0 == T * (3 + (k > 1) + R_) + 1, (T, k, env.batch.launches - n0, R_)
    print("\n%s: R = %d" % (case, R_))


@pytest.mark.gpu
def test_input_checks_without_launch():
    import torch
    from myosuite_b200 import abi, vec_env
    env = vec_env.MyoVecEnv("myoElbowPose1D6MRandom-v0", 8, seed=SEED)
    m, dev, T = env.mj_model, env.device, 3
    nq, nv, nu = m.nq, m.nv, m.nu
    RQ = torch.zeros(8, T, nq, dtype=torch.float64, device=dev)
    RV = torch.zeros(8, T, nv, dtype=torch.float64, device=dev)
    n0 = env.batch.launches
    bad_refs = (dict(ref_qpos=torch.zeros(8, T, nq + 1, dtype=torch.float64, device=dev)), dict(ref_qpos=RQ.float()), dict(ref_qpos=RQ.cpu()),
                dict(ref_qvel=torch.zeros(8, T + 1, nv, dtype=torch.float64, device=dev)),
                dict(ref_qacc=torch.zeros(8, T, 2 * nv, dtype=torch.float64, device=dev)[:, :, ::2]),
                dict(ref_qpos=torch.zeros(8, 0, nq, dtype=torch.float64, device=dev)), dict(ref_qpos=RQ[0]))
    for kw in bad_refs:
        args = dict(ref_qpos=RQ, ref_qvel=RV, ref_qacc=RV); args.update(kw)
        with pytest.raises(ValueError):
            env.cmc(args["ref_qpos"], args["ref_qvel"], args["ref_qacc"], KP, KV, 1.0)
    for kw in (dict(kp=-1.0), dict(kv=-1e-3), dict(kp=float("nan")), dict(kv=float("inf")), dict(kp=np.ones(nv + 1)),
               dict(kv=torch.full((nv,), -1.0, dtype=torch.float64, device=dev)), dict(reserve=0.0), dict(reserve=-1.0),
               dict(reserve=float("nan")), dict(weight=np.zeros(nu)), dict(weight=-np.ones(nu)), dict(substeps=0), dict(max_iter=-1),
               dict(tol=-1.0), dict(tol=float("inf")), dict(warmstart=torch.zeros(8, nv + 1, dtype=torch.float64, device=dev)),
               dict(initial_state={"qpos": torch.zeros(8, nq + 1, dtype=torch.float64, device=dev)})):
        args = dict(kp=KP, kv=KV, reserve=1.0); args.update(kw)
        with pytest.raises(ValueError):
            env.cmc(RQ, RV, RV, **args)
    with pytest.raises(KeyError):
        env.cmc(RQ, RV, RV, KP, KV, 1.0, fields=("ref_qpos",))
    vec = lambda x, w: torch.full((w,), x, dtype=torch.float64, device=dev)
    good = dict(ref_qpos=RQ, ref_qvel=RV, ref_qacc=RV, kp=vec(KP, nv), kv=vec(KV, nv), reserve=vec(1.0, nv))
    P = abi.MyoCmcParams(max_iter=50, substeps=1, tol=1e-12)
    cases = [(P, T, 4, good, "unknown flag"), (P, 0, 0, good, "nstep"), (abi.MyoCmcParams(max_iter=50, substeps=0, tol=0.0), T, 0, good, "substeps"),
             (abi.MyoCmcParams(max_iter=-1, substeps=1, tol=0.0), T, 0, good, "max_iter"),
             (abi.MyoCmcParams(max_iter=5, substeps=1, tol=-1.0), T, 0, good, "tol"),
             (abi.MyoCmcParams(max_iter=5, substeps=1, tol=float("nan")), T, 0, good, "finite")]
    for k in ("ref_qpos", "ref_qvel", "ref_qacc", "kp", "kv", "reserve"):
        cases.append((P, T, 0, {x: v for x, v in good.items() if x != k}, "required"))
    for params, nstep, flags, bufs, msg in cases:
        with pytest.raises(abi.MyoError, match=msg):
            env.batch.cmc(params, nstep, flags=flags, **bufs)
    unbound = abi.Batch(env.dev_model, env.device_index, 8, env.cfg)
    with pytest.raises(abi.MyoError, match="bound"):
        unbound.cmc(P, T, **good)
    assert env.batch.launches == n0 and unbound.launches == 0
    sv = env.state_version
    env.cmc(RQ, RV, RV, KP, KV, 1.0)
    assert env.batch.launches > n0 and env.state_version == sv


@pytest.mark.gpu
def test_myoenv_cmc():
    """MyoEnv.cmc equals env 0 of a batch run from the same state."""
    import torch
    from myosuite_b200 import vec_env
    env = vec_env.MyoEnv("myoHandPoseRandom-v0", seed=3)
    m, T = env.mj_model, 6
    env.step(env.action_space.sample())
    rng = np.random.default_rng(0)
    q0 = env.vec.t["qpos"][0].cpu().numpy()
    RQ, RV, RA = q0[None] + rng.normal(0, 0.05, (T, m.nq)), rng.normal(0, 0.5, (T, m.nv)), rng.normal(0, 5, (T, m.nv))
    for k in (1, 3):
        r = env.cmc(RQ, RV, RA, KP, KV, RESERVE, substeps=k, fields=ALL + ("overflow",))
        assert r["qpos"].shape == (T, m.nq) and r["niter"].shape == (T,) and isinstance(r["overflow"], int)
        d = lambda x: torch.as_tensor(x[None], device=env.vec.device).contiguous()
        v = env.vec.cmc(d(RQ), d(RV), d(RA), KP, KV, RESERVE, substeps=k, fields=ALL)
        for f, x in v.items():
            assert np.array_equal(np.asarray(r[f]), x[0].cpu().numpy()), (k, f)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\ncomputed muscle control:")
        for k in sorted(REPORT):
            print("  %-36s %s" % (k, REPORT[k]))
