"""Computed muscle control on the device (myo_batch_cmc) against the CPU reference of one frame (tests/cmc_ref.py), frame by frame.

CPU: the vectorised k-step bisection of cmc_ref against test_cmc.excitation_k, and one reference frame per shipped model (the bounded
least-squares solution against its optimality conditions, act at the end of the oracle interval against a*).
GPU: on every base task, at substeps 1 and frame_skip, on both row storages, 64 envs follow a self-generated reference for 100 frames
(test_cmc._self_reference, the per-model reserves).  The checked envs (the most contact-heavy of the batch's start states and a seeded
random rest) are teacher-forced: frame t of the CPU reference runs from the call's own row t - 1, so a chaotic trajectory never has to be
followed.  Every frame of the first 20 and every 5th after that is checked, up to the env's first non-finite row: qacc_des against the
CPU's; the static optimisation by the KKT certificate of test_static_opt.py (constraints on) and against the lsq reference (constraints
off); act after the CPU interval, run with the call's ctrl and reserve force, against a* where ctrl is not clipped; and the state after
the interval against the CPU's with the mid-episode bounds, up to the frame at which the env's |qvel| passes 1e3.  On the three tasks whose frame_skip runs diverge (hold, walk_fatigue, stand) the CPU reference run
free from the same start is held to diverge too, within a stated number of frames of the device."""
import time

import numpy as np
import pytest

import cmc_ref as C
from parity_helpers import ACT_ATOL, QACC_REL, QPOS_ATOL, QVEL_REL, relerr
from test_cmc import DIVERGING, FRAME_SKIP, QDES_REL, QDES_REL_FREE, _env, _row_state, _self_reference, excitation_k
from test_mj_data import CASES, QACC_MAX, QACC_SHARE, ROWS, SEED
from test_static_opt import ACT_REF, CASE_RESERVE, EXCITE_TOL, KP, KV, RESERVE, SHIPPED, kkt

N_ENV, T_FRAMES = 64, 100          # the tracking test's horizon
N_CHECK, N_CONTACT = 6, 3          # envs checked per case, of which the most contact-heavy at the start
N_FREE, FREE_FRAMES = 4, (0, 1, 2, 5, 10, 20, 40, 60, 80, 99)     # constraints off: envs and frames whose solve is checked (bvls on the
                                   # torso's 210 muscles takes about 0.4 s)
DIVERGED = 1e3                     # |qvel| beyond which a run counts as diverged (with a non-finite output)
F64_CASES = DIVERGING + ("hand_pose",)
REPORT = {}


def _checked_frames(stop):
    return [t for t in range(min(T_FRAMES, stop)) if t < 20 or t % 5 == 0]


# ----------------------------------------------------------------------------- CPU
def test_vectorised_excitation_matches_excitation_k(models, tmp_path):
    """cmc_ref.excitation (all muscles at once) against test_cmc.excitation_k (one muscle at a time), bit for bit, at k = 2, 5 and
    frame_skip on every shipped model and the zoo's MUSCLE model (tausmooth > 0), with targets inside and out of reach."""
    from parity_helpers import _states
    from test_static_opt import _zoo
    rng = np.random.default_rng(SEED)
    z = _zoo(tmp_path)["MUSCLE"]
    cases = [(name, models[name], _states(models[name], 2, rng, overshoot=0.0, vel=0.3)[2]) for name in SHIPPED]
    cases.append(("zoo/MUSCLE", z["m"], z["act"][:2]))
    n = 0
    for name, m, act in cases:
        for k in (2, 5, FRAME_SKIP):
            for e in range(len(act)):
                a0 = np.clip(act[e], 0, 1)
                target = np.clip(a0 + rng.normal(0, 0.1, m.nu), 0, 1)
                target[::4] = rng.uniform(0, 1, len(target[::4]))
                got = C.excitation(m, a0, target, k)
                ref = np.array([excitation_k(m, i, a0[i], target[i], k) for i in range(m.nu)])
                assert np.array_equal(got, ref), (name, k, e, float(np.abs(got - ref).max()))
                n += m.nu
    print("\nvectorised k-step excitation: %d muscles bit-identical to excitation_k" % n)


KKT_LSQ = 1e-12            # the lsq solution's |a - clip(G' lambda / w, 0, 1)|, relative: 6.7e-14 measured (hand); bvls stops at its
                           # own optimality tolerance


def test_reference_frame_per_model(models):
    """One CPU frame per shipped model at random states, reference one frame ahead of a passive step: the lsq solution meets its
    optimality conditions (a = clip(G' lambda / w, 0, 1), G a + r = t); act at the end of the oracle interval of k steps equals a* where
    ctrl is not clipped, and a* is out of reach where it is; the interval adds k timesteps; qacc_des is ref_qacc when the state is the
    reference's."""
    from myosuite_b200 import blob
    from fd_oracle import FdOracle
    from inverse_oracle import InvOracle
    from parity_helpers import _states
    rng = np.random.default_rng(SEED)
    worst = {}
    for name in SHIPPED:
        m = models[name]
        I, D = blob.pack(m)
        io, fo = InvOracle(I, D), FdOracle(I, D)
        qpos, qvel, act, _ = _states(m, 2, rng, overshoot=0.0, vel=0.3)
        lo, hi = C.ctrl_bounds(m)
        for k in (1, FRAME_SKIP):
            for con in (True, False):
                ref = C.CmcRef(m, io, fo, KP, KV, 100.0 if name in ("myolegs", "myotorso") else RESERVE, fl=C.flags(con), k=k)
                for e in range(len(qpos)):
                    s = dict(qpos=qpos[e], qvel=qvel[e], act=act[e], qacc_warmstart=np.zeros(m.nv), time=np.array([0.25]))
                    ra = rng.normal(0, 1, m.nv)
                    assert np.array_equal(ref.qacc_des(s, qpos[e], qvel[e], ra), ra)
                    # a reference row one passive step ahead
                    nxt, _, _ = ref.interval(s, np.zeros(m.nu), np.zeros(m.nv))
                    F = ref.frame(s, nxt["qpos"], nxt["qvel"], ra)
                    S = ref.solve(s, F["qacc_des"])
                    ke, fe = C.kkt_error(S, ref.w)
                    assert ke <= KKT_LSQ and fe <= 1e-12, (name, k, con, ke, fe)
                    got, c, a = F["next"]["act"], F["ctrl"], F["act_opt"]
                    free = (c > lo) & (c < hi)
                    assert np.all(np.abs(got - a)[free] <= EXCITE_TOL), (name, k, float(np.abs(got - a)[free].max()))
                    assert np.all(got[c >= hi] <= a[c >= hi] + EXCITE_TOL) and np.all(got[c <= lo] >= a[c <= lo] - EXCITE_TOL)
                    tnow = 0.25
                    for _ in range(k):
                        tnow += m.opt_timestep
                    assert F["next"]["time"][0] == tnow and np.all(np.isfinite(F["next"]["qpos"]))
                    worst[name] = max(worst.get(name, 0.0), ke)
    print("\nCPU reference frame: lsq optimality %s" % {k: "%.1e" % v for k, v in worst.items()})


# ----------------------------------------------------------------------------- GPU helpers
def _host(D):
    return {k: v.cpu().numpy().copy() for k, v in D.items()}


OUT = ("qacc_des", "ctrl", "act_opt", "reserve_force", "lambda", "converged", "residual", "qpos", "qvel", "act", "qacc", "time")
WATCH = ("qacc_des", "reserve_force", "ctrl", "act_opt", "qpos", "qvel", "act", "qacc")


def _first_bad(H):
    """per env: the first frame at which any output is non-finite or |qvel| exceeds DIVERGED (T if none), and per output the first
    frame at which that output alone goes bad"""
    n, T = H["qpos"].shape[:2]
    per = {}
    for k in WATCH:
        x = H[k].reshape(n, T, -1)
        bad = ~np.isfinite(x).all(2)
        if k == "qvel":
            bad |= ~(np.abs(np.nan_to_num(x, nan=np.inf)) <= DIVERGED).all(2)
        per[k] = np.where(bad.any(1), bad.argmax(1), T)
    return np.minimum.reduce(list(per.values())), per


def _first_nonfinite(H):
    n, T = H["qpos"].shape[:2]
    bad = np.zeros((n, T), bool)
    for k in WATCH:
        bad |= ~np.isfinite(H[k].reshape(n, T, -1)).all(2)
    return np.where(bad.any(1), bad.argmax(1), T)


def _row(H, S0, e, t):
    """env e's state at the start of frame t: the call's row t - 1 (the start for t = 0)"""
    if t == 0:
        return {k: np.atleast_1d(S0[k][e]).copy() for k in C.STATE}
    return dict(qpos=H["qpos"][e, t - 1], qvel=H["qvel"][e, t - 1], act=H["act"][e, t - 1], qacc_warmstart=H["qacc"][e, t - 1],
                time=np.atleast_1d(H["time"][e, t - 1]))


def _pick(env, S0, pairs, prm):
    """the checked envs: the N_CONTACT most contact-heavy start states of the batch (one oracle forward each, as replay_product_step picks
    them) and a seeded random rest"""
    n = env.num_envs
    ncon = []
    for e in range(n):
        _, fo = pairs.get(e, None if prm is None else prm[e])
        fo.reset(); fo.set(qpos=S0["qpos"][e], qvel=S0["qvel"][e], act=S0["act"][e]); fo.forward(); ncon.append(fo.ncon)
    top = np.argsort(ncon, kind="stable")[::-1][:N_CONTACT]
    rest = np.random.default_rng(SEED).choice(np.setdiff1d(np.arange(n), top), N_CHECK - N_CONTACT, replace=False)
    return [int(e) for e in top] + [int(e) for e in rest]


def _run(case, rows, frame_skip, con=True, mean_acc=False):
    """the batch, its substeps, reserve, reference rows (host), start state and the call's outputs"""
    import torch
    env = _env(case, N_ENV, rows)
    k = env.n_frames if frame_skip else 1
    if mean_acc:            # the interval's mean acceleration (ref_qvel[t + 1] - ref_qvel[t]) / (k h) in place of its last substep's qacc
        RQ, RV, _, start, _ = _self_reference(env, T_FRAMES + 1, k)
        RA = ((RV[:, 1:] - RV[:, :-1]) / (k * env.mj_model.opt_timestep)).contiguous()
        RQ, RV = RQ[:, :T_FRAMES].contiguous(), RV[:, :T_FRAMES].contiguous()
    else:
        RQ, RV, RA, start, _ = _self_reference(env, T_FRAMES, k)
    rho = CASE_RESERVE.get(case, RESERVE)
    out = env.cmc(RQ, RV, RA, KP, KV, rho, substeps=k, constraints=con, initial_state=start, fields=OUT + ("overflow",))
    torch.cuda.synchronize()
    ref = {"qpos": RQ, "qvel": RV, "qacc": RA}
    return env, k, rho, {k_: v.cpu().numpy() for k_, v in ref.items()}, start, out


def _kkt_frames(env, out, start, H, bad, rho, worst, cnt):
    """the static optimisation's KKT certificate at every frame, on every env whose row is not yet diverged and whose solve converged"""
    m = env.mj_model
    rho_v, w = np.full(m.nv, rho), np.ones(m.nu)
    for t in range(T_FRAMES):
        live = bad > t
        if not live.any():
            break
        conv = live & (H["converged"][:, t] == 1)
        cnt["unconverged"] += int((live & ~conv).sum())
        if not conv.any():
            continue
        s = _row_state(out, start, t)
        for key in ("qpos", "qvel", "act"):
            env.t[key].copy_(s[key])
        qd = out["qacc_des"][:, t].contiguous()
        G = _host(env.static_opt(qd, rho, fields=("muscle_gain", "muscle_bias", "qfrc_inverse")))
        S = dict(G, act=H["act_opt"][:, t], reserve_force=H["reserve_force"][:, t], converged=H["converged"][:, t],
                 residual=H["residual"][:, t], **{"lambda": H["lambda"][:, t]})
        ke, _ = kkt(env, S, qd, rho_v, w, con=True, rows=np.nonzero(conv)[0])
        worst["kkt"] = max(worst["kkt"], ke)
        cnt["kkt_envframes"] += int(conv.sum())


def _diverges(F):
    return not all(np.isfinite(F[k]).all() for k in ("qacc_des", "reserve_force", "ctrl", "act_opt")) or \
        not all(np.isfinite(F["next"][k]).all() for k in C.STATE) or np.abs(F["next"]["qvel"]).max() > DIVERGED


# ----------------------------------------------------------------------------- GPU: frame-by-frame parity
@pytest.mark.gpu
@pytest.mark.parametrize("substeps", ["1", "frame_skip"])
@pytest.mark.parametrize("rows,case", [(r, c) for r in ROWS for c in CASES if r == "p48" or c in F64_CASES])
def test_cmc_frames_vs_cpu_reference(case, rows, substeps):
    """Teacher-forced frames of the call against the CPU reference, with constraints (and the KKT certificate on every env and frame
    before the env diverges) and without (act against the lsq reference).  Frames in which the CPU interval has more contacts than the
    batch's capacity (the device dropped some) or leaves the contact regime are outside the parity claim: they are skipped and counted."""
    t0 = time.time()
    worst = dict(qacc_des=0.0, kkt=0.0, act_vs_lsq=0.0, excite=0.0, act=0.0, qpos=0.0, qvel=0.0, qacc=0.0, qpos_diverged=0.0)
    cnt = dict(frames=0, diverging=0, qacc_over_mid=0, kkt_envframes=0, unconverged=0, overflow=0, regime=0, clipped=0, lsq=0)
    stops = {}
    for con in (True, False):
        env, k, rho, REF, start, out = _run(case, rows, substeps == "frame_skip", con=con)
        m = env.mj_model
        H, S0 = _host(out), _host(start)
        pairs = C.OraclePair(env)
        prm = env.get_env_state().get("env_prm")
        free_jnt = bool(np.any(np.asarray(m.jnt_type) == 0))
        lo, hi = C.ctrl_bounds(m)
        bad, _ = _first_bad(H)
        stop = _first_nonfinite(H)
        stops[con] = (int((bad < T_FRAMES).sum()), int(bad.min()))
        if con:
            _kkt_frames(env, out, start, H, bad, rho, worst, cnt)
        envs = _pick(env, S0, pairs, prm)
        for e in envs:
            io, fo = pairs.get(e, None if prm is None else prm[e])
            ref = C.CmcRef(m, io, fo, KP, KV, rho, fl=C.flags(con), k=k)
            for t in (_checked_frames(int(stop[e])) if con else [t for t in FREE_FRAMES if t < stop[e]]):
                msg = "%s[%s] k %d con %s env %d frame %d (diverges at %d)" % (case, rows, k, con, e, t, bad[e])
                s = _row(H, S0, e, t)
                qd = ref.qacc_des(s, REF["qpos"][e, t], REF["qvel"][e, t], REF["qacc"][e, t])
                dv = KV * (REF["qvel"][e, t] - s["qvel"])
                terms = max(np.abs(REF["qacc"][e, t]).max(), np.abs(dv).max(), np.abs(qd - REF["qacc"][e, t] - dv).max(), 1e-300)
                err = float(np.abs(H["qacc_des"][e, t] - qd).max() / terms)
                worst["qacc_des"] = max(worst["qacc_des"], err)
                assert err <= (QDES_REL_FREE if free_jnt else QDES_REL), (msg, err)
                if not con:
                    if e in envs[N_CHECK - N_FREE:] and t < bad[e]:
                        da = float(np.abs(H["act_opt"][e, t] - ref.solve(s, H["qacc_des"][e, t])["act_opt"]).max())
                        worst["act_vs_lsq"] = max(worst["act_vs_lsq"], da)
                        assert da <= ACT_REF, (msg, da)
                        cnt["lsq"] += 1
                    continue
                c, a = H["ctrl"][e, t], H["act_opt"][e, t]
                nxt, ok, ncon = ref.interval(s, c, H["reserve_force"][e, t])
                if ncon > env.dims.maxcon:    # the device dropped contacts in this interval
                    cnt["overflow"] += 1
                    continue
                if not ok:                    # deep ellipsoid penetration on some substep
                    cnt["regime"] += 1
                    continue
                cnt["frames"] += 1
                got = nxt["act"]
                inside = (c > lo) & (c < hi)
                if inside.any():
                    worst["excite"] = max(worst["excite"], float(np.abs(got - a)[inside].max()))
                assert np.all(np.abs(got - a)[inside] <= EXCITE_TOL), (msg, float(np.abs(got - a)[inside].max()))
                assert np.all(got[c >= hi] <= a[c >= hi] + EXCITE_TOL) and np.all(got[c <= lo] >= a[c <= lo] - EXCITE_TOL), msg
                cnt["clipped"] += int((~inside).sum())
                worst["act"] = max(worst["act"], float(np.abs(H["act"][e, t] - got).max()))
                np.testing.assert_allclose(H["act"][e, t], got, rtol=0, atol=ACT_ATOL, err_msg=msg)
                assert H["time"][e, t] == nxt["time"][0], msg
                dq, dv, da = (float(np.abs(H["qpos"][e, t] - nxt["qpos"]).max()), relerr(H["qvel"][e, t], nxt["qvel"]),
                              relerr(H["qacc"][e, t], nxt["qacc_warmstart"]))
                if t >= bad[e]:
                    # the frame starts from a row past |qvel| = 1e3 (a flung object, a leg through the floor): the interval amplifies
                    # round-off beyond the mid-episode bounds (qpos 7.4e-6 on p48 and 2.9e-3 on f64 rows in the hold's frames after its
                    # object passed 1e3, on an H100), so only its deviation is reported
                    cnt["diverging"] += 1; worst["qpos_diverged"] = max(worst["qpos_diverged"], dq)
                    continue
                worst["qpos"], worst["qvel"], worst["qacc"] = max(worst["qpos"], dq), max(worst["qvel"], dv), max(worst["qacc"], da)
                cnt["qacc_over_mid"] += int(da >= QACC_REL)
                assert dq <= QPOS_ATOL and dv < QVEL_REL and da < QACC_MAX, (msg, dq, dv, da)
    dt = time.time() - t0
    line = ("k %2d: %d frames checked (%d after |qvel| > 1e3; qacc above %.0e on %d), KKT on %d env-frames (%d unconverged not "
            "certified), act vs lsq on %d; skipped frames: contact overflow %d, deep penetration %d; diverged envs (first frame): constraints %d (%s), without %d (%s); "
            "worst %s; %d clipped ctrl [%.0f s]"
            % (k, cnt["frames"], cnt["diverging"], QACC_REL, cnt["qacc_over_mid"], cnt["kkt_envframes"], cnt["unconverged"], cnt["lsq"],
               cnt["overflow"], cnt["regime"],
               stops[True][0], stops[True][1], stops[False][0], stops[False][1],
               ", ".join("%s %.1e" % kv for kv in worst.items()), cnt["clipped"], dt))
    REPORT["%s[%s] %s" % (case, rows, substeps)] = line
    print("\n%s[%s] %s" % (case, rows, line))
    assert cnt["frames"] >= 2 * N_CHECK and cnt["lsq"] > 0
    assert cnt["overflow"] + cnt["regime"] <= cnt["frames"] // 2
    assert cnt["unconverged"] <= 0.01 * cnt["kkt_envframes"]
    # qacc: the readout's rule (test_mj_data.py), QACC_REL on QACC_SHARE of the frames and QACC_MAX on all; one frame in a sample of under
    # a hundred is below the share's resolution (1.05e-6 measured on one of the stand's 72 frame_skip frames on an H100)
    assert cnt["qacc_over_mid"] <= max(1, (1 - QACC_SHARE) * (cnt["frames"] - cnt["diverging"]))


# ----------------------------------------------------------------------------- GPU: the divergence
DIVERGE_LAG = 5            # the CPU reference run free diverges within this many frames of the device: 3 measured on an H100 (one
                           # walk env of 24 env runs; every other at the same frame)


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", ["last_substep", "mean"])
@pytest.mark.parametrize("case", DIVERGING)
def test_divergence_is_the_methods(case, fixture):
    """At frame_skip the call diverges on the hold and leg tasks.  The CPU reference run free from the same start along the same reference
    (no device output enters it) diverges too, on the same envs, within DIVERGE_LAG frames of the device; with the fixture's last-substep
    ref_qacc and with the interval's mean acceleration."""
    t0 = time.time()
    env, k, rho, REF, start, out = _run(case, "p48", True, mean_acc=fixture == "mean")
    m = env.mj_model
    H, S0 = _host(out), _host(start)
    bad, per = _first_bad(H)
    pairs = C.OraclePair(env)
    prm = env.get_env_state().get("env_prm")
    envs = _pick(env, S0, pairs, prm)[:N_FREE]
    res = []
    for e in envs:
        io, fo = pairs.get(e, None if prm is None else prm[e])
        ref = C.CmcRef(m, io, fo, KP, KV, rho, k=k)
        s, t_cpu = _row(H, S0, e, 0), T_FRAMES
        for t in range(T_FRAMES):
            try:
                F = ref.frame(s, REF["qpos"][e, t], REF["qvel"][e, t], REF["qacc"][e, t])
            except ValueError:            # lsq_linear refuses non-finite data
                t_cpu = t
                break
            if _diverges(F):
                t_cpu = t
                break
            s = F["next"]
        res.append((e, int(bad[e]), t_cpu))
    first = {q: int(v.min()) for q, v in per.items()}
    line = ("k %d: device diverges on %d of %d envs (first frame %d, first per output %s); checked envs (env, device t*, CPU t*): %s [%.0f s]"
            % (k, int((bad < T_FRAMES).sum()), N_ENV, int(bad.min()), first, res, time.time() - t0))
    REPORT["diverge %s %s" % (case, fixture)] = line
    print("\ndiverge %s %s %s" % (case, fixture, line))
    assert (bad < T_FRAMES).any()
    for e, td, tc in res:
        assert (td < T_FRAMES) == (tc < T_FRAMES) and abs(td - tc) <= DIVERGE_LAG, (e, td, tc)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\ncomputed muscle control against the CPU reference:")
        for k in sorted(REPORT):
            print("  %-28s %s" % (k, REPORT[k]))
