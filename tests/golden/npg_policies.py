"""Loader for the NPG baseline policies the reference ships (agents/baslines_NPG/<env>/*/*/iterations/best_policy.pickle).

The pickles are mjrl `MLP` objects (mjrl is not installed here); two stub classes with the pickled attribute layout are enough to
unpickle them with torch alone.  Forward pass restated from mjrl (policies/gaussian_mlp.py, utils/fc_network.py):
    x = (obs - in_shift) / (in_scale + 1e-8) ; tanh after every layer but the last ; mean = out * out_scale + out_shift
    action = mean + exp(log_std) * N(0, 1)          (evaluation mode: action = mean)
`python tests/golden/npg_policies.py` extracts the weights and the logged scores of the envs this repo implements into
tests/golden/npg_policies.npz (small: 32x32 MLPs), so that the tests replay them without a MyoSuite checkout.
"""
import csv
import glob
import io
import os
import pickle
import sys
import types

import numpy as np

REF = os.path.join(os.environ.get("MYOSUITE_CHECKOUT", "."), "myosuite/agents/baslines_NPG")
ENVS = ["myoElbowPose1D6MFixed-v0", "myoElbowPose1D6MRandom-v0", "myoHandPoseFixed-v0", "myoHandPoseRandom-v0", "myoHandReachFixed-v0",
        "myoHandReachRandom-v0", "myoHandObjHoldFixed-v0", "myoHandObjHoldRandom-v0", "myoHandKeyTurnFixed-v0", "myoHandKeyTurnRandom-v0",
        "myoHandPenTwirlFixed-v0", "myoHandPenTwirlRandom-v0"]


def _stub_modules():
    import torch.nn as nn

    class MLP:            # mjrl.policies.gaussian_mlp.MLP: plain attribute bag after unpickling
        pass

    class FCNetwork(nn.Module):     # mjrl.utils.fc_network.FCNetwork
        pass
    for name, cls in (("mjrl.policies.gaussian_mlp", MLP), ("mjrl.utils.fc_network", FCNetwork)):
        parts = name.split(".")
        for i in range(1, len(parts) + 1):
            sys.modules.setdefault(".".join(parts[:i]), types.ModuleType(".".join(parts[:i])))
        setattr(sys.modules[name], cls.__name__, cls)


def load_pickle(path):
    """-> dict(W=[...], b=[...], in_shift, in_scale, out_shift, out_scale, log_std) as float64 numpy arrays."""
    _stub_modules()
    with open(path, "rb") as f:
        pol = pickle.load(f)
    net = pol.model
    layers = list(net.fc_layers)
    g = lambda t: np.asarray(t.detach().cpu().numpy(), dtype=np.float64)
    return dict(W=[g(l.weight) for l in layers], b=[g(l.bias) for l in layers], in_shift=g(net.in_shift).ravel(), in_scale=g(net.in_scale).ravel(),
                out_shift=g(net.out_shift).ravel(), out_scale=g(net.out_scale).ravel(), log_std=g(pol.log_std).ravel(), n=int(pol.n), m=int(pol.m))


def mean_action(p, obs):
    """obs [..., n] -> mean action [..., m] (float64)."""
    x = (np.asarray(obs, dtype=np.float64) - p["in_shift"]) / (p["in_scale"] + 1e-8)
    for i, (W, b) in enumerate(zip(p["W"], p["b"])):
        x = x @ W.T + b
        if i < len(p["W"]) - 1:
            x = np.tanh(x)
    return x * p["out_scale"] + p["out_shift"]


def runs(env_id):
    return sorted(glob.glob(os.path.join(REF, env_id, "*", "*")))


def logged(run_dir):
    """Last-iteration statistics of the run's log.csv + the evaluation score of results.txt."""
    rows = list(csv.DictReader(open(os.path.join(run_dir, "logs", "log.csv"))))
    last = rows[-1]
    keys = ("stoc_pol_mean", "stoc_pol_std", "stoc_pol_max", "stoc_pol_min", "success_percentage", "eval_score", "eval_success", "rwd_sparse", "rwd_dense")
    out = {k: float(last[k]) for k in keys if k in last and last[k] != ""}
    out["iteration"] = int(float(last["iteration"]))
    best = max(rows, key=lambda r: float(r["stoc_pol_mean"]))
    out["best_stoc_pol_mean"], out["best_iteration"] = float(best["stoc_pol_mean"]), int(float(best["iteration"]))
    return out


def pack(path):
    blob = {}
    for env_id in ENVS:
        for k, rd in enumerate(runs(env_id)):
            pk = os.path.join(rd, "iterations", "best_policy.pickle")
            if not os.path.exists(pk):
                continue
            p = load_pickle(pk); lg = logged(rd)
            key = "%s/%d" % (env_id, k)
            for i, (W, b) in enumerate(zip(p["W"], p["b"])):
                blob[key + "/W%d" % i] = W.astype(np.float32); blob[key + "/b%d" % i] = b.astype(np.float32)
            for f in ("in_shift", "in_scale", "out_shift", "out_scale", "log_std"):
                blob[key + "/" + f] = p[f].astype(np.float32)
            blob[key + "/logged"] = np.array([lg.get(q, np.nan) for q in LOG_KEYS])
    np.savez_compressed(path, **blob)
    return blob


LOG_KEYS = ("stoc_pol_mean", "stoc_pol_std", "stoc_pol_max", "stoc_pol_min", "success_percentage", "eval_score", "eval_success", "iteration", "best_stoc_pol_mean", "best_iteration")


def load_npz(path=os.path.join(os.path.dirname(os.path.abspath(__file__)), "npg_policies.npz")):
    """-> {env_id: [policy dict + 'logged' dict, ...]} from the committed fixture."""
    z = np.load(path)
    out = {}
    for key in sorted({"/".join(k.split("/")[:2]) for k in z.files}):
        env_id, _ = key.split("/")
        nl = len([k for k in z.files if k.startswith(key + "/W")])
        p = dict(W=[z[key + "/W%d" % i].astype(np.float64) for i in range(nl)], b=[z[key + "/b%d" % i].astype(np.float64) for i in range(nl)])
        for f in ("in_shift", "in_scale", "out_shift", "out_scale", "log_std"):
            p[f] = z[key + "/" + f].astype(np.float64)
        p["logged"] = dict(zip(LOG_KEYS, z[key + "/logged"]))
        p["n"], p["m"] = p["W"][0].shape[1], p["W"][-1].shape[0]
        out.setdefault(env_id, []).append(p)
    return out


if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "npg_policies.npz")
    pack(out)
    for env_id, ps in load_npz(out).items():
        for p in ps:
            print(env_id, "obs", p["n"], "act", p["m"], "log_std %.2f" % p["log_std"].mean(), {k: round(float(v), 2) for k, v in p["logged"].items()})
    print(os.path.getsize(out), "bytes")
