"""Dump the registry kwargs of the hot-path env ids from the reference into a JSON fixture.

Executes myosuite/envs/myo/myobase/__init__.py UNMODIFIED with `gym.register` and
`register_env_variant` stubbed to recorders (no gym / mujoco needed), and writes
myosuite_b200/assets/registry.json.  Run:  python tools/extract_registry.py <MyoSuite checkout root>
"""
import json
import os
import sys
import types

ref = sys.argv[1]
src = os.path.join(ref, "myosuite/envs/myo/myobase/__init__.py")
records, variants = {}, {}


def register(id, entry_point, max_episode_steps=None, kwargs=None, **kw):
    records[id] = dict(entry_point=entry_point, max_episode_steps=max_episode_steps, kwargs=kwargs or {})


def register_env_variant(env_id, variants, variant_id=None, silent=False):
    globals()["variants"][variant_id] = dict(base=env_id, variants=variants)


gym = types.SimpleNamespace(register=register)
for name, mod in (("myosuite", types.ModuleType("myosuite")), ("myosuite.utils", types.ModuleType("myosuite.utils")),
                  ("myosuite.envs", types.ModuleType("myosuite.envs")),
                  ("myosuite.envs.env_variants", types.ModuleType("myosuite.envs.env_variants"))):
    sys.modules[name] = mod
sys.modules["myosuite.utils"].gym = gym
sys.modules["myosuite.envs.env_variants"].register_env_variant = register_env_variant
g = {"__file__": src, "__name__": "myobase_registry"}
exec(compile(open(src).read(), src, "exec"), g)

WANT = ["myoElbowPose1D6MRandom-v0", "myoHandPoseRandom-v0", "myoLegWalk-v0", "myoHandObjHoldRandom-v0",
        "myoElbowPose1D6MFixed-v0", "myoHandPoseFixed-v0", "myoHandObjHoldFixed-v0", "myoHandReachFixed-v0", "myoHandReachRandom-v0", "myoTorsoPoseFixed-v0",
        "myoLegStandRandom-v0"]
pkg = os.path.join(ref, "myosuite")


def clean(v):
    import numpy as np
    if isinstance(v, dict):
        return {k: clean(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [clean(x) for x in v]
    if isinstance(v, np.ndarray):
        return v.tolist()
    if isinstance(v, (np.floating, np.integer)):
        return v.item()
    if isinstance(v, str) and v.startswith(pkg):
        return os.path.relpath(os.path.normpath(v), pkg)
    return v


out = {"envs": {}, "variants": {}}
for k in WANT:
    if k in records:
        out["envs"][k] = clean(records[k])
for vid, v in variants.items():
    if v["base"] in out["envs"]:
        out["variants"][vid] = clean(v)
dst = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "myosuite_b200", "assets", "registry.json")
json.dump(out, open(dst, "w"), indent=1, sort_keys=False)
print("wrote", dst, list(out["envs"]), len(out["variants"]), "variants")
