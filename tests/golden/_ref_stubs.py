"""Import the UNMODIFIED reference Python modules in a container that lacks mujoco / gym.

Installs permissive stub modules for the absent third-party imports (mujoco, gym, gymnasium, ...) so
that pure-numpy reference code (fatigue.py, PoseEnvV0.get_obs_dict / get_reward_dict) can be executed to
generate golden vectors.  Used only by the golden-vector generators in this directory.
"""
import importlib
import importlib.machinery
import importlib.util
import os
import sys
import types

import numpy as np


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        v = _Stub(self.__name__ + "." + name)
        setattr(self, name, v)
        return v

    def __call__(self, *a, **k):
        return _Stub(self.__name__ + "()")

    def __iter__(self):
        return iter(())

    def __mro_entries__(self, bases):
        return (object,)


def install(ref_root=None):
    ref_root = ref_root or os.environ["MYOSUITE_CHECKOUT"]
    for name in ("mujoco", "gym", "gymnasium", "termcolor", "flatten_dict", "h5py", "imageio", "click", "skvideo", "skvideo.io",
                 "PIL", "PIL.Image", "dm_control", "git", "torchvision", "gymnasium.utils", "gym.utils", "gymnasium.envs", "gymnasium.envs.registration"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                st = _Stub(name)
                st.__spec__ = importlib.machinery.ModuleSpec(name, None)
                st.__path__ = []
                sys.modules[name] = st
    mj = sys.modules["mujoco"]
    mj.mjtDyn = types.SimpleNamespace(mjDYN_MUSCLE=4, mjDYN_NONE=0)
    mj.mjtTrn = types.SimpleNamespace(mjTRN_JOINT=0, mjTRN_TENDON=3)
    mj.mjtJoint = types.SimpleNamespace(mjJNT_FREE=0, mjJNT_BALL=1, mjJNT_SLIDE=2, mjJNT_HINGE=3)
    for g in ("gym", "gymnasium"):
        G = sys.modules[g]
        if isinstance(G, _Stub):
            G.__version__ = "0.29.1"
            G.utils.seeding.np_random = lambda seed=None: (np.random.default_rng(seed), seed)
            G.Env = type("Env", (), {})
            G.utils.EzPickle = type("EzPickle", (), {"__init__": lambda self, *a, **k: None})
    # minimal working registry so that `import myosuite` (which registers every suite) succeeds
    G = sys.modules["gymnasium"]
    if isinstance(G, _Stub):
        reg = {}

        def register(id, entry_point=None, max_episode_steps=None, kwargs=None, **kw):
            reg[id] = types.SimpleNamespace(id=id, entry_point=entry_point, max_episode_steps=max_episode_steps, kwargs=kwargs or {})
        G.register = register
        G.envs.registry = reg
        G.envs.registration.registry = reg
    fd = sys.modules["flatten_dict"]
    if isinstance(fd, _Stub):
        def flatten(d, reducer="dot", keep_empty_types=(), _pre=""):
            out = {}
            for k, v in d.items():
                key = _pre + "." + str(k) if _pre else str(k)
                if isinstance(v, dict) and v:
                    out.update(flatten(v, _pre=key))
                else:
                    out[key] = v
            return out

        def unflatten(d, splitter="dot"):
            out = {}
            for k, v in d.items():
                cur = out
                parts = k.split(".")
                for p_ in parts[:-1]:
                    cur = cur.setdefault(p_, {})
                cur[parts[-1]] = v
            return out
        fd.flatten, fd.unflatten = flatten, unflatten
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
