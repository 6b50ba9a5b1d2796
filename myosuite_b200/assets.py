"""Model assets: name -> compiled Model.

Models are compiled from the simhive MJCF files when a MyoSuite checkout is reachable
(``MYOSUITE_ROOT`` env var, or an installed ``myosuite`` package), otherwise the
pre-compiled fixtures committed under ``myosuite_b200/assets/`` (made by tools/compile_assets.py with this
repo's own compiler) are used.
"""
import os

from . import mjcf

# name -> (path relative to the myosuite package dir, compile kwargs)
MODEL_XML = {
    "myoelbow_1dof6muscles": ("envs/myo/assets/elbow/myoelbow_1dof6muscles.xml", {}),
    "myohand_pose": ("envs/myo/assets/hand/myohand_pose.xml", {}),
    "myohand_hold": ("envs/myo/assets/hand/myohand_hold.xml", {}),
    # Walk moves the hfield terrain out of reach (walk_v0.py:262-266): compile without it
    "myolegs": ("simhive/myo_sim/leg/myolegs.xml", {"drop_geoms": ("terrain",)}),
    "myotorso": ("simhive/myo_sim/torso/myotorso.xml", {}),
}
_HERE = os.path.dirname(os.path.abspath(__file__))
_CACHE = {}


def _myosuite_root():
    r = os.environ.get("MYOSUITE_ROOT")
    if r and os.path.isdir(r):
        return r
    try:
        import importlib.util
        spec = importlib.util.find_spec("myosuite")
        if spec and spec.submodule_search_locations:
            return list(spec.submodule_search_locations)[0]
    except Exception:
        pass
    return None


def model_from_xml(path, **kwargs):
    return mjcf.compile_mjcf(path, **kwargs)


def load(name, prefer_xml=False):
    if name in _CACHE:
        return _CACHE[name]
    rel, kwargs = MODEL_XML[name]
    npz = os.path.join(_HERE, "assets", name + ".npz")
    root = _myosuite_root()
    if root and (prefer_xml or not os.path.exists(npz)) and os.path.exists(os.path.join(root, rel)):
        m = mjcf.compile_mjcf(os.path.join(root, rel), **kwargs)
    elif os.path.exists(npz):
        m = mjcf.load_model(npz)
    else:
        raise FileNotFoundError("model %r: no MyoSuite checkout (set MYOSUITE_ROOT) and no compiled fixture %s" % (name, npz))
    _CACHE[name] = m
    return m
