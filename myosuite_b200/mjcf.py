"""MJCF loader + model compiler for the subset of MJCF used by the MyoSuite hot-path models.

Replaces the reference's loader seam ``mujoco.MjSpec.from_file(path).compile()``
(myosuite/envs/env_base.py:70-72,96-106).  MuJoCo itself is third-party and absent,
so the compile rules below restate MuJoCo's documented XML semantics (SURVEY.md Appendix A.7/B.3):
includes, nested default classes + childclass, euler/fromto/zaxis frames, explicit and geom-derived
inertia (incl. binary-STL mesh inertia), the <muscle> shortcut, spatial tendons with sphere/cylinder
wraps and side-sites, joint equalities, contact pairs/excludes, keyframes, and the compile-time
constants (qpos0, invweight0, meaninertia).

Output: a :class:`Model` -- a bag of numpy arrays named after the ``mjModel`` fields the path reads
(SURVEY.md Appendix B.2) so that host code written against ``mj_model.<field>`` keeps working.
"""
import os
import struct
import xml.etree.ElementTree as ET

import numpy as np

from . import mjmath as mm

# enums (values follow mujoco's mjtJoint / mjtGeom / mjtWrap / mjtDyn / mjtGain / mjtBias / mjtTrn)
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = 0, 1, 2, 3
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = range(8)
WRAP_NONE, WRAP_JOINT, WRAP_PULLEY, WRAP_SITE, WRAP_SPHERE, WRAP_CYLINDER = range(6)
DYN_NONE, DYN_INTEGRATOR, DYN_FILTER, DYN_FILTEREXACT, DYN_MUSCLE, DYN_USER = range(6)
GAIN_FIXED, GAIN_AFFINE, GAIN_MUSCLE, GAIN_USER = range(4)
BIAS_NONE, BIAS_AFFINE, BIAS_MUSCLE, BIAS_USER = range(4)
TRN_JOINT, TRN_JOINTINPARENT, TRN_SLIDERCRANK, TRN_TENDON, TRN_SITE, TRN_BODY = range(6)
EQ_CONNECT, EQ_WELD, EQ_JOINT, EQ_TENDON = 0, 1, 2, 3

GEOM_TYPES = {"plane": 0, "hfield": 1, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6, "mesh": 7}
NPRM = 10  # mjNDYN = mjNGAIN = mjNBIAS
MINVAL = 1e-15
DEFAULT_SOLREF = (0.02, 1.0)
DEFAULT_SOLIMP = (0.9, 0.95, 0.001, 0.5, 2.0)


class MJCFError(ValueError):
    pass


class Model:
    """Compiled model: numpy arrays named like mjModel fields, plus name->id maps."""

    def __init__(self):
        self.names = {k: {} for k in ("body", "joint", "geom", "site", "tendon", "actuator", "equality", "mesh")}

    def name2id(self, kind, name):
        try:
            return self.names[kind][name]
        except KeyError:
            raise KeyError("no %s named %r" % (kind, name))

    def id2name(self, kind, idx):
        for k, v in self.names[kind].items():
            if v == idx:
                return k
        return None


# ----------------------------------------------------------------------------- XML loading

def _fvec(s, n=None, default=None):
    if s is None:
        return None if default is None else np.array(default, dtype=np.float64)
    v = np.array([float(x) for x in s.replace(",", " ").split()], dtype=np.float64)
    if n is not None and default is not None and len(v) < n:
        full = np.array(default, dtype=np.float64)
        full[: len(v)] = v
        v = full
    return v


def _expand_includes(elem, base_dir, main_dir, depth=0):
    if depth > 8:
        raise MJCFError("include depth")
    out = []
    for child in list(elem):
        if child.tag == "include":
            f = child.get("file")
            path = os.path.join(base_dir, f)
            if not os.path.exists(path):
                path = os.path.join(main_dir, f)
            if not os.path.exists(path):
                raise MJCFError("include not found: %s" % f)
            sub = ET.parse(path).getroot()
            _expand_includes(sub, os.path.dirname(path), main_dir, depth + 1)
            out.extend(list(sub))
        else:
            _expand_includes(child, base_dir, main_dir, depth)
            out.append(child)
    for c in list(elem):
        elem.remove(c)
    for c in out:
        elem.append(c)


def load_xml(path):
    path = os.path.abspath(path)
    root = ET.parse(path).getroot()
    if root.tag != "mujoco":
        raise MJCFError("root element must be <mujoco>")
    d = os.path.dirname(path)
    _expand_includes(root, d, d)
    return root, d


# ----------------------------------------------------------------------------- defaults

def _new_actuator_default():
    return dict(dyntype=DYN_NONE, gaintype=GAIN_FIXED, biastype=BIAS_NONE,
                dynprm=[1.0] + [0.0] * (NPRM - 1), gainprm=[1.0] + [0.0] * (NPRM - 1), biasprm=[0.0] * NPRM,
                ctrllimited="auto", ctrlrange=[0.0, 0.0], forcelimited="auto", forcerange=[0.0, 0.0],
                actlimited="auto", actrange=[0.0, 0.0], gear=[1.0, 0, 0, 0, 0, 0], lengthrange=[0.0, 0.0],
                tendon=None, joint=None, name=None)


_DYN = {"none": DYN_NONE, "integrator": DYN_INTEGRATOR, "filter": DYN_FILTER, "filterexact": DYN_FILTEREXACT,
        "muscle": DYN_MUSCLE, "user": DYN_USER}
_GAIN = {"fixed": GAIN_FIXED, "affine": GAIN_AFFINE, "muscle": GAIN_MUSCLE, "user": GAIN_USER}
_BIAS = {"none": BIAS_NONE, "affine": BIAS_AFFINE, "muscle": BIAS_MUSCLE, "user": BIAS_USER}


def _set_partial(dst, s):
    v = [float(x) for x in s.split()]
    dst[: len(v)] = v


def _apply_actuator(act, tag, attrib):
    """Apply <general>/<muscle> attributes onto a resolved actuator dict (used for defaults and elements)."""
    a = attrib
    for k in ("name", "tendon", "joint"):
        if k in a:
            act[k] = a[k]
    for k in ("ctrllimited", "forcelimited", "actlimited"):
        if k in a:
            act[k] = a[k]
    for k in ("ctrlrange", "forcerange", "actrange", "lengthrange"):
        if k in a:
            act[k] = [float(x) for x in a[k].split()]
    if "gear" in a:
        _set_partial(act["gear"], a["gear"])
    if tag == "general":
        if "dyntype" in a:
            act["dyntype"] = _DYN[a["dyntype"]]
        if "gaintype" in a:
            act["gaintype"] = _GAIN[a["gaintype"]]
        if "biastype" in a:
            act["biastype"] = _BIAS[a["biastype"]]
        for k in ("dynprm", "gainprm", "biasprm"):
            if k in a:
                _set_partial(act[k], a[k])
    elif tag == "muscle":
        # MuJoCo's <muscle> shortcut: switch to muscle defaults where the general defaults are untouched
        g, dprm = act["gainprm"], act["dynprm"]
        if dprm[0] == 1:
            dprm[0] = 0.01
        if dprm[1] == 0:
            dprm[1] = 0.04
        if g[0] == 1:
            g[0] = 0.75
        for i, dv in ((1, 1.05), (2, -1.0), (3, 200.0), (4, 0.5), (5, 1.6), (6, 1.5), (7, 1.3), (8, 1.2)):
            if g[i] == 0:
                g[i] = dv
        if "timeconst" in a:
            _set_partial(dprm, a["timeconst"])
        if "tausmooth" in a:
            dprm[2] = float(a["tausmooth"])
        if "range" in a:
            _set_partial(g, a["range"])
        for k, i in (("force", 2), ("scale", 3), ("lmin", 4), ("lmax", 5), ("vmax", 6), ("fpmax", 7), ("fvmax", 8)):
            if k in a:
                g[i] = float(a[k])
        act["biasprm"] = list(g)
        act["dyntype"], act["gaintype"], act["biastype"] = DYN_MUSCLE, GAIN_MUSCLE, BIAS_MUSCLE
    else:
        raise MJCFError("unsupported actuator element <%s>" % tag)


class _DefClass:
    SIMPLE = ("joint", "geom", "site", "tendon", "mesh", "pair", "equality")

    def __init__(self, parent=None):
        if parent is None:
            self.attr = {k: {} for k in self.SIMPLE}
            self.act = _new_actuator_default()
        else:
            self.attr = {k: dict(v) for k, v in parent.attr.items()}
            self.act = {k: (list(v) if isinstance(v, list) else v) for k, v in parent.act.items()}


def _parse_defaults(root):
    classes = {"main": _DefClass()}

    def rec(elem, cls):
        for ch in elem:
            if ch.tag == "default":
                name = ch.get("class")
                if name is None:
                    raise MJCFError("nested default without class")
                sub = _DefClass(cls)
                classes[name] = sub
                rec(ch, sub)
            elif ch.tag in _DefClass.SIMPLE:
                cls.attr[ch.tag].update(ch.attrib)
            elif ch.tag in ("general", "muscle"):
                _apply_actuator(cls.act, ch.tag, ch.attrib)
            # camera/light/material/... defaults are irrelevant to the path

    for d in root.findall("default"):
        name = d.get("class")
        if name in (None, "main"):
            rec(d, classes["main"])
        else:  # top-level named class
            sub = _DefClass(classes["main"])
            classes[name] = sub
            rec(d, sub)
    # children defined before a parent got later attributes: MuJoCo processes in document order too
    return classes


# ----------------------------------------------------------------------------- geometry helpers

def _frame_quat(a, comp):
    if "quat" in a:
        return mm.quat_normalize(_fvec(a["quat"]))
    if "euler" in a:
        e = _fvec(a["euler"])
        if comp["angle"] == "degree":
            e = np.deg2rad(e)
        return mm.euler2quat(e, comp["eulerseq"])
    if "axisangle" in a:
        v = _fvec(a["axisangle"])
        ang = np.deg2rad(v[3]) if comp["angle"] == "degree" else v[3]
        return mm.quat_normalize(mm.axisangle2quat(v[:3], ang))
    if "zaxis" in a:
        return mm.z2quat(_fvec(a["zaxis"]))
    if "xyaxes" in a:
        v = _fvec(a["xyaxes"])
        x = v[:3] / np.linalg.norm(v[:3])
        y = v[3:] - x * np.dot(x, v[3:])
        y /= np.linalg.norm(y)
        return mm.mat2quat(np.stack([x, y, np.cross(x, y)], axis=1))
    return np.array([1.0, 0.0, 0.0, 0.0])


def _eig_inertia(full):
    """Symmetric 3x3 -> (principal moments sorted descending, quaternion of the principal frame)."""
    w, v = np.linalg.eigh(full)
    order = np.argsort(-w)
    w = w[order]
    v = v[:, order]
    if np.linalg.det(v) < 0:
        v[:, 2] = -v[:, 2]
    return w, mm.mat2quat(v)


def read_stl(path):
    with open(path, "rb") as f:
        data = f.read()
    ntri = struct.unpack_from("<I", data, 80)[0]
    if 84 + 50 * ntri != len(data):
        raise MJCFError("not a binary STL: %s" % path)
    rec = np.frombuffer(data, dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("a", "<u2")]), count=ntri, offset=84)
    return rec["v"].astype(np.float64)  # [ntri, 3, 3]


def mesh_mass_props(tris, mode="legacy"):
    """Volume, COM and full inertia (unit density) of a triangle mesh.

    'legacy' restates MuJoCo's historical rule: apex at the area-weighted face centroid and
    absolute tetrahedron volumes; 'exact' uses signed volumes about the origin.
    """
    v0, v1, v2 = tris[:, 0], tris[:, 1], tris[:, 2]
    cen = (v0 + v1 + v2) / 3.0
    nrm = np.cross(v1 - v0, v2 - v0)
    area = 0.5 * np.linalg.norm(nrm, axis=1)
    facecen = (cen * area[:, None]).sum(0) / area.sum() if mode == "legacy" else np.zeros(3)
    a, b, c = v0 - facecen, v1 - facecen, v2 - facecen
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)) / 6.0
    if mode == "legacy":
        vol = np.abs(vol)
    volume = vol.sum()
    com = ((a + b + c) / 4.0 * vol[:, None]).sum(0) / volume + facecen
    a, b, c = v0 - com, v1 - com, v2 - com
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)) / 6.0
    if mode == "legacy":
        vol = np.abs(vol)
    # second moments of a tetrahedron (origin, a, b, c): int x_i x_j dV = V/20 * (sum_k p_k_i p_k_j + s_i s_j), s=a+b+c
    s = a + b + c
    P = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            P[i, j] = (vol / 20.0 * (a[:, i] * a[:, j] + b[:, i] * b[:, j] + c[:, i] * c[:, j] + s[:, i] * s[:, j])).sum()
    full = np.eye(3) * np.trace(P) - P
    return volume, com, full


def _geom_volume_inertia(gtype, size):
    """(volume, principal inertia per unit density) of a primitive in its own frame."""
    if gtype == GEOM_SPHERE:
        r = size[0]
        v = 4.0 / 3.0 * np.pi * r ** 3
        return v, np.full(3, 0.4 * v * r * r)
    if gtype == GEOM_CAPSULE:
        r, h = size[0], 2 * size[1]
        vc, vs = np.pi * r * r * h, 4.0 / 3.0 * np.pi * r ** 3
        ixx = vc * (h * h / 12 + r * r / 4) + vs * (0.4 * r * r + h * h / 4 + 0.375 * h * r)
        izz = vc * r * r / 2 + vs * 0.4 * r * r
        return vc + vs, np.array([ixx, ixx, izz])
    if gtype == GEOM_CYLINDER:
        r, h = size[0], 2 * size[1]
        v = np.pi * r * r * h
        ixx = v * (3 * r * r + h * h) / 12
        return v, np.array([ixx, ixx, v * r * r / 2])
    if gtype == GEOM_ELLIPSOID:
        a, b, c = size
        v = 4.0 / 3.0 * np.pi * a * b * c
        return v, v / 5 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
    if gtype == GEOM_BOX:
        a, b, c = size
        v = 8 * a * b * c
        return v, v / 3 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
    return 0.0, np.zeros(3)


def _rbound(gtype, size):
    if gtype == GEOM_SPHERE:
        return size[0]
    if gtype == GEOM_CAPSULE:
        return size[0] + size[1]
    if gtype == GEOM_CYLINDER:
        return float(np.hypot(size[0], size[1]))
    if gtype == GEOM_ELLIPSOID:
        return float(np.max(size))
    if gtype == GEOM_BOX:
        return float(np.linalg.norm(size))
    return 0.0


# ----------------------------------------------------------------------------- compiler

class _Body:
    def __init__(self):
        self.name = None
        self.parent = -1
        self.pos = np.zeros(3)
        self.quat = np.array([1.0, 0, 0, 0])
        self.inertial = None
        self.joints, self.geoms, self.sites = [], [], []


def compile_mjcf(path, mesh_inertia="legacy", drop_geoms=()):
    """Parse + compile an MJCF file into a :class:`Model`.

    drop_geoms: geom names removed from collision (the Walk task moves the hfield out of reach,
    myosuite/envs/myo/myobase/walk_v0.py:262-266 -- mirrored by dropping it).
    """
    root, main_dir = load_xml(path)
    comp = dict(angle="degree", eulerseq="xyz", inertiafromgeom="auto", balanceinertia=False,
                boundmass=0.0, boundinertia=0.0, meshdir="", autolimits=True, settotalmass=-1.0)
    for c in root.findall("compiler"):
        for k, v in c.attrib.items():
            if k in ("angle", "eulerseq", "inertiafromgeom", "meshdir"):
                comp[k] = v
            elif k in ("balanceinertia", "autolimits"):
                comp[k] = v == "true"
            elif k in ("boundmass", "boundinertia", "settotalmass"):
                comp[k] = float(v)
    opt = dict(timestep=0.002, gravity=np.array([0, 0, -9.81]), iterations=100, tolerance=1e-8,
               ls_iterations=50, ls_tolerance=0.01, impratio=1.0)
    for o in root.findall("option"):
        for k, v in o.attrib.items():
            if k == "gravity":
                opt[k] = _fvec(v)
            elif k in ("timestep", "tolerance", "ls_tolerance", "impratio"):
                opt[k] = float(v)
            elif k in ("iterations", "ls_iterations"):
                opt[k] = int(v)
            elif k in ("integrator", "solver", "cone", "jacobian"):
                if v not in ("Euler", "Newton", "pyramidal", "auto", "dense", "sparse"):
                    raise MJCFError("unsupported option %s=%s" % (k, v))
    classes = _parse_defaults(root)

    def merged(tag, elem, childclass):
        cname = elem.get("class") or childclass or "main"
        if cname not in classes:
            raise MJCFError("unknown default class %r" % cname)
        a = dict(classes[cname].attr.get(tag, {}))
        a.update(elem.attrib)
        return a

    # ---- assets (meshes only)
    meshes = {}
    for asset in root.findall("asset"):
        for me in asset.findall("mesh"):
            a = merged("mesh", me, None)
            name = a.get("name") or os.path.splitext(os.path.basename(a["file"]))[0]
            meshes[name] = dict(file=a.get("file"), scale=_fvec(a.get("scale"), 3, (1, 1, 1)), props=None)

    def mesh_props(name):
        me = meshes[name]
        if me["props"] is None:
            f = me["file"]
            p = f if os.path.isabs(f) else os.path.join(main_dir, comp["meshdir"], f)
            if not p.lower().endswith(".stl"):
                raise MJCFError("mesh inertia needs STL: %s" % p)
            tris = read_stl(p) * me["scale"]
            vol, com, full = mesh_mass_props(tris, mesh_inertia)
            w, q = _eig_inertia(full)
            verts = tris.reshape(-1, 3)
            me["props"] = dict(volume=vol, com=com, inertia=w, quat=q,
                               rbound=float(np.linalg.norm(verts - com, axis=1).max()))
        return me["props"]

    # ---- bodies (depth-first pre-order, like MuJoCo)
    bodies = []

    def parse_body_contents(elem, bid, childclass):
        b = bodies[bid]
        for ch in elem:
            if ch.tag == "inertial":
                a = ch.attrib
                ine = dict(pos=_fvec(a.get("pos"), 3, (0, 0, 0)), mass=float(a["mass"]))
                q = _frame_quat(a, comp)
                if "fullinertia" in a:
                    f = _fvec(a["fullinertia"])
                    full = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
                    w, qe = _eig_inertia(full)
                    ine["inertia"], ine["quat"] = w, mm.quat_normalize(mm.quat_mul(q, qe))
                else:
                    ine["inertia"], ine["quat"] = _fvec(a["diaginertia"]), q
                b.inertial = ine
            elif ch.tag in ("joint", "freejoint"):
                if ch.tag == "freejoint":
                    a = dict(ch.attrib)
                    a["type"] = "free"
                else:
                    a = merged("joint", ch, childclass)
                b.joints.append(a)
            elif ch.tag == "geom":
                b.geoms.append(merged("geom", ch, childclass))
            elif ch.tag == "site":
                b.sites.append(merged("site", ch, childclass))
            elif ch.tag == "body":
                nb = _Body()
                nb.name = ch.get("name")
                nb.parent = bid
                nb.pos = _fvec(ch.get("pos"), 3, (0, 0, 0))
                nb.quat = _frame_quat(ch.attrib, comp)
                bodies.append(nb)
                parse_body_contents(ch, len(bodies) - 1, ch.get("childclass") or childclass)
            elif ch.tag in ("camera", "light", "composite", "flexcomp"):
                pass
            elif ch.tag == "frame":
                raise MJCFError("<frame> not supported")

    world = _Body()
    world.name = "world"
    bodies.append(world)
    for wb in root.findall("worldbody"):
        parse_body_contents(wb, 0, wb.get("childclass"))

    m = Model()
    m.opt_timestep = float(opt["timestep"])
    m.opt_gravity = np.asarray(opt["gravity"], dtype=np.float64)
    m.opt_iterations, m.opt_tolerance = int(opt["iterations"]), float(opt["tolerance"])
    m.opt_ls_iterations, m.opt_ls_tolerance = int(opt["ls_iterations"]), float(opt["ls_tolerance"])
    m.opt_impratio = float(opt["impratio"])
    nbody = m.nbody = len(bodies)
    m.body_parentid = np.array([max(b.parent, 0) for b in bodies], dtype=np.int32)
    m.body_pos = np.array([b.pos for b in bodies])
    m.body_quat = np.array([b.quat for b in bodies])
    for i, b in enumerate(bodies):
        if b.name:
            m.names["body"][b.name] = i

    # ---- joints / dofs
    jt, jq, jd, jb, jpos, jax, jrange, jlim, jstiff, jmargin, jsolref, jsolimp = ([] for _ in range(12))
    dof_body, dof_jnt, dof_arm, dof_damp, qpos0 = [], [], [], [], []
    body_jntadr, body_jntnum = np.full(nbody, -1, np.int32), np.zeros(nbody, np.int32)
    body_dofadr, body_dofnum = np.full(nbody, -1, np.int32), np.zeros(nbody, np.int32)
    nq = nv = 0
    for bi, b in enumerate(bodies):
        for a in b.joints:
            jid = len(jt)
            if body_jntnum[bi] == 0:
                body_jntadr[bi], body_dofadr[bi] = jid, nv
            body_jntnum[bi] += 1
            tname = a.get("type", "hinge")
            t = {"free": JNT_FREE, "ball": JNT_BALL, "slide": JNT_SLIDE, "hinge": JNT_HINGE}[tname]
            if t == JNT_BALL:
                raise MJCFError("ball joints are not used by the hot-path models")
            if a.get("name"):
                m.names["joint"][a["name"]] = jid
            jt.append(t); jq.append(nq); jd.append(nv); jb.append(bi)
            jpos.append(_fvec(a.get("pos"), 3, (0, 0, 0)))
            ax = _fvec(a.get("axis"), 3, (0, 0, 1))
            jax.append(ax / max(np.linalg.norm(ax), MINVAL))
            rng = _fvec(a.get("range"), 2, (0, 0))
            if comp["angle"] == "degree" and t == JNT_HINGE:
                rng = np.deg2rad(rng)
            lim = a.get("limited", "auto")
            limited = (lim == "true") or (lim == "auto" and comp["autolimits"] and rng[0] < rng[1])
            jrange.append(rng); jlim.append(bool(limited) and t != JNT_FREE)
            jstiff.append(float(a.get("stiffness", 0))); jmargin.append(float(a.get("margin", 0)))
            jsolref.append(_fvec(a.get("solreflimit"), 2, DEFAULT_SOLREF))
            jsolimp.append(_fvec(a.get("solimplimit"), 5, DEFAULT_SOLIMP))
            if float(a.get("frictionloss", 0)) != 0:
                raise MJCFError("frictionloss not supported")
            ndof = 6 if t == JNT_FREE else 1
            for k in range(ndof):
                dof_body.append(bi); dof_jnt.append(jid)
                dof_arm.append(float(a.get("armature", 0))); dof_damp.append(float(a.get("damping", 0)))
            body_dofnum[bi] += ndof
            if t == JNT_FREE:
                qpos0.extend(list(b.pos) + list(b.quat))
                nq += 7
            else:
                ref = float(a.get("ref", 0))
                if comp["angle"] == "degree" and t == JNT_HINGE:
                    ref = np.deg2rad(ref)
                qpos0.append(ref)
                nq += 1
            nv += ndof
    m.nq, m.nv, m.njnt = nq, nv, len(jt)
    m.jnt_type = np.array(jt, np.int32); m.jnt_qposadr = np.array(jq, np.int32); m.jnt_dofadr = np.array(jd, np.int32)
    m.jnt_bodyid = np.array(jb, np.int32)
    m.jnt_pos = np.array(jpos).reshape(-1, 3); m.jnt_axis = np.array(jax).reshape(-1, 3)
    m.jnt_range = np.array(jrange).reshape(-1, 2); m.jnt_limited = np.array(jlim, np.uint8)
    m.jnt_stiffness = np.array(jstiff); m.jnt_margin = np.array(jmargin)
    m.jnt_solref = np.array(jsolref).reshape(-1, 2); m.jnt_solimp = np.array(jsolimp).reshape(-1, 5)
    m.dof_bodyid = np.array(dof_body, np.int32); m.dof_jntid = np.array(dof_jnt, np.int32)
    m.dof_armature = np.array(dof_arm); m.dof_damping = np.array(dof_damp)
    m.qpos0 = np.array(qpos0); m.qpos_spring = m.qpos0.copy()
    m.body_jntadr, m.body_jntnum, m.body_dofadr, m.body_dofnum = body_jntadr, body_jntnum, body_dofadr, body_dofnum
    # dof_parentid: previous dof in the same body, else last dof of the nearest ancestor with dofs
    dpar = np.full(nv, -1, np.int32)
    for bi in range(nbody):
        if body_dofnum[bi] == 0:
            continue
        p = m.body_parentid[bi]
        last = -1
        while True:
            if body_dofnum[p] > 0:
                last = body_dofadr[p] + body_dofnum[p] - 1
                break
            if p == 0:
                break
            p = m.body_parentid[p]
        for k in range(body_dofnum[bi]):
            d = body_dofadr[bi] + k
            dpar[d] = last if k == 0 else d - 1
    m.dof_parentid = dpar
    madr, nM = np.zeros(nv, np.int32), 0
    for d in range(nv):
        madr[d] = nM
        k = d
        while k >= 0:
            nM += 1
            k = dpar[k]
    m.dof_Madr, m.nM = madr, nM
    weld, rootid = np.zeros(nbody, np.int32), np.zeros(nbody, np.int32)
    for bi in range(1, nbody):
        p = m.body_parentid[bi]
        weld[bi] = bi if body_jntnum[bi] > 0 else weld[p]
        rootid[bi] = bi if p == 0 else rootid[p]
    m.body_weldid, m.body_rootid = weld, rootid

    # ---- geoms
    G = dict(type=[], body=[], pos=[], quat=[], size=[], contype=[], conaffinity=[], condim=[], friction=[],
             margin=[], gap=[], solref=[], solimp=[], solmix=[], priority=[], rbound=[], group=[], mass=[], density=[],
             mesh=[])
    body_geomadr, body_geomnum = np.full(nbody, -1, np.int32), np.zeros(nbody, np.int32)
    for bi, b in enumerate(bodies):
        for a in b.geoms:
            gid = len(G["type"])
            if body_geomnum[bi] == 0:
                body_geomadr[bi] = gid
            body_geomnum[bi] += 1
            if a.get("name"):
                m.names["geom"][a["name"]] = gid
            t = GEOM_TYPES[a.get("type", "sphere")]
            size = _fvec(a.get("size"), 3, (0, 0, 0))
            pos = _fvec(a.get("pos"), 3, (0, 0, 0))
            quat = _frame_quat(a, comp)
            if "fromto" in a:
                ft = _fvec(a["fromto"])
                vec = ft[:3] - ft[3:]
                pos = 0.5 * (ft[:3] + ft[3:])
                size = np.array([size[0], np.linalg.norm(vec) / 2, 0.0])
                quat = mm.z2quat(vec)
            if t == GEOM_MESH:
                has_inertial = b.inertial is not None
                dynamic = weld[bi] != 0
                if dynamic and (not has_inertial or int(a.get("contype", 1)) or int(a.get("conaffinity", 1))):
                    mp = mesh_props(a["mesh"])
                    # the mesh is re-centred on its COM / principal axes; compose with the geom frame
                    pos = pos + mm.rot_vec(quat, mp["com"])
                    quat = mm.quat_normalize(mm.quat_mul(quat, mp["quat"]))
                    size = np.array([mp["rbound"], 0, 0])
            G["type"].append(t); G["body"].append(bi); G["pos"].append(pos); G["quat"].append(quat); G["size"].append(size)
            G["contype"].append(int(a.get("contype", 1))); G["conaffinity"].append(int(a.get("conaffinity", 1)))
            G["condim"].append(int(a.get("condim", 3)))
            G["friction"].append(_fvec(a.get("friction"), 3, (1, 0.005, 0.0001)))
            G["margin"].append(float(a.get("margin", 0))); G["gap"].append(float(a.get("gap", 0)))
            G["solref"].append(_fvec(a.get("solref"), 2, DEFAULT_SOLREF))
            G["solimp"].append(_fvec(a.get("solimp"), 5, DEFAULT_SOLIMP))
            G["solmix"].append(float(a.get("solmix", 1))); G["priority"].append(int(a.get("priority", 0)))
            G["group"].append(int(a.get("group", 0)))
            G["mass"].append(float(a["mass"]) if "mass" in a else np.nan); G["density"].append(float(a.get("density", 1000)))
            G["mesh"].append(a.get("mesh"))
            G["rbound"].append(size[0] if t == GEOM_MESH else _rbound(t, size))
    m.ngeom = len(G["type"])
    m.geom_type = np.array(G["type"], np.int32); m.geom_bodyid = np.array(G["body"], np.int32)
    m.geom_pos = np.array(G["pos"]).reshape(-1, 3); m.geom_quat = np.array(G["quat"]).reshape(-1, 4)
    m.geom_size = np.array(G["size"]).reshape(-1, 3)
    m.geom_contype = np.array(G["contype"], np.int32); m.geom_conaffinity = np.array(G["conaffinity"], np.int32)
    m.geom_condim = np.array(G["condim"], np.int32); m.geom_friction = np.array(G["friction"]).reshape(-1, 3)
    m.geom_margin = np.array(G["margin"]); m.geom_gap = np.array(G["gap"])
    m.geom_solref = np.array(G["solref"]).reshape(-1, 2); m.geom_solimp = np.array(G["solimp"]).reshape(-1, 5)
    m.geom_solmix = np.array(G["solmix"]); m.geom_priority = np.array(G["priority"], np.int32)
    m.geom_rbound = np.array(G["rbound"], dtype=np.float64); m.geom_group = np.array(G["group"], np.int32)
    m.body_geomadr, m.body_geomnum = body_geomadr, body_geomnum

    # ---- sites
    spos, squat, sbody, ssize = [], [], [], []
    for bi, b in enumerate(bodies):
        for a in b.sites:
            if a.get("name"):
                m.names["site"][a["name"]] = len(spos)
            spos.append(_fvec(a.get("pos"), 3, (0, 0, 0))); squat.append(_frame_quat(a, comp)); sbody.append(bi)
            ssize.append(_fvec(a.get("size"), 3, (0.005, 0.005, 0.005)))
    m.nsite = len(spos)
    m.site_pos = np.array(spos).reshape(-1, 3); m.site_quat = np.array(squat).reshape(-1, 4)
    m.site_bodyid = np.array(sbody, np.int32); m.site_size = np.array(ssize).reshape(-1, 3)

    # ---- body inertial properties
    bmass, bipos, biquat, binertia = np.zeros(nbody), np.zeros((nbody, 3)), np.tile([1.0, 0, 0, 0], (nbody, 1)), np.zeros((nbody, 3))
    for bi, b in enumerate(bodies):
        if bi == 0:
            continue
        if b.inertial is not None and comp["inertiafromgeom"] != "true":
            ine = b.inertial
            bmass[bi], bipos[bi], biquat[bi], binertia[bi] = ine["mass"], ine["pos"], ine["quat"], ine["inertia"]
        elif comp["inertiafromgeom"] != "false" and body_geomnum[bi] > 0 and weld[bi] != 0:
            tot, com, parts = 0.0, np.zeros(3), []
            for g in range(body_geomadr[bi], body_geomadr[bi] + body_geomnum[bi]):
                t = m.geom_type[g]
                if t == GEOM_MESH:
                    mp = mesh_props(G["mesh"][g])
                    vol, I = mp["volume"], mp["inertia"].copy()
                elif t in (GEOM_PLANE, GEOM_HFIELD):
                    continue
                else:
                    vol, I = _geom_volume_inertia(t, m.geom_size[g])
                if vol <= 0:
                    continue
                gm = G["mass"][g] if not np.isnan(G["mass"][g]) else G["density"][g] * vol
                I = I * (gm / vol)
                parts.append((gm, m.geom_pos[g], m.geom_quat[g], I))
                tot += gm
                com += gm * m.geom_pos[g]
            if tot > 0:
                com /= tot
                full = np.zeros((3, 3))
                for gm, p, q, I in parts:
                    R = mm.quat2mat(q)
                    d = p - com
                    full += R @ np.diag(I) @ R.T + gm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
                w, q = _eig_inertia(full)
                bmass[bi], bipos[bi], biquat[bi], binertia[bi] = tot, com, q, w
        # static bodies without <inertial> keep zero mass (never enter the dynamics)
        if comp["balanceinertia"]:
            I = binertia[bi]
            if I[0] + I[1] < I[2] or I[0] + I[2] < I[1] or I[1] + I[2] < I[0]:
                binertia[bi] = I.mean()
        if weld[bi] != 0 or b.inertial is not None:
            bmass[bi] = max(bmass[bi], comp["boundmass"])
            binertia[bi] = np.maximum(binertia[bi], comp["boundinertia"])
    m.body_mass, m.body_ipos, m.body_iquat, m.body_inertia = bmass, bipos, biquat, binertia

    # ---- tendons (spatial only)
    tadr, tnum, wtype, wobj, wprm = [], [], [], [], []
    for tsec in root.findall("tendon"):
        for te in tsec:
            if te.tag != "spatial":
                raise MJCFError("only spatial tendons are used by the hot-path models")
            a = merged("tendon", te, None)
            for k in ("stiffness", "damping", "frictionloss"):
                if float(a.get(k, 0)) != 0:
                    raise MJCFError("tendon %s not supported" % k)
            if a.get("limited", "false") == "true":
                raise MJCFError("tendon limits not supported")
            if a.get("name"):
                m.names["tendon"][a["name"]] = len(tadr)
            tadr.append(len(wtype)); n = 0
            for w in te:
                if w.tag == "site":
                    wtype.append(WRAP_SITE); wobj.append(m.name2id("site", w.get("site"))); wprm.append(-1.0)
                elif w.tag == "geom":
                    g = m.name2id("geom", w.get("geom"))
                    gt = m.geom_type[g]
                    if gt not in (GEOM_SPHERE, GEOM_CYLINDER):
                        raise MJCFError("tendon wrap geom must be sphere or cylinder")
                    wtype.append(WRAP_SPHERE if gt == GEOM_SPHERE else WRAP_CYLINDER); wobj.append(g)
                    ss = w.get("sidesite")
                    wprm.append(float(m.name2id("site", ss)) if ss else -1.0)
                elif w.tag == "pulley":
                    raise MJCFError("pulleys not supported")
                n += 1
            tnum.append(n)
    m.ntendon, m.nwrap = len(tadr), len(wtype)
    m.tendon_adr, m.tendon_num = np.array(tadr, np.int32), np.array(tnum, np.int32)
    m.wrap_type, m.wrap_objid, m.wrap_prm = np.array(wtype, np.int32), np.array(wobj, np.int32), np.array(wprm, np.float64)

    # ---- actuators
    acts = []
    for asec in root.findall("actuator"):
        for ae in asec:
            cname = ae.get("class") or "main"
            base = classes[cname].act
            act = {k: (list(v) if isinstance(v, list) else v) for k, v in base.items()}
            _apply_actuator(act, ae.tag, ae.attrib)
            acts.append(act)
    nu = m.nu = len(acts)
    m.actuator_trntype = np.zeros(nu, np.int32); m.actuator_trnid = np.full((nu, 2), -1, np.int32)
    m.actuator_dyntype = np.zeros(nu, np.int32); m.actuator_gaintype = np.zeros(nu, np.int32); m.actuator_biastype = np.zeros(nu, np.int32)
    m.actuator_dynprm = np.zeros((nu, NPRM)); m.actuator_gainprm = np.zeros((nu, NPRM)); m.actuator_biasprm = np.zeros((nu, NPRM))
    m.actuator_ctrllimited = np.zeros(nu, np.uint8); m.actuator_ctrlrange = np.zeros((nu, 2))
    m.actuator_gear = np.zeros((nu, 6)); m.actuator_lengthrange = np.zeros((nu, 2)); m.actuator_acc0 = np.zeros(nu)
    for i, act in enumerate(acts):
        if act["name"]:
            m.names["actuator"][act["name"]] = i
        if act["tendon"] is not None:
            m.actuator_trntype[i], m.actuator_trnid[i, 0] = TRN_TENDON, m.name2id("tendon", act["tendon"])
        elif act["joint"] is not None:
            m.actuator_trntype[i], m.actuator_trnid[i, 0] = TRN_JOINT, m.name2id("joint", act["joint"])
        else:
            raise MJCFError("actuator transmission must be tendon or joint")
        m.actuator_dyntype[i], m.actuator_gaintype[i], m.actuator_biastype[i] = act["dyntype"], act["gaintype"], act["biastype"]
        m.actuator_dynprm[i], m.actuator_gainprm[i], m.actuator_biasprm[i] = act["dynprm"], act["gainprm"], act["biasprm"]
        cl = act["ctrllimited"]
        rng = act["ctrlrange"]
        m.actuator_ctrllimited[i] = (cl == "true") or (cl == "auto" and comp["autolimits"] and rng[0] < rng[1])
        m.actuator_ctrlrange[i] = rng
        for k in ("forcelimited", "actlimited"):
            if act[k] == "true":
                raise MJCFError("%s not supported" % k)
        m.actuator_gear[i] = act["gear"]; m.actuator_lengthrange[i] = act["lengthrange"]
        if act["dyntype"] == DYN_MUSCLE and act["gainprm"][2] < 0:
            raise MJCFError("muscle force<0 (acc0-scaled peak force) not supported: every hot-path muscle sets force")
        if act["gaintype"] == GAIN_MUSCLE and not (act["lengthrange"][0] < act["lengthrange"][1]):
            raise MJCFError("muscle without explicit lengthrange")
    m.na = int(np.sum(m.actuator_dyntype != DYN_NONE))
    if m.na not in (0, nu):
        raise MJCFError("mixed stateful/stateless actuators not supported")

    # ---- equality (joint polynomial couplings)
    e1, e2, edata, esolref, esolimp, eact = [], [], [], [], [], []
    for esec in root.findall("equality"):
        for ee in esec:
            if ee.tag != "joint":
                raise MJCFError("only <equality><joint> is used by the hot-path models")
            a = merged("equality", ee, None)
            if a.get("name"):
                m.names["equality"][a["name"]] = len(e1)
            e1.append(m.name2id("joint", a["joint1"])); e2.append(m.name2id("joint", a["joint2"]) if "joint2" in a else -1)
            edata.append(_fvec(a.get("polycoef"), 5, (0, 1, 0, 0, 0)))
            esolref.append(_fvec(a.get("solref"), 2, DEFAULT_SOLREF)); esolimp.append(_fvec(a.get("solimp"), 5, DEFAULT_SOLIMP))
            eact.append(a.get("active", "true") == "true")
    m.neq = len(e1)
    m.eq_type = np.full(m.neq, EQ_JOINT, np.int32)
    m.eq_obj1id, m.eq_obj2id = np.array(e1, np.int32), np.array(e2, np.int32)
    m.eq_data = np.array(edata).reshape(-1, 5); m.eq_solref = np.array(esolref).reshape(-1, 2)
    m.eq_solimp = np.array(esolimp).reshape(-1, 5); m.eq_active0 = np.array(eact, np.uint8)

    # ---- contact: excludes + explicit pairs
    excludes, xpairs = set(), []
    for csec in root.findall("contact"):
        for ce in csec:
            if ce.tag == "exclude":
                b1, b2 = m.name2id("body", ce.get("body1")), m.name2id("body", ce.get("body2"))
                excludes.add((min(b1, b2), max(b1, b2)))
            elif ce.tag == "pair":
                xpairs.append(merged("pair", ce, None))
    m.exclude_pairs = sorted(excludes)

    # ---- keyframes
    kq, kv = [], []
    for ksec in root.findall("keyframe"):
        for ke in ksec.findall("key"):
            kq.append(_fvec(ke.get("qpos"), nq, m.qpos0)); kv.append(_fvec(ke.get("qvel"), nv, np.zeros(nv)))
    m.nkey = len(kq)
    m.key_qpos = np.array(kq).reshape(-1, nq); m.key_qvel = np.array(kv).reshape(-1, nv)

    _set_const(m)
    _build_collision_pairs(m, xpairs, set(drop_geoms), meshes, mesh_props, G)
    m.source_path = os.path.abspath(path)
    return m


# ----------------------------------------------------------------------------- compile-time constants

def kinematics(m, qpos):
    """numpy forward kinematics (host-side utility; also used for compile-time constants)."""
    nb = m.nbody
    xpos, xquat = np.zeros((nb, 3)), np.tile([1.0, 0, 0, 0], (nb, 1))
    anchor, axis = np.zeros((m.njnt, 3)), np.zeros((m.njnt, 3))
    for b in range(1, nb):
        p = m.body_parentid[b]
        pos = xpos[p] + mm.rot_vec(xquat[p], m.body_pos[b])
        quat = mm.quat_mul(xquat[p], m.body_quat[b])
        for j in range(m.body_jntadr[b], m.body_jntadr[b] + m.body_jntnum[b]):
            qa = m.jnt_qposadr[j]
            t = m.jnt_type[j]
            if t == JNT_FREE:
                pos = qpos[qa:qa + 3].copy()
                quat = mm.quat_normalize(qpos[qa + 3:qa + 7])
                anchor[j], axis[j] = pos, np.array([0, 0, 1.0])
                continue
            anchor[j] = pos + mm.rot_vec(quat, m.jnt_pos[j])
            axis[j] = mm.rot_vec(quat, m.jnt_axis[j])
            if t == JNT_SLIDE:
                pos = pos + axis[j] * (qpos[qa] - m.qpos0[qa])
            else:
                quat = mm.quat_mul(quat, mm.axisangle2quat(m.jnt_axis[j], qpos[qa] - m.qpos0[qa]))
                pos = anchor[j] - mm.rot_vec(quat, m.jnt_pos[j])
        xpos[b], xquat[b] = pos, mm.quat_normalize(quat)
    xmat = np.array([mm.quat2mat(q) for q in xquat])
    xipos = xpos + np.einsum("bij,bj->bi", xmat, m.body_ipos)
    return dict(xpos=xpos, xquat=xquat, xmat=xmat, xipos=xipos, anchor=anchor, axis=axis)


def dof_chain(m, body):
    """dofs affecting a body, root first."""
    out = []
    b = body
    while b > 0:
        if m.body_dofnum[b] > 0:
            out = list(range(m.body_dofadr[b], m.body_dofadr[b] + m.body_dofnum[b])) + out
        b = m.body_parentid[b]
    return out


def jac_point(m, kin, point, body):
    """3xnv translational and rotational Jacobians of a world point attached to `body`."""
    jp, jr = np.zeros((3, m.nv)), np.zeros((3, m.nv))
    for d in dof_chain(m, body):
        j = m.dof_jntid[d]
        t = m.jnt_type[j]
        k = d - m.jnt_dofadr[j]
        if t == JNT_FREE:
            if k < 3:
                jp[k, d] = 1.0
            else:
                ax = kin["xmat"][m.jnt_bodyid[j]][:, k - 3]
                jr[:, d] = ax
                jp[:, d] = np.cross(ax, point - kin["xpos"][m.jnt_bodyid[j]])
        elif t == JNT_SLIDE:
            jp[:, d] = kin["axis"][j]
        else:
            jr[:, d] = kin["axis"][j]
            jp[:, d] = np.cross(kin["axis"][j], point - kin["anchor"][j])
    return jp, jr


def mass_matrix(m, kin):
    M = np.diag(m.dof_armature.astype(np.float64)).copy()
    for b in range(1, m.nbody):
        if m.body_weldid[b] == 0 or m.body_mass[b] == 0:
            continue
        jp, jr = jac_point(m, kin, kin["xipos"][b], b)
        R = kin["xmat"][b] @ mm.quat2mat(m.body_iquat[b])
        I = R @ np.diag(m.body_inertia[b]) @ R.T
        M += m.body_mass[b] * jp.T @ jp + jr.T @ I @ jr
    return M


def _set_const(m):
    nv = m.nv
    m.dof_invweight0 = np.zeros(nv); m.body_invweight0 = np.zeros((m.nbody, 2)); m.stat_meaninertia = 1.0
    m.body_subtreemass = m.body_mass.copy()
    for b in range(m.nbody - 1, 0, -1):
        m.body_subtreemass[m.body_parentid[b]] += m.body_subtreemass[b]
    if nv == 0:
        return
    kin = kinematics(m, m.qpos0)
    M = mass_matrix(m, kin)
    Minv = np.linalg.inv(M)
    m.stat_meaninertia = float(np.mean(np.diag(M)))
    for j in range(m.njnt):
        d = m.jnt_dofadr[j]
        if m.jnt_type[j] == JNT_FREE:
            m.dof_invweight0[d:d + 3] = np.mean(np.diag(Minv)[d:d + 3])
            m.dof_invweight0[d + 3:d + 6] = np.mean(np.diag(Minv)[d + 3:d + 6])
        else:
            m.dof_invweight0[d] = Minv[d, d]
    for b in range(1, m.nbody):
        if m.body_weldid[b] == 0:
            continue
        jp, jr = jac_point(m, kin, kin["xipos"][b], b)
        m.body_invweight0[b, 0] = np.trace(jp @ Minv @ jp.T) / 3
        m.body_invweight0[b, 1] = np.trace(jr @ Minv @ jr.T) / 3


# ----------------------------------------------------------------------------- collision candidate pairs

def _mix_params(m, g1, g2):
    p1, p2 = m.geom_priority[g1], m.geom_priority[g2]
    if p1 != p2:
        g = g1 if p1 > p2 else g2
        return dict(condim=int(m.geom_condim[g]), friction=m.geom_friction[g].copy(), solref=m.geom_solref[g].copy(),
                    solimp=m.geom_solimp[g].copy())
    s1, s2 = m.geom_solmix[g1], m.geom_solmix[g2]
    if s1 >= MINVAL and s2 >= MINVAL:
        mix = s1 / (s1 + s2)
    elif s1 < MINVAL and s2 < MINVAL:
        mix = 0.5
    else:
        mix = 0.0 if s1 < MINVAL else 1.0
    r1, r2 = m.geom_solref[g1], m.geom_solref[g2]
    solref = mix * r1 + (1 - mix) * r2 if (r1[0] > 0 and r2[0] > 0) else np.minimum(r1, r2)
    return dict(condim=int(max(m.geom_condim[g1], m.geom_condim[g2])),
                friction=np.maximum(m.geom_friction[g1], m.geom_friction[g2]),
                solref=solref, solimp=mix * m.geom_solimp[g1] + (1 - mix) * m.geom_solimp[g2])


def _reach_sphere(m, geom):
    """Conservative (centre, radius) of the region a geom can occupy, or None if unbounded (free joint)."""
    b = m.geom_bodyid[geom]
    reach = np.linalg.norm(m.geom_pos[geom]) + m.geom_rbound[geom]
    while b > 0 and m.body_weldid[b] != 0:
        for j in range(m.body_jntadr[b], m.body_jntadr[b] + m.body_jntnum[b]):
            if m.jnt_type[j] == JNT_FREE:
                return None
            if m.jnt_type[j] == JNT_SLIDE:
                if not m.jnt_limited[j]:
                    return None
                reach += np.max(np.abs(m.jnt_range[j] - m.qpos0[m.jnt_qposadr[j]]))
            # a hinge with an off-origin anchor swings the body origin on a circle of radius |jnt_pos| around the anchor
            reach += 2.0 * np.linalg.norm(m.jnt_pos[j])
        reach += np.linalg.norm(m.body_pos[b])
        b = m.body_parentid[b]
    # b is static: its world pose at qpos0 is its pose always
    kin = kinematics(m, m.qpos0)
    return kin["xpos"][b], reach


def _build_collision_pairs(m, xpairs, drop, meshes, mesh_props, G):
    """Static candidate list after MuJoCo's filters (contype/conaffinity, same weld body, parent-child
    with both dynamic, <exclude>), plus explicit <pair>s; sorted by (geom1, geom2).  Candidates that a
    conservative reach bound proves can never come within margin are dropped (recorded in
    ``m.pair_dropped``) -- this is how the unreachable floor/pedestal pairs disappear (SURVEY A.4)."""
    kin = kinematics(m, m.qpos0)
    cands = {}
    explicit = {}
    for a in xpairs:
        g1, g2 = m.name2id("geom", a["geom1"]), m.name2id("geom", a["geom2"])
        prm = _mix_params(m, g1, g2)
        if "condim" in a:
            prm["condim"] = int(a["condim"])
        if "friction" in a:
            f = _fvec(a["friction"], 5, (1, 1, 0.005, 0.0001, 0.0001))
            prm["friction5"] = f
        if "solref" in a:
            prm["solref"] = _fvec(a["solref"], 2, DEFAULT_SOLREF)
        if "solimp" in a:
            prm["solimp"] = _fvec(a["solimp"], 5, DEFAULT_SOLIMP)
        prm["margin"] = float(a["margin"]) if "margin" in a else max(m.geom_margin[g1], m.geom_margin[g2])
        prm["gap"] = float(a["gap"]) if "gap" in a else max(m.geom_gap[g1], m.geom_gap[g2])
        explicit[(g1, g2)] = prm
    collidable = [g for g in range(m.ngeom) if (m.geom_contype[g] or m.geom_conaffinity[g])]
    for i, g1 in enumerate(collidable):
        for g2 in collidable[i + 1:]:
            if not ((m.geom_contype[g1] & m.geom_conaffinity[g2]) or (m.geom_contype[g2] & m.geom_conaffinity[g1])):
                continue
            b1, b2 = m.geom_bodyid[g1], m.geom_bodyid[g2]
            w1, w2 = m.body_weldid[b1], m.body_weldid[b2]
            if w1 == w2:
                continue
            wp1, wp2 = m.body_weldid[m.body_parentid[w1]], m.body_weldid[m.body_parentid[w2]]
            if w1 != 0 and w2 != 0 and (w1 == wp2 or w2 == wp1):
                continue
            if (min(b1, b2), max(b1, b2)) in set(m.exclude_pairs):
                continue
            if (g1, g2) in explicit or (g2, g1) in explicit:
                continue
            prm = _mix_params(m, g1, g2)
            prm["margin"] = max(m.geom_margin[g1], m.geom_margin[g2])
            prm["gap"] = max(m.geom_gap[g1], m.geom_gap[g2])
            cands[(g1, g2)] = prm
    cands.update(explicit)
    names = {v: k for k, v in m.names["geom"].items()}
    kept, dropped = [], []
    for (g1, g2), prm in sorted(cands.items()):
        if names.get(g1) in drop or names.get(g2) in drop:
            dropped.append((g1, g2, "dropped by task"))
            continue
        # canonical order: lower geom type first (plane before sphere before capsule ...), like MuJoCo's collider table
        if m.geom_type[g1] > m.geom_type[g2]:
            g1, g2 = g2, g1
        reason = _unreachable(m, kin, g1, g2, prm["margin"])
        if reason:
            dropped.append((g1, g2, reason))
            continue
        kept.append((g1, g2, prm))
    m.npair = len(kept)
    m.pair_geom1 = np.array([k[0] for k in kept], np.int32); m.pair_geom2 = np.array([k[1] for k in kept], np.int32)
    m.pair_dim = np.array([k[2]["condim"] for k in kept], np.int32)
    fr = []
    for k in kept:
        p = k[2]
        if "friction5" in p:
            fr.append(p["friction5"])
        else:
            f = p["friction"]
            fr.append([f[0], f[0], f[1], f[2], f[2]])
    m.pair_friction = np.array(fr, dtype=np.float64).reshape(-1, 5)
    m.pair_solref = np.array([k[2]["solref"] for k in kept]).reshape(-1, 2)
    m.pair_solimp = np.array([k[2]["solimp"] for k in kept]).reshape(-1, 5)
    m.pair_margin = np.array([k[2]["margin"] for k in kept], dtype=np.float64)
    m.pair_gap = np.array([k[2]["gap"] for k in kept], dtype=np.float64)
    m.pair_dropped = dropped
    supported = {(GEOM_PLANE, GEOM_SPHERE), (GEOM_PLANE, GEOM_CAPSULE), (GEOM_SPHERE, GEOM_SPHERE),
                 (GEOM_SPHERE, GEOM_CAPSULE), (GEOM_CAPSULE, GEOM_CAPSULE), (GEOM_PLANE, GEOM_ELLIPSOID),
                 (GEOM_CAPSULE, GEOM_ELLIPSOID), (GEOM_ELLIPSOID, GEOM_ELLIPSOID)}
    m.pair_unsupported = [(int(a), int(b)) for a, b in zip(m.pair_geom1, m.pair_geom2)
                          if (int(m.geom_type[a]), int(m.geom_type[b])) not in supported]


def _unreachable(m, kin, g1, g2, margin):
    r1, r2 = _reach_sphere(m, g1), _reach_sphere(m, g2)
    if r1 is None or r2 is None:
        return None
    (c1, rad1), (c2, rad2) = r1, r2
    t1 = m.geom_type[g1]
    if t1 == GEOM_PLANE:
        b = m.geom_bodyid[g1]
        if m.body_weldid[b] != 0:
            return None
        R = kin["xmat"][b] @ mm.quat2mat(m.geom_quat[g1])
        p0 = kin["xpos"][b] + kin["xmat"][b] @ m.geom_pos[g1]
        dist = float(np.dot(R[:, 2], c2 - p0)) - rad2
        return "plane out of reach (%.3f m clear)" % dist if dist > margin else None
    if m.geom_type[g2] == GEOM_CYLINDER and m.body_weldid[m.geom_bodyid[g2]] == 0:
        g1, g2, c1, rad1, c2, rad2 = g2, g1, c2, rad2, c1, rad1
        t1 = GEOM_CYLINDER
    b1 = m.geom_bodyid[g1]
    if t1 == GEOM_CYLINDER and m.body_weldid[b1] == 0:
        # exact distance from the other geom's reach sphere to a static cylinder
        R = kin["xmat"][b1] @ mm.quat2mat(m.geom_quat[g1])
        loc = R.T @ (c2 - (kin["xpos"][b1] + kin["xmat"][b1] @ m.geom_pos[g1]))
        da, dr = abs(loc[2]) - m.geom_size[g1][1], np.hypot(loc[0], loc[1]) - m.geom_size[g1][0]
        dist = float(np.hypot(max(da, 0.0), max(dr, 0.0))) - rad2
        return "static cylinder out of reach (%.3f m clear)" % dist if dist > margin else None
    dist = float(np.linalg.norm(c1 - c2)) - rad1 - rad2
    return "bounding reach spheres %.3f m apart" % dist if dist > margin else None


# ----------------------------------------------------------------------------- (de)serialisation of compiled models

def save_model(m, path):
    """Write a compiled Model to a single .npz (arrays + a JSON blob of scalars / names)."""
    import json
    arrays, meta = {}, {"names": m.names, "scalars": {}, "lists": {}}
    for k, v in m.__dict__.items():
        if k == "names":
            continue
        if isinstance(v, np.ndarray):
            arrays[k] = v
        elif isinstance(v, (int, float, str, np.integer, np.floating)):
            meta["scalars"][k] = v.item() if hasattr(v, "item") else v
        elif isinstance(v, (list, tuple)):
            meta["lists"][k] = [list(map(lambda x: x.item() if hasattr(x, "item") else x, e)) if isinstance(e, (list, tuple)) else e for e in v]
    arrays["__meta__"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(path, **arrays)


def load_model(path):
    import json
    z = np.load(path, allow_pickle=False)
    m = Model()
    meta = json.loads(bytes(z["__meta__"]).decode())
    for k in z.files:
        if k != "__meta__":
            setattr(m, k, z[k])
    for k, v in meta["scalars"].items():
        setattr(m, k, v)
    for k, v in meta["lists"].items():
        setattr(m, k, [tuple(e) if isinstance(e, list) else e for e in v])
    m.names = meta["names"]
    return m
