"""MJCF -> constant-table model compiler (host side, numpy).

This is the stand-in for ``mujoco.MjModel.from_xml_path`` at
``gymnasium_robotics/envs/robot_env.py:293`` (reference), restricted to the MJCF
subset the in-scope models use (SURVEY.md Appendix A).  It produces

* ``Full``   - an unfused, mjModel-like set of arrays (one entry per MJCF body), used to
               apply MuJoCo's compile-time rules (collision filtering on weld ids,
               ``body_invweight0`` / ``dof_invweight0`` at ``qpos0``, ``stat.meaninertia``);
* ``Model``  - the runtime model: jointless non-mocap bodies are fused into their parents
               (dynamically equivalent; MuJoCo's ``fusestatic``), collision candidates are
               a static pre-filtered pair list with pre-mixed contact parameters;
* a binary blob (``Model.to_blob()``) read by both the CUDA library and the CPU oracle
  through ``include/b200sim_model.h``.

Semantics follow the public MuJoCo documentation (XML reference / Computation chapters);
nothing here is copied from MuJoCo or from the reference.  Mesh geoms are represented by
the oriented bounding box of their vertices (see DESIGN.md "mesh proxy").
"""
from __future__ import annotations

import json
import os
import struct
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field

import numpy as np

# --------------------------------------------------------------------------------------
# enums shared with include/b200sim_model.h
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = 0, 1, 2, 3
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = range(8)
GEOM_NAMES = {"plane": 0, "hfield": 1, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6, "mesh": 7}
EQ_CONNECT, EQ_WELD, EQ_JOINT = 0, 1, 2
INT_EULER, INT_RK4 = 0, 1
MINVAL = 1e-15
BLOB_MAGIC = 0x4D303242  # "B20M"
BLOB_VERSION = 5


# --------------------------------------------------------------------------------------
# small quaternion / rotation helpers (w, x, y, z)
def qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return np.array([
        aw * bw - ax * bx - ay * by - az * bz,
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by - ax * bz + ay * bw + az * bx,
        aw * bz + ax * by - ay * bx + az * bw,
    ])


def qconj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def qnorm(q):
    q = np.asarray(q, dtype=np.float64)
    n = np.linalg.norm(q)
    return np.array([1.0, 0, 0, 0]) if n < MINVAL else q / n


def q2mat(q):
    w, x, y, z = q
    return np.array([
        [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ])


def mat2q(m):
    """Rotation matrix -> unit quaternion (largest-pivot method)."""
    t = np.trace(m)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s])
    elif m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
        s = np.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]) * 2
        q = np.array([(m[2, 1] - m[1, 2]) / s, 0.25 * s, (m[0, 1] + m[1, 0]) / s, (m[0, 2] + m[2, 0]) / s])
    elif m[1, 1] > m[2, 2]:
        s = np.sqrt(1.0 + m[1, 1] - m[0, 0] - m[2, 2]) * 2
        q = np.array([(m[0, 2] - m[2, 0]) / s, (m[0, 1] + m[1, 0]) / s, 0.25 * s, (m[1, 2] + m[2, 1]) / s])
    else:
        s = np.sqrt(1.0 + m[2, 2] - m[0, 0] - m[1, 1]) * 2
        q = np.array([(m[1, 0] - m[0, 1]) / s, (m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s, 0.25 * s])
    return qnorm(q)


def qrot(q, v):
    return q2mat(q) @ np.asarray(v, dtype=np.float64)


def axisangle2q(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * axis])


def euler2q(e, seq="xyz"):
    """MJCF ``euler`` attribute; lower-case letters are intrinsic rotations."""
    q = np.array([1.0, 0, 0, 0])
    for ang, ax in zip(e, seq):
        a = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1]}[ax.lower()]
        r = axisangle2q(a, ang)
        q = qmul(q, r) if ax.islower() else qmul(r, q)
    return q


def zaxis2q(v):
    """Quaternion rotating +z onto v (MJCF ``fromto`` / ``zaxis``)."""
    v = np.asarray(v, dtype=np.float64)
    v = v / np.linalg.norm(v)
    z = np.array([0, 0, 1.0])
    ax = np.cross(z, v)
    s = np.linalg.norm(ax)
    if s < 1e-10:
        return np.array([1.0, 0, 0, 0]) if v[2] > 0 else np.array([0, 1.0, 0, 0])
    ang = np.arctan2(s, v[2])
    return axisangle2q(ax / s, ang)


def floats(s, n=None, default=None):
    if s is None:
        return None if default is None else np.array(default, dtype=np.float64)
    a = np.array([float(x) for x in s.split()], dtype=np.float64)
    if n is not None and default is not None and len(a) < n:  # partial spec keeps default tail
        a = np.concatenate([a, np.asarray(default, dtype=np.float64)[len(a):]])
    return a


# --------------------------------------------------------------------------------------
# inertia helpers
def box_inertia(mass, size):
    x, y, z = size
    return mass / 3.0 * np.array([y * y + z * z, x * x + z * z, x * x + y * y])


def geom_volume_inertia(gtype, size):
    """Volume and unit-density diagonal inertia about the geom centre, in the geom frame."""
    if gtype == GEOM_BOX:
        v = 8 * size[0] * size[1] * size[2]
        return v, box_inertia(v, size)
    if gtype == GEOM_SPHERE:
        r = size[0]
        v = 4.0 / 3 * np.pi * r ** 3
        return v, np.full(3, 0.4 * v * r * r)
    if gtype == GEOM_CYLINDER:
        r, h = size[0], size[1]
        v = np.pi * r * r * 2 * h
        ixy = v * (3 * r * r + (2 * h) ** 2) / 12
        return v, np.array([ixy, ixy, v * r * r / 2])
    if gtype == GEOM_CAPSULE:
        r, h = size[0], size[1]
        vc = np.pi * r * r * 2 * h
        vs = 4.0 / 3 * np.pi * r ** 3
        v = vc + vs
        izz = vc * r * r / 2 + vs * 0.4 * r * r
        # hemispheres offset from the centre: each half-sphere com at h + 3r/8
        ixy = vc * (3 * r * r + 4 * h * h) / 12 + vs * (0.4 * r * r + h * h + 0.75 * h * r)
        return v, np.array([ixy, ixy, izz])
    if gtype == GEOM_ELLIPSOID:
        a, b, c = size
        v = 4.0 / 3 * np.pi * a * b * c
        return v, v / 5 * np.array([b * b + c * c, a * a + c * c, a * a + b * b])
    raise ValueError(f"no inertia rule for geom type {gtype}")


HULL_MAX_VERTS = 32


def hull_vertices(points, kmax=HULL_MAX_VERTS):
    """At most `kmax` vertices of the convex hull of `points` [n, 3]: the hull's own vertices (scipy / qhull) when there are few,
    otherwise the support points of a fixed direction set (axes, cube diagonals, a Fibonacci sphere) thinned by farthest-point
    selection -- an inner approximation whose support function is exact in the sampled directions.  Deterministic."""
    from scipy.spatial import ConvexHull

    pts = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    hv = pts[np.sort(ConvexHull(pts).vertices)]
    if len(hv) <= kmax:
        return hv
    dirs = [np.array(d, dtype=np.float64) for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))]
    dirs += [np.array((a, b, c), dtype=np.float64) for a in (-1, 1) for b in (-1, 1) for c in (-1, 1)]
    n, ga = 96, np.pi * (3.0 - np.sqrt(5.0))
    for i in range(n):
        z = 1.0 - 2.0 * (i + 0.5) / n
        r = np.sqrt(max(0.0, 1.0 - z * z))
        dirs.append(np.array((r * np.cos(ga * i), r * np.sin(ga * i), z)))
    idx = sorted({int(np.argmax(hv @ (d / np.linalg.norm(d)))) for d in dirs})
    cand = hv[idx]
    if len(cand) <= kmax:
        return cand
    # farthest-point thinning, seeded with the six axis extremes
    keep = sorted({int(np.argmax(cand @ d)) for d in dirs[:6]})
    dist = np.min(np.linalg.norm(cand[:, None, :] - cand[keep][None, :, :], axis=2), axis=1)
    while len(keep) < kmax:
        j = int(np.argmax(dist))
        keep.append(j)
        dist = np.minimum(dist, np.linalg.norm(cand - cand[j], axis=1))
    return cand[sorted(keep)]


def mesh_volume_inertia(tris):
    """Volume, centre of mass and unit-density inertia tensor (about the centre of mass, mesh frame) of a closed triangle
    mesh [n, 3, 3] by signed tetrahedra against the origin (the exact integrals of a polyhedron)."""
    a, b, c = tris[:, 0], tris[:, 1], tris[:, 2]
    v6 = np.einsum("ij,ij->i", a, np.cross(b, c))          # 6 x signed volume of (0, a, b, c)
    vol = v6.sum() / 6.0
    if vol < 0:                                             # inward-facing winding
        v6, vol = -v6, -vol
    com = (v6[:, None] * (a + b + c)).sum(0) / (24.0 * vol)
    s = a + b + c
    S = (np.einsum("i,ij,ik->jk", v6, s, s) + np.einsum("i,ij,ik->jk", v6, a, a) + np.einsum("i,ij,ik->jk", v6, b, b) +
         np.einsum("i,ij,ik->jk", v6, c, c)) / 120.0       # integral of x x^T over the volume
    I0 = np.trace(S) * np.eye(3) - S                        # inertia about the origin
    Ic = I0 - vol * (com @ com * np.eye(3) - np.outer(com, com))
    return vol, com, Ic


def combine_inertias(parts):
    """parts: list of (mass, com[3], R[3,3] (frame->parent), diag[3]).  Returns mass, com, quat, diag."""
    mtot = sum(p[0] for p in parts)
    if mtot < MINVAL:
        return 0.0, np.zeros(3), np.array([1.0, 0, 0, 0]), np.zeros(3)
    com = sum(p[0] * p[1] for p in parts) / mtot
    I = np.zeros((3, 3))
    for m, c, R, d in parts:
        I += R @ np.diag(d) @ R.T
        r = c - com
        I += m * (r @ r * np.eye(3) - np.outer(r, r))
    w, V = np.linalg.eigh(I)
    order = np.argsort(-w)  # MuJoCo sorts principal inertias in decreasing order
    w, V = w[order], V[:, order]
    if np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    # if the tensor is already diagonal keep the identity frame (avoids arbitrary axis permutations)
    if np.allclose(I, np.diag(np.diag(I)), atol=1e-14 * max(1.0, np.abs(I).max())):
        return mtot, com, np.array([1.0, 0, 0, 0]), np.diag(I).copy()
    return mtot, com, mat2q(V), w


# --------------------------------------------------------------------------------------
# STL
def load_stl(path):
    d = open(path, "rb").read()
    n = struct.unpack("<I", d[80:84])[0]
    if 84 + 50 * n != len(d):  # ascii STL
        verts = []
        for line in d.decode("ascii", "ignore").splitlines():
            t = line.split()
            if len(t) == 4 and t[0] == "vertex":
                verts.append([float(x) for x in t[1:]])
        return np.array(verts, dtype=np.float64)
    a = np.frombuffer(d[84:84 + 50 * n], dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("a", "<u2")]))
    return a["v"].reshape(-1, 3).astype(np.float64)


# --------------------------------------------------------------------------------------
@dataclass
class Full:
    """Unfused, mjModel-like arrays (lists of per-element dicts kept simple on purpose)."""
    opt: dict = field(default_factory=dict)
    bodies: list = field(default_factory=list)
    joints: list = field(default_factory=list)
    geoms: list = field(default_factory=list)
    sites: list = field(default_factory=list)
    actuators: list = field(default_factory=list)
    equalities: list = field(default_factory=list)
    excludes: list = field(default_factory=list)
    pairs: list = field(default_factory=list)
    tendons: list = field(default_factory=list)
    sensors: list = field(default_factory=list)
    meshes: dict = field(default_factory=dict)


_DEFAULT_TAGS = ("geom", "joint", "site", "position", "motor", "general", "velocity", "mesh", "tendon", "equality",
                 "pair", "camera", "light", "material")


class _Parser:
    def __init__(self, path, overrides=None, root=None):
        self.path = os.path.abspath(path)
        self.dir = os.path.dirname(self.path)
        if root is not None:
            self.root = root
            self._expand_includes(self.root, self.dir)
        else:
            self.root = self._load(self.path)
        self.compiler = {"angle": "degree", "eulerseq": "xyz", "meshdir": "", "inertiafromgeom": "auto",
                         "autolimits": "true", "coordinate": "local"}
        self.defaults = {"main": {t: {} for t in _DEFAULT_TAGS}}
        self.default_parent = {"main": None}
        self.full = Full()
        self.overrides = overrides or {}
        # bodies removed before compilation (e.g. the Hand's decoupled, unobserved visual `target` free body)
        drop = set(self.overrides.get("drop_bodies", ()))
        if drop:
            for parent in list(self.root.iter()):
                for ch in list(parent):
                    if ch.tag == "body" and ch.get("name") in drop:
                        parent.remove(ch)

    # -- xml loading with <include>
    def _load(self, path):
        root = ET.parse(path).getroot()
        self._expand_includes(root, os.path.dirname(path))
        return root

    def _expand_includes(self, elem, base):
        i = 0
        while i < len(elem):
            ch = elem[i]
            if ch.tag == "include":
                inc = ET.parse(os.path.join(base, ch.get("file"))).getroot()
                self._expand_includes(inc, base)
                elem.remove(ch)
                for k, sub in enumerate(list(inc)):
                    elem.insert(i + k, sub)
                i += len(inc)
            else:
                self._expand_includes(ch, base)
                i += 1

    # -- defaults
    def _parse_defaults(self, elem, cls, parent):
        if cls not in self.defaults:
            self.defaults[cls] = {t: dict(self.defaults[parent][t]) for t in _DEFAULT_TAGS} if parent else \
                {t: {} for t in _DEFAULT_TAGS}
            self.default_parent[cls] = parent
        for ch in elem:
            if ch.tag == "default":
                self._parse_defaults(ch, ch.get("class"), cls)
            elif ch.tag in _DEFAULT_TAGS:
                self.defaults[cls][ch.tag].update(ch.attrib)

    def attrs(self, elem, childclass, tag=None):
        cls = elem.get("class") or childclass or "main"
        a = dict(self.defaults[cls][tag or elem.tag])
        a.update(elem.attrib)
        return a

    def angle(self, v):
        return np.deg2rad(v) if self.compiler["angle"] == "degree" else v

    def orient(self, a):
        if "quat" in a:
            return qnorm(floats(a["quat"]))
        if "euler" in a:
            return euler2q(self.angle(floats(a["euler"])), self.compiler["eulerseq"])
        if "axisangle" in a:
            v = floats(a["axisangle"])
            return axisangle2q(v[:3] / np.linalg.norm(v[:3]), self.angle(v[3]))
        if "zaxis" in a:
            return zaxis2q(floats(a["zaxis"]))
        if "xyaxes" in a:
            v = floats(a["xyaxes"])
            x = v[:3] / np.linalg.norm(v[:3])
            y = v[3:] - x * (x @ v[3:])
            y /= np.linalg.norm(y)
            return mat2q(np.stack([x, y, np.cross(x, y)], axis=1))
        return np.array([1.0, 0, 0, 0])

    # -- main
    def parse(self):
        r = self.root
        for c in r.findall("compiler"):
            self.compiler.update(c.attrib)
        opt = {"timestep": 0.002, "gravity": np.array([0, 0, -9.81]), "tolerance": 1e-8, "impratio": 1.0,
               "iterations": 100, "ls_iterations": 50, "ls_tolerance": 0.01, "noslip_iterations": 0,
               "integrator": INT_EULER, "cone": "pyramidal", "solver": "Newton", "warmstart": 1}
        for o in r.findall("option"):
            for k, v in o.attrib.items():
                if k == "gravity":
                    opt["gravity"] = floats(v)
                elif k == "integrator":
                    opt["integrator"] = {"Euler": INT_EULER, "RK4": INT_RK4}[v]
                elif k in ("iterations", "ls_iterations", "noslip_iterations"):
                    opt[k] = int(v)
                elif k in ("cone", "solver"):
                    opt[k] = v
                elif k in opt:
                    opt[k] = float(v)
            for f in o.findall("flag"):
                if f.get("warmstart") == "disable":
                    opt["warmstart"] = 0
        if opt["cone"] != "pyramidal" or opt["solver"] != "Newton":
            raise NotImplementedError("only pyramidal cones with the Newton solver are in scope")
        opt.update(self.overrides.get("opt", {}))
        self.full.opt = opt
        for d in r.findall("default"):
            self._parse_defaults(d, d.get("class") or "main", None if (d.get("class") in (None, "main")) else "main")
        for a in r.findall("asset"):
            for m in a.findall("mesh"):
                ma = self.attrs(m, None)
                if "vertex" in ma:     # MJCF: vertex coordinates given inline (the hull of the points is the mesh)
                    name = ma["name"]
                    v = floats(ma["vertex"]).reshape(-1, 3)
                else:
                    name = ma.get("name") or os.path.splitext(os.path.basename(ma["file"]))[0]
                    v = load_stl(os.path.join(self.dir, self.compiler["meshdir"], ma["file"]))
                v = v * floats(ma.get("scale"), 3, [1, 1, 1])
                self.full.meshes[name] = v
        # world body (id 0)
        self.full.bodies.append(dict(name="world", parent=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]),
                                     mocap=False, inertial=None, childclass=None))
        for wb in r.findall("worldbody"):
            self._parse_body_children(wb, 0, None)
        for act in r.findall("actuator"):
            for a in act:
                self._parse_actuator(a)
        for eq in r.findall("equality"):
            for e in eq:
                self._parse_equality(e)
        for c in r.findall("contact"):
            for e in c.findall("exclude"):
                self.full.excludes.append((e.get("body1"), e.get("body2")))
            for p in c.findall("pair"):
                self.full.pairs.append(self.attrs(p, None))
        for t in r.findall("tendon"):
            for f in t.findall("fixed"):
                a = self.attrs(f, None, "tendon")
                a["joints"] = [(j.get("joint"), float(j.get("coef"))) for j in f.findall("joint")]
                self.full.tendons.append(a)
            if t.findall("spatial"):
                raise NotImplementedError("spatial tendons are out of scope")
        for s in r.findall("sensor"):
            for e in s:
                d = dict(e.attrib)
                d["type"] = e.tag
                self.full.sensors.append(d)
        return self.full

    def _parse_body_children(self, elem, bid, childclass):
        F = self.full
        for ch in elem:
            if ch.tag == "body":
                cc = ch.get("childclass") or childclass
                nb = len(F.bodies)
                F.bodies.append(dict(name=ch.get("name") or f"body{nb}", parent=bid, pos=floats(ch.get("pos"), 3, [0, 0, 0]),
                                     quat=self.orient(ch.attrib), mocap=ch.get("mocap") == "true", inertial=None,
                                     childclass=cc))
                self._parse_body_children(ch, nb, cc)
            elif ch.tag == "inertial":
                a = ch.attrib
                if "fullinertia" in a:
                    f = floats(a["fullinertia"])
                    I = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
                    w, V = np.linalg.eigh(I)
                    if np.linalg.det(V) < 0:
                        V[:, 2] = -V[:, 2]
                    quat, diag = qmul(self.orient(a), mat2q(V)), w
                else:
                    quat, diag = self.orient(a), floats(a.get("diaginertia"), 3, [0, 0, 0])
                F.bodies[bid]["inertial"] = dict(pos=floats(a.get("pos"), 3, [0, 0, 0]), quat=quat,
                                                 mass=float(a.get("mass", 0)), diag=diag)
            elif ch.tag in ("joint", "freejoint"):
                a = self.attrs(ch, childclass, "joint") if ch.tag == "joint" else dict(ch.attrib, type="free")
                jt = {"free": JNT_FREE, "ball": JNT_BALL, "slide": JNT_SLIDE, "hinge": JNT_HINGE}[a.get("type", "hinge")]
                rng = floats(a.get("range"), 2, [0, 0])
                if jt == JNT_HINGE:
                    rng = self.angle(rng)
                lim = a.get("limited", "auto")
                limited = (lim == "true") or (lim == "auto" and self.compiler["autolimits"] == "true" and "range" in a)
                ref = float(a.get("ref", 0))
                sref = float(a.get("springref", 0))
                if jt == JNT_HINGE:
                    ref, sref = self.angle(ref), self.angle(sref)
                axis = floats(a.get("axis"), 3, [0, 0, 1])
                F.joints.append(dict(
                    name=a.get("name") or f"joint{len(F.joints)}", type=jt, body=bid, pos=floats(a.get("pos"), 3, [0, 0, 0]),
                    axis=axis / max(np.linalg.norm(axis), MINVAL), range=rng, limited=limited, ref=ref, springref=sref,
                    stiffness=float(a.get("stiffness", 0)), damping=float(a.get("damping", 0)),
                    armature=float(a.get("armature", 0)), frictionloss=float(a.get("frictionloss", 0)),
                    margin=float(a.get("margin", 0)),
                    solref=floats(a.get("solreflimit"), 2, [0.02, 1]), solimp=floats(a.get("solimplimit"), 5, [0.9, 0.95, 0.001, 0.5, 2]),
                    solref_fri=floats(a.get("solreffriction"), 2, [0.02, 1]),
                    solimp_fri=floats(a.get("solimpfriction"), 5, [0.9, 0.95, 0.001, 0.5, 2])))
            elif ch.tag == "geom":
                a = self.attrs(ch, childclass)
                F.geoms.append(self._make_geom(a, bid))
            elif ch.tag == "site":
                a = self.attrs(ch, childclass)
                F.sites.append(dict(name=a.get("name") or f"site{len(F.sites)}", body=bid, pos=floats(a.get("pos"), 3, [0, 0, 0]),
                                    quat=self.orient(a), size=floats(a.get("size"), 3, [0.005, 0.005, 0.005]),
                                    type=a.get("type", "sphere")))

    def _make_geom(self, a, bid):
        F = self.full
        gtype = GEOM_NAMES[a.get("type", "sphere")]
        size = floats(a.get("size"), 3, [0, 0, 0])
        pos = floats(a.get("pos"), 3, [0, 0, 0])
        quat = self.orient(a)
        if "fromto" in a:
            ft = floats(a["fromto"])
            p0, p1 = ft[:3], ft[3:]
            pos = 0.5 * (p0 + p1)
            quat = zaxis2q(p1 - p0)
            size = np.array([size[0], 0.5 * np.linalg.norm(p1 - p0), 0.0])
        mesh = a.get("mesh")
        g = dict(name=a.get("name") or f"geom{len(F.geoms)}", type=gtype, body=bid, pos=pos, quat=quat, size=size,
                 contype=int(a.get("contype", 1)), conaffinity=int(a.get("conaffinity", 1)), condim=int(a.get("condim", 3)),
                 friction=floats(a.get("friction"), 3, [1, 0.005, 0.0001]), margin=float(a.get("margin", 0)),
                 gap=float(a.get("gap", 0)), solref=floats(a.get("solref"), 2, [0.02, 1]),
                 solimp=floats(a.get("solimp"), 5, [0.9, 0.95, 0.001, 0.5, 2]), solmix=float(a.get("solmix", 1)),
                 priority=int(a.get("priority", 0)), mass=(float(a["mass"]) if "mass" in a else None),
                 density=float(a.get("density", 1000)), mesh=mesh, group=int(a.get("group", 0)))
        if gtype == GEOM_MESH:
            # mesh proxy: oriented bounding box of the vertices in the mesh frame (DESIGN.md)
            v = F.meshes[mesh]
            lo, hi = v.min(0), v.max(0)
            g["mesh_center"] = 0.5 * (lo + hi)
            g["mesh_half"] = 0.5 * (hi - lo)
        return g

    def _parse_actuator(self, e):
        a = self.attrs(e, None)
        kind = e.tag
        gain = np.array([1.0, 0, 0])
        bias = np.zeros(3)
        biastype = 0
        if kind == "position":
            kp = float(a.get("kp", 1))
            gain = np.array([kp, 0, 0])
            bias = np.array([0, -kp, -float(a.get("kv", 0))])
            biastype = 1
        elif kind == "velocity":
            kv = float(a.get("kv", 1))
            gain = np.array([kv, 0, 0])
            bias = np.array([0, 0, -kv])
            biastype = 1
        elif kind == "general":
            gain = floats(a.get("gainprm"), 3, [1, 0, 0])[:3]
            bias = floats(a.get("biasprm"), 3, [0, 0, 0])[:3]
            biastype = {"none": 0, "affine": 1}[a.get("biastype", "none")]
            if a.get("dyntype", "none") != "none" or a.get("gaintype", "fixed") != "fixed":
                raise NotImplementedError("stateful actuators are out of scope")
        elif kind != "motor":
            raise NotImplementedError(f"actuator <{kind}>")
        if "joint" not in a:
            raise NotImplementedError("only joint transmissions are in scope")
        cl = a.get("ctrllimited", "auto")
        fl = a.get("forcelimited", "auto")
        auto = self.compiler["autolimits"] == "true"
        self.full.actuators.append(dict(
            name=a.get("name") or f"actuator{len(self.full.actuators)}", joint=a["joint"], gear=floats(a.get("gear"), 1, [1])[0],
            gainprm=gain, biasprm=bias, biastype=biastype,
            ctrllimited=(cl == "true") or (cl == "auto" and auto and "ctrlrange" in a),
            ctrlrange=floats(a.get("ctrlrange"), 2, [0, 0]),
            forcelimited=(fl == "true") or (fl == "auto" and auto and "forcerange" in a),
            forcerange=floats(a.get("forcerange"), 2, [0, 0])))

    def _parse_equality(self, e):
        a = self.attrs(e, None, "equality")
        a.update(e.attrib)
        d = dict(kind=e.tag, active=a.get("active", "true") == "true", solref=floats(a.get("solref"), 2, [0.02, 1]),
                 solimp=floats(a.get("solimp"), 5, [0.9, 0.95, 0.001, 0.5, 2]), attrs=a)
        if e.tag not in ("weld", "joint", "connect"):
            raise NotImplementedError(f"equality <{e.tag}>")
        self.full.equalities.append(d)


# --------------------------------------------------------------------------------------
class Model:
    """Runtime (fused) model as flat numpy arrays + name tables."""

    INT_FIELDS = ["sizes", "opt_int", "body_parent", "body_jntadr", "body_jntnum", "body_dofadr", "body_dofnum",
                  "body_mocapid", "body_rootid", "jnt_type", "jnt_body", "jnt_qposadr", "jnt_dofadr", "jnt_limited",
                  "dof_body", "dof_jnt", "dof_parent", "geom_type", "geom_body", "pair_geom1", "pair_geom2", "pair_condim",
                  "site_body", "act_trnid", "act_ctrllimited", "act_forcelimited", "eq_type", "eq_obj1", "eq_obj2",
                  "eq_active", "mocap_body", "ten_adr", "ten_num", "ten_limited", "wrap_dof", "sensor_site", "sensor_body", "sensor_type",
                  "pair_grid", "grid_dims", "grid_walls", "geom_mjbody", "mjbody_rt", "geom_hull"]
    FLT_FIELDS = ["opt", "body_pos", "body_quat", "body_ipos", "body_iquat", "body_mass", "body_inertia", "jnt_pos",
                  "jnt_axis", "jnt_range", "jnt_margin", "jnt_stiffness", "jnt_solref", "jnt_solimp", "qpos0",
                  "qpos_spring", "dof_armature", "dof_damping", "dof_frictionloss", "dof_invweight0", "dof_solref_fri",
                  "dof_solimp_fri", "geom_pos", "geom_quat",
                  "geom_size", "geom_rbound", "pair_friction", "pair_margin", "pair_gap", "pair_solref", "pair_solimp",
                  "pair_invweight", "site_pos", "site_quat", "act_gear", "act_gainprm", "act_biasprm", "act_ctrlrange",
                  "act_forcerange", "eq_data", "eq_solref", "eq_solimp", "eq_invweight", "ten_range", "ten_margin",
                  "ten_solref", "ten_solimp", "ten_invweight0", "wrap_coef", "sensor_size", "key_qpos", "grid_param", "hull_vert"]
    # written only when non-empty, read as empty when absent: blobs of models without such data are byte-identical to older ones
    OPTIONAL_FIELDS = ("geom_hull", "hull_vert")

    def __init__(self):
        self.names = {}

    # sizes layout (keep in sync with include/b200sim_model.h)
    SIZES = ["nbody", "njnt", "nq", "nv", "nu", "ngeom", "nsite", "nmocap", "neq", "npair", "ntendon", "nwrap",
             "nsensor", "nM"]

    def __getattr__(self, k):
        if k in Model.SIZES:
            return int(self.sizes[Model.SIZES.index(k)])
        raise AttributeError(k)

    def to_blob(self) -> bytes:
        entries, payload = [], b""
        for name in self.INT_FIELDS:
            arr = np.ascontiguousarray(getattr(self, name), dtype=np.int32).ravel()
            if name in self.OPTIONAL_FIELDS and arr.size == 0:
                continue
            entries.append((name, 0, arr.size, len(payload)))
            payload += arr.tobytes()
            payload += b"\0" * ((-len(payload)) % 8)
        for name in self.FLT_FIELDS:
            arr = np.ascontiguousarray(getattr(self, name), dtype=np.float64).ravel()
            if name in self.OPTIONAL_FIELDS and arr.size == 0:
                continue
            entries.append((name, 1, arr.size, len(payload)))
            payload += arr.tobytes()
        meta = json.dumps(self.names).encode()
        entries.append(("names_json", 2, len(meta), len(payload)))
        payload += meta + b"\0" * ((-len(meta)) % 8)
        head = struct.pack("<IIII", BLOB_MAGIC, BLOB_VERSION, len(entries), 0)
        table = b"".join(struct.pack("<32sIIQ", n.encode(), t, c, o) for n, t, c, o in entries)
        return head + table + payload

    @staticmethod
    def from_blob(blob: bytes) -> "Model":
        magic, ver, n, _ = struct.unpack_from("<IIII", blob, 0)
        if magic != BLOB_MAGIC or ver != BLOB_VERSION:
            raise ValueError("not a b200sim model blob (magic/version mismatch)")
        m = Model()
        base = 16 + 48 * n
        for i in range(n):
            name, t, c, o = struct.unpack_from("<32sIIQ", blob, 16 + 48 * i)
            name = name.rstrip(b"\0").decode()
            if t == 0:
                setattr(m, name, np.frombuffer(blob, dtype=np.int32, count=c, offset=base + o).copy())
            elif t == 1:
                setattr(m, name, np.frombuffer(blob, dtype=np.float64, count=c, offset=base + o).copy())
            else:
                m.names = json.loads(blob[base + o: base + o + c].decode())
        for name in Model.INT_FIELDS:    # blobs written before a field existed: the field reads as empty
            if name not in m.__dict__:
                setattr(m, name, np.zeros(0, dtype=np.int32))
        for name in Model.OPTIONAL_FIELDS:
            if name not in m.__dict__:
                setattr(m, name, np.zeros(0, dtype=np.float64 if name in Model.FLT_FIELDS else np.int32))
        m._reshape()
        return m

    _SHAPES = {"body_pos": 3, "body_quat": 4, "body_ipos": 3, "body_iquat": 4, "body_inertia": 3, "jnt_pos": 3,
               "jnt_axis": 3, "jnt_range": 2, "jnt_solref": 2, "jnt_solimp": 5, "dof_solref_fri": 2, "dof_solimp_fri": 5,
               "geom_pos": 3, "geom_quat": 4, "geom_size": 3,
               "pair_friction": 5, "pair_solref": 2, "pair_solimp": 5, "pair_invweight": 2, "site_pos": 3, "site_quat": 4,
               "act_gainprm": 3, "act_biasprm": 3, "act_ctrlrange": 2, "act_forcerange": 2, "eq_data": 11, "eq_solref": 2,
               "eq_solimp": 5, "eq_invweight": 2, "ten_range": 2, "ten_solref": 2, "ten_solimp": 5, "sensor_size": 3, "hull_vert": 3}

    def _reshape(self):
        for k, w in self._SHAPES.items():
            setattr(self, k, np.asarray(getattr(self, k), dtype=np.float64).reshape(-1, w))

    # name helpers --------------------------------------------------------------
    def joint_id(self, name):
        return self.names["joint"].index(name)

    def site_id(self, name):
        return self.names["site"].index(name)

    def body_id(self, name):
        """Runtime body id that carries the MJCF body ``name`` (after fusing)."""
        return self.names["body_map"][name]

    def frame_site(self, body_name):
        """Site id of the synthetic site that tracks the frame of MJCF body ``body_name``."""
        return self.names["site"].index("bodyframe:" + body_name)


# --------------------------------------------------------------------------------------
def _kin_tree(nbody, parent, bpos, bquat, ipos, iquat, joints, body_jnts, qpos):
    """Forward kinematics for the compile-time computations. Returns xpos, xmat, xipos, ximat, jnt anchors/axes."""
    xpos = np.zeros((nbody, 3))
    xquat = np.zeros((nbody, 4))
    xquat[0, 0] = 1
    xanchor, xaxis = {}, {}
    for b in range(1, nbody):
        p = parent[b]
        jl = body_jnts[b]
        if len(jl) == 1 and joints[jl[0]]["type"] == JNT_FREE:
            a = joints[jl[0]]["qposadr"]
            xpos[b] = qpos[a:a + 3]
            xquat[b] = qnorm(qpos[a + 3:a + 7])
            xanchor[jl[0]], xaxis[jl[0]] = xpos[b].copy(), np.array([0, 0, 1.0])
            continue
        xpos[b] = xpos[p] + qrot(xquat[p], bpos[b])
        xquat[b] = qmul(xquat[p], bquat[b])
        for j in jl:
            J = joints[j]
            anchor = xpos[b] + qrot(xquat[b], J["pos"])
            axis = qrot(xquat[b], J["axis"])
            dq = qpos[J["qposadr"]] - J["ref"]
            if J["type"] == JNT_SLIDE:
                xpos[b] = xpos[b] + axis * dq
            elif J["type"] == JNT_HINGE:
                r = axisangle2q(axis, dq)
                xquat[b] = qmul(r, xquat[b])
                xpos[b] = anchor - qrot(xquat[b], J["pos"])
            else:
                raise NotImplementedError("ball joints are out of scope")
            xanchor[j], xaxis[j] = anchor, axis
    xmat = np.array([q2mat(q) for q in xquat])
    xipos = np.array([xpos[b] + xmat[b] @ ipos[b] for b in range(nbody)])
    ximat = np.array([q2mat(qmul(xquat[b], iquat[b])) for b in range(nbody)])
    return xpos, xquat, xmat, xipos, ximat, xanchor, xaxis


def _dense_mass_matrix(nbody, nv, parent, mass, inertia, xipos, ximat, xmat, joints, body_jnts, xanchor, xaxis, armature):
    """M = sum_b Jb^T diag(m, I) Jb from body-com Jacobians (plain definition; compile-time only)."""
    # ancestors' dofs per body
    jacs = []
    M = np.zeros((nv, nv))
    anc = [[] for _ in range(nbody)]
    for b in range(1, nbody):
        anc[b] = list(anc[parent[b]])
        for j in body_jnts[b]:
            anc[b].append(j)
    for b in range(nbody):
        Jp = np.zeros((3, nv))
        Jr = np.zeros((3, nv))
        for j in anc[b]:
            J = joints[j]
            d = J["dofadr"]
            if J["type"] == JNT_FREE:
                Jp[:, d:d + 3] = np.eye(3)
                # rotational dofs of a free joint are expressed in the body frame
                Rm = xmat[J["body"]]
                for k in range(3):
                    ax = Rm[:, k]
                    Jr[:, d + 3 + k] = ax
                    Jp[:, d + 3 + k] = np.cross(ax, xipos[b] - xanchor[j])
            elif J["type"] == JNT_SLIDE:
                Jp[:, d] = xaxis[j]
            else:
                Jr[:, d] = xaxis[j]
                Jp[:, d] = np.cross(xaxis[j], xipos[b] - xanchor[j])
        jacs.append((Jp, Jr))
        if mass[b] > 0 or np.any(inertia[b] > 0):
            Iw = ximat[b] @ np.diag(inertia[b]) @ ximat[b].T
            M += mass[b] * Jp.T @ Jp + Jr.T @ Iw @ Jr
    M += np.diag(armature)
    return M, jacs


def maze_walls(maze_map, maze_size_scaling, maze_height):
    """The geometry part of `Maze.make_maze` (gymnasium_robotics/envs/maze/maze_v4.py:148-242): one static box per wall cell,
    as (name, centre, half extents) in row-major order on a grid centred at the origin, and the wall grid of the step kernel's
    wall lookup."""
    length, width = len(maze_map), len(maze_map[0])
    xc, yc = width / 2 * maze_size_scaling, length / 2 * maze_size_scaling
    half = (0.5 * maze_size_scaling, 0.5 * maze_size_scaling, maze_height / 2 * maze_size_scaling)
    walls = [(f"block_{i}_{j}", ((j + 0.5) * maze_size_scaling - xc, yc - (i + 0.5) * maze_size_scaling, half[2]), half)
             for i in range(length) for j in range(width) if maze_map[i][j] == 1]
    grid = dict(length=length, width=width, scaling=float(maze_size_scaling), height=float(maze_height),
                walls=[[1 if maze_map[i][j] == 1 else 0 for j in range(width)] for i in range(length)])
    return walls, grid


def make_maze_xml(agent_xml_path, maze_map, maze_size_scaling, maze_height):
    """MJCF tree of an agent placed in a maze: the agent's MJCF, the wall boxes of `maze_walls` and the target site."""
    tree = ET.parse(agent_xml_path)
    root = tree.getroot()
    worldbody = root.find(".//worldbody")
    walls, grid = maze_walls(maze_map, maze_size_scaling, maze_height)
    for name, pos, size in walls:
        ET.SubElement(worldbody, "geom", name=name, pos=" ".join(map(str, pos)), size=" ".join(map(str, size)),
                      type="box", contype="1", conaffinity="1")
    ET.SubElement(worldbody, "site", name="target", pos=f"0 0 {maze_height / 2 * maze_size_scaling}",
                  size=f"{0.2 * maze_size_scaling}", type="sphere")
    return root, grid


def _grid_tables(grid, pair_geom2_names):
    """pair_grid, grid_dims, grid_walls, grid_param: a pair whose second geom is a maze wall block is served by the step
    kernel's grid lookup instead of the pair list."""
    pair_grid = np.array([1 if (grid is not None and n.startswith("block_")) else 0 for n in pair_geom2_names], dtype=np.int32)
    if grid is None:
        return pair_grid, np.zeros(2, dtype=np.int32), np.zeros(0, dtype=np.int32), np.zeros(4)
    return (pair_grid, np.array([grid["length"], grid["width"]], dtype=np.int32), np.array(grid["walls"], dtype=np.int32).ravel(),
            np.array([grid["scaling"], grid["height"], grid["width"] / 2 * grid["scaling"], grid["length"] / 2 * grid["scaling"]]))


def _geom_rbound(typ, size, hull=None):
    """Bounding-sphere radius of a runtime geom about its centre."""
    return {GEOM_PLANE: 0.0, GEOM_SPHERE: size[0], GEOM_CAPSULE: size[0] + size[1], GEOM_CYLINDER: np.hypot(size[0], size[1]),
            GEOM_BOX: np.linalg.norm(size), GEOM_ELLIPSOID: max(size),
            GEOM_MESH: (float(np.linalg.norm(hull, axis=1).max()) if hull is not None else 0.0)}[typ]


def replace_maze_walls(model, maze_map, maze_size_scaling, maze_height) -> "Model":
    """The compiled agent-in-a-maze `model` with its walls replaced by those of `maze_map`: the model `compile_mjcf` makes of
    `make_maze_xml` on that map, without the agent's MJCF.

    All wall blocks are world geoms with the same attributes, so the model's own wall pairs give each agent geom's contact
    parameters against any wall.  compile_mjcf lists the wall blocks last (they are the last geoms of the MJCF) and the
    dynamic pairs in the order of its candidate loop, by (lower geom index, higher geom index); the new pair list keeps that
    order.  The target site does not depend on the layout and stays."""
    m = Model.from_blob(model.to_blob())
    names = m.names["geom"]
    wall = np.array([n.startswith("block_") for n in names], dtype=bool)
    na = len(names) - int(wall.sum())
    if not wall.any() or wall[:na].any() or m.geom_hull.size:
        raise ValueError("not a compiled maze model: its wall blocks must be its last geoms")
    if not np.array_equal(m.site_pos[m.site_id("target")], [0.0, 0.0, maze_height / 2 * maze_size_scaling]):
        raise ValueError("the model's maze has another scaling or height")
    keys = [(min(a, b), max(a, b)) for a, b in zip(m.pair_geom1.tolist(), m.pair_geom2.tolist())]
    if keys != sorted(keys):
        raise ValueError("the model has explicit contact pairs: its wall pairs cannot be rebuilt")
    walls, grid = maze_walls(maze_map, maze_size_scaling, maze_height)
    rows, template = [], {}    # rows: (lower geom, higher geom, geom1, geom2, pair row that carries the parameters)
    for k, (a, b) in enumerate(zip(m.pair_geom1.tolist(), m.pair_geom2.tolist())):
        if wall[a] or wall[b]:
            template.setdefault(b if wall[a] else a, (k, bool(wall[a])))
        else:
            rows.append((*keys[k], a, b, k))
    for a, (k, wall_first) in template.items():
        for w in range(na, na + len(walls)):
            rows.append((a, w, w, a, k) if wall_first else (a, w, a, w, k))
    rows.sort()
    src = np.array([r[4] for r in rows], dtype=np.int64)
    m.pair_geom1, m.pair_geom2 = np.array([r[2] for r in rows], dtype=np.int32), np.array([r[3] for r in rows], dtype=np.int32)
    for f in ("pair_condim", "pair_friction", "pair_margin", "pair_gap", "pair_solref", "pair_solimp", "pair_invweight"):
        setattr(m, f, getattr(m, f)[src])
    nw = len(walls)
    m.geom_type = np.concatenate([m.geom_type[:na], np.full(nw, GEOM_BOX, dtype=np.int32)])
    m.geom_body = np.concatenate([m.geom_body[:na], np.zeros(nw, dtype=np.int32)])
    m.geom_mjbody = np.concatenate([m.geom_mjbody[:na], np.zeros(nw, dtype=np.int32)])
    m.geom_pos = np.concatenate([m.geom_pos[:na], np.array([p for _, p, _ in walls]).reshape(-1, 3)])
    m.geom_quat = np.concatenate([m.geom_quat[:na], np.tile([1.0, 0, 0, 0], (nw, 1))])
    m.geom_size = np.concatenate([m.geom_size[:na], np.array([s for _, _, s in walls]).reshape(-1, 3)])
    m.geom_rbound = np.concatenate([m.geom_rbound[:na], [_geom_rbound(GEOM_BOX, np.array(s)) for _, _, s in walls]])
    m.names["geom"] = names[:na] + [n for n, _, _ in walls]
    m.pair_grid, m.grid_dims, m.grid_walls, m.grid_param = _grid_tables(grid, [m.names["geom"][g] for g in m.pair_geom2])
    m.sizes[Model.SIZES.index("ngeom")], m.sizes[Model.SIZES.index("npair")] = na + nw, len(rows)
    m._reshape()
    return m


def compile_mjcf(path, overrides=None, mesh_mesh=False, root=None, grid=None, mesh_hull=False) -> Model:
    """Compile an MJCF file to the runtime :class:`Model`.

    ``overrides`` may carry ``{"opt": {...}, "actuator_gainprm": {name: [...]}, ...}`` for
    constructor-time edits the reference performs on the loaded model.  ``mesh_hull``: mesh geoms keep the type MESH and carry a
    reduced convex-hull vertex table (`hull_vertices`) for a support-map narrow phase instead of becoming box proxies.
    """
    P = _Parser(path, overrides, root=root)
    F = P.parse()
    nb = len(F.bodies)
    name2body = {b["name"]: i for i, b in enumerate(F.bodies)}
    parent = [b["parent"] for b in F.bodies]
    body_jnts = [[] for _ in range(nb)]
    nq = nv = 0
    for j, J in enumerate(F.joints):
        body_jnts[J["body"]].append(j)
        J["qposadr"], J["dofadr"] = nq, nv
        nq += 7 if J["type"] == JNT_FREE else 1
        nv += 6 if J["type"] == JNT_FREE else 1
    # body inertial properties
    ipos, iquat, mass, inertia = np.zeros((nb, 3)), np.tile([1.0, 0, 0, 0], (nb, 1)), np.zeros(nb), np.zeros((nb, 3))
    for b, B in enumerate(F.bodies):
        if B["inertial"] is not None and P.compiler["inertiafromgeom"] != "true":
            I = B["inertial"]
            ipos[b], iquat[b], mass[b], inertia[b] = I["pos"], I["quat"], I["mass"], I["diag"]
        elif b > 0:
            parts = []
            for g in F.geoms:
                if g["body"] != b or g["type"] in (GEOM_PLANE, GEOM_HFIELD):
                    continue
                if g["type"] == GEOM_MESH:
                    # mass properties of the triangle mesh itself (the Franka links of the kitchen model carry `mass=` on
                    # their collision meshes and no <inertial>); visual meshes with mass="0" contribute nothing
                    if g["mass"] is not None and g["mass"] <= 0:
                        continue
                    vol, cm, Ic = mesh_volume_inertia(F.meshes[g["mesh"]].reshape(-1, 3, 3))
                    if vol < MINVAL:
                        continue
                    m = g["mass"] if g["mass"] is not None else g["density"] * vol
                    w, V = np.linalg.eigh(Ic)
                    if np.linalg.det(V) < 0:
                        V[:, 2] = -V[:, 2]
                    Rg = q2mat(g["quat"])
                    parts.append((m, g["pos"] + Rg @ cm, Rg @ V, w * (m / vol)))
                    continue
                vol, Iu = geom_volume_inertia(g["type"], g["size"])
                m = g["mass"] if g["mass"] is not None else g["density"] * vol
                parts.append((m, g["pos"], q2mat(g["quat"]), Iu * (m / vol)))
            if parts:
                mass[b], ipos[b], iquat[b], inertia[b] = combine_inertias(parts)
    bpos = np.array([B["pos"] for B in F.bodies])
    bquat = np.array([B["quat"] for B in F.bodies])
    # qpos0
    qpos0 = np.zeros(nq)
    qspring = np.zeros(nq)
    for J in F.joints:
        a = J["qposadr"]
        if J["type"] == JNT_FREE:
            b = J["body"]
            assert parent[b] == 0, "free joints must be children of the world"
            qpos0[a:a + 3], qpos0[a + 3:a + 7] = bpos[b], bquat[b]
            qspring[a:a + 7] = qpos0[a:a + 7]
        else:
            qpos0[a], qspring[a] = J["ref"], J["springref"]
    xpos, xquat, xmat, xipos, ximat, xanchor, xaxis = _kin_tree(nb, parent, bpos, bquat, ipos, iquat, F.joints, body_jnts, qpos0)
    arm = np.zeros(nv)
    damp = np.zeros(nv)
    fl = np.zeros(nv)
    dof_jnt = np.zeros(nv, dtype=int)
    for j, J in enumerate(F.joints):
        n = 6 if J["type"] == JNT_FREE else 1
        arm[J["dofadr"]:J["dofadr"] + n] = J["armature"]
        damp[J["dofadr"]:J["dofadr"] + n] = J["damping"]
        fl[J["dofadr"]:J["dofadr"] + n] = J["frictionloss"]
        dof_jnt[J["dofadr"]:J["dofadr"] + n] = j
    M0, jacs = _dense_mass_matrix(nb, nv, parent, mass, inertia, xipos, ximat, xmat, F.joints, body_jnts, xanchor, xaxis, arm)
    Minv = np.linalg.inv(M0) if nv else np.zeros((0, 0))
    dof_invw = np.diag(Minv).copy() if nv else np.zeros(0)
    for J in F.joints:
        if J["type"] == JNT_FREE:
            d = J["dofadr"]
            dof_invw[d:d + 3] = dof_invw[d:d + 3].mean()
            dof_invw[d + 3:d + 6] = dof_invw[d + 3:d + 6].mean()
    # weld ids (body welded to its parent when it has no joints)
    weld = list(range(nb))
    for b in range(1, nb):
        if not body_jnts[b]:
            weld[b] = weld[parent[b]]
    body_invw = np.zeros((nb, 2))
    for b in range(1, nb):
        if weld[b] == 0:
            continue
        Jp, Jr = jacs[b]
        A = np.vstack([Jp, Jr]) @ Minv @ np.vstack([Jp, Jr]).T
        body_invw[b] = [max(MINVAL, np.trace(A[:3, :3]) / 3), max(MINVAL, np.trace(A[3:, 3:]) / 3)]
    meaninertia = float(np.mean(np.diag(M0))) if nv else 1.0

    # ---------------------------------------------------------------- fusing
    # runtime body = weld group, except mocap bodies which stay separate bodies (children of world)
    # `keep_bodies` (override): jointless bodies that stay runtime bodies because an env rewrites their body_pos per episode
    keep_names = set((overrides or {}).get("keep_bodies", ()))
    keep = [b for b in range(nb) if b == 0 or body_jnts[b] or F.bodies[b]["mocap"] or F.bodies[b]["name"] in keep_names]
    rt_of = {}
    for b in range(nb):
        a = b
        while a not in keep:
            a = parent[a]
        rt_of[b] = keep.index(a)
    # pose of every MJCF body relative to its runtime body (constant)
    rel_pos, rel_quat = np.zeros((nb, 3)), np.tile([1.0, 0, 0, 0], (nb, 1))
    for b in range(nb):
        if b in keep:
            continue
        p = parent[b]
        rel_pos[b] = rel_pos[p] + qrot(rel_quat[p], bpos[b])
        rel_quat[b] = qmul(rel_quat[p], bquat[b])
    m = Model()
    nrb = len(keep)
    m.body_parent = np.array([rt_of[parent[b]] for b in keep], dtype=np.int32)
    m.body_pos = np.array([rel_pos[parent[b]] + qrot(rel_quat[parent[b]], bpos[b]) if b else np.zeros(3) for b in keep])
    m.body_quat = np.array([qmul(rel_quat[parent[b]], bquat[b]) if b else [1.0, 0, 0, 0] for b in keep])
    m.body_mocapid = np.full(nrb, -1, dtype=np.int32)
    mocap_body = []
    for i, b in enumerate(keep):
        if F.bodies[b]["mocap"]:
            m.body_mocapid[i] = len(mocap_body)
            mocap_body.append(i)
    m.mocap_body = np.array(mocap_body, dtype=np.int32)
    m.body_mass, m.body_ipos, m.body_iquat, m.body_inertia = np.zeros(nrb), np.zeros((nrb, 3)), np.zeros((nrb, 4)), np.zeros((nrb, 3))
    for i, k in enumerate(keep):
        parts = [(mass[b], rel_pos[b] + qrot(rel_quat[b], ipos[b]), q2mat(qmul(rel_quat[b], iquat[b])), inertia[b])
                 for b in range(nb) if rt_of[b] == i and (mass[b] > 0 or np.any(inertia[b] > 0))]
        if i == 0:
            parts = []  # world inertia is irrelevant
        if len(parts) == 1:
            mm, c, R, d = parts[0]
            m.body_mass[i], m.body_ipos[i], m.body_iquat[i], m.body_inertia[i] = mm, c, mat2q(R), d
        else:
            m.body_mass[i], m.body_ipos[i], m.body_iquat[i], m.body_inertia[i] = combine_inertias(parts)
    # joints / dofs
    m.jnt_type = np.array([J["type"] for J in F.joints], dtype=np.int32)
    m.jnt_body = np.array([rt_of[J["body"]] for J in F.joints], dtype=np.int32)
    m.jnt_qposadr = np.array([J["qposadr"] for J in F.joints], dtype=np.int32)
    m.jnt_dofadr = np.array([J["dofadr"] for J in F.joints], dtype=np.int32)
    m.jnt_limited = np.array([int(J["limited"]) for J in F.joints], dtype=np.int32)
    m.jnt_pos = np.array([J["pos"] for J in F.joints]).reshape(-1, 3)
    m.jnt_axis = np.array([J["axis"] for J in F.joints]).reshape(-1, 3)
    m.jnt_range = np.array([J["range"] for J in F.joints]).reshape(-1, 2)
    m.jnt_margin = np.array([J["margin"] for J in F.joints])
    m.jnt_stiffness = np.array([J["stiffness"] for J in F.joints])
    m.jnt_solref = np.array([J["solref"] for J in F.joints]).reshape(-1, 2)
    m.jnt_solimp = np.array([J["solimp"] for J in F.joints]).reshape(-1, 5)
    m.qpos0, m.qpos_spring = qpos0, qspring
    m.body_jntadr = np.full(nrb, -1, dtype=np.int32)
    m.body_jntnum = np.zeros(nrb, dtype=np.int32)
    m.body_dofadr = np.full(nrb, -1, dtype=np.int32)
    m.body_dofnum = np.zeros(nrb, dtype=np.int32)
    for j, J in enumerate(F.joints):
        rb = rt_of[J["body"]]
        if m.body_jntnum[rb] == 0:
            m.body_jntadr[rb], m.body_dofadr[rb] = j, J["dofadr"]
        m.body_jntnum[rb] += 1
        m.body_dofnum[rb] += 6 if J["type"] == JNT_FREE else 1
    m.dof_jnt = dof_jnt.astype(np.int32)
    m.dof_body = m.jnt_body[dof_jnt].astype(np.int32) if nv else np.zeros(0, dtype=np.int32)
    m.dof_parent = np.full(nv, -1, dtype=np.int32)
    for d in range(nv):
        rb = m.dof_body[d]
        if d > m.body_dofadr[rb]:
            m.dof_parent[d] = d - 1
        else:
            p = m.body_parent[rb]
            while p > 0 and m.body_dofnum[p] == 0:
                p = m.body_parent[p]
            m.dof_parent[d] = (m.body_dofadr[p] + m.body_dofnum[p] - 1) if p > 0 else -1
    m.dof_armature, m.dof_damping, m.dof_frictionloss, m.dof_invweight0 = arm, damp, fl, dof_invw
    m.dof_solref_fri = np.array([F.joints[j]["solref_fri"] for j in dof_jnt]).reshape(-1, 2)
    m.dof_solimp_fri = np.array([F.joints[j]["solimp_fri"] for j in dof_jnt]).reshape(-1, 5)
    m.body_rootid = np.zeros(nrb, dtype=np.int32)
    for i in range(1, nrb):
        m.body_rootid[i] = i if m.body_parent[i] == 0 else m.body_rootid[m.body_parent[i]]
    nM = 0
    for d in range(nv):
        k = d
        while k >= 0:
            nM += 1
            k = m.dof_parent[k]

    # geoms (only those that can collide are kept at runtime)
    def geom_can_collide(g):
        return g["contype"] != 0 or g["conaffinity"] != 0

    pair_geoms = set()
    for pr in F.pairs:
        pair_geoms.update([pr["geom1"], pr["geom2"]])
    gkeep = [i for i, g in enumerate(F.geoms) if geom_can_collide(g) or g["name"] in pair_geoms]
    gidx = {g: i for i, g in enumerate(gkeep)}
    gt, gb, gp, gq, gs, gr = [], [], [], [], [], []
    ghull, hverts = [], []
    for gi in gkeep:
        g = F.geoms[gi]
        b = g["body"]
        pos, quat, size, typ = g["pos"], g["quat"], g["size"], g["type"]
        hull = None
        if typ == GEOM_MESH:
            pos = pos + qrot(quat, g["mesh_center"])
            size = g["mesh_half"]
            if mesh_hull:
                # support-map narrow phase: hull vertices in the geom frame (= mesh frame re-centred on the bounding box); the box
                # half extents stay in geom_size as the bounding volume of the broad phase
                hull = hull_vertices(F.meshes[g["mesh"]].reshape(-1, 3) - g["mesh_center"])
            else:
                typ = GEOM_BOX
        ghull.append((len(hverts), 0 if hull is None else len(hull)))
        if hull is not None:
            hverts.extend(hull.tolist())
        gt.append(typ)
        gb.append(rt_of[b])
        gp.append(rel_pos[b] + qrot(rel_quat[b], pos))
        gq.append(qmul(rel_quat[b], quat))
        gs.append(size)
        gr.append(_geom_rbound(typ, size, hull))
    m.geom_type, m.geom_body = np.array(gt, dtype=np.int32), np.array(gb, dtype=np.int32)
    if hverts:     # optional blob fields (absent from models without hull geoms: their blobs do not change)
        m.geom_hull, m.hull_vert = np.array(ghull, dtype=np.int32).reshape(-1, 2), np.array(hverts, dtype=np.float64).reshape(-1, 3)
    else:
        m.geom_hull, m.hull_vert = np.zeros((0, 2), dtype=np.int32), np.zeros((0, 3))
    # the MJCF (unfused) body of every runtime geom and the runtime body every MJCF body was fused into: per-MJCF-body quantities
    # such as data.cfrc_ext (one row per mjModel body; Ant-v5's contact-force observation) keep the reference's row layout
    m.geom_mjbody = np.array([F.geoms[gi]["body"] for gi in gkeep], dtype=np.int32)
    m.mjbody_rt = np.array([rt_of[b] for b in range(nb)], dtype=np.int32)
    m.geom_pos, m.geom_quat, m.geom_size = np.array(gp).reshape(-1, 3), np.array(gq).reshape(-1, 4), np.array(gs).reshape(-1, 3)
    m.geom_rbound = np.array(gr)

    # candidate pairs with MuJoCo's static filters, parameters pre-mixed
    excl = {(name2body[a], name2body[b]) for a, b in F.excludes} | {(name2body[b], name2body[a]) for a, b in F.excludes}
    P1, P2, PC, PF, PM, PG, PSR, PSI, PIW = [], [], [], [], [], [], [], [], []

    def add_pair(i1, i2, condim, fri5, margin, gap, solref, solimp):
        g1, g2 = F.geoms[i1], F.geoms[i2]
        t1, t2 = m.geom_type[gidx[i1]], m.geom_type[gidx[i2]]
        if t1 > t2:
            i1, i2, g1, g2 = i2, i1, g2, g1
        P1.append(gidx[i1]); P2.append(gidx[i2]); PC.append(condim); PF.append(fri5); PM.append(margin); PG.append(gap)
        PSR.append(solref); PSI.append(solimp)
        PIW.append(body_invw[g1["body"]] + body_invw[g2["body"]])

    for a in range(len(gkeep)):
        for b in range(a + 1, len(gkeep)):
            i1, i2 = gkeep[a], gkeep[b]
            g1, g2 = F.geoms[i1], F.geoms[i2]
            b1, b2 = g1["body"], g2["body"]
            w1, w2 = weld[b1], weld[b2]
            if w1 == w2:
                continue
            if w1 != 0 and w2 != 0 and (weld[parent[w1]] == w2 or weld[parent[w2]] == w1):
                continue
            if (b1, b2) in excl:
                continue
            if not ((g1["contype"] & g2["conaffinity"]) or (g2["contype"] & g1["conaffinity"])):
                continue
            if g1["type"] == GEOM_PLANE and g2["type"] == GEOM_PLANE:
                continue
            if g1["type"] == GEOM_MESH and g2["type"] == GEOM_MESH and not mesh_mesh:
                continue  # mesh-mesh narrow phase not restated yet (DESIGN.md "collision coverage")
            if g1["priority"] != g2["priority"]:
                hi = g1 if g1["priority"] > g2["priority"] else g2
                solref, solimp, fri = hi["solref"], hi["solimp"], hi["friction"]
            else:
                s1, s2 = g1["solmix"], g2["solmix"]
                mix = s1 / (s1 + s2) if (s1 >= MINVAL and s2 >= MINVAL) else (0.5 if s1 < MINVAL and s2 < MINVAL else (0.0 if s1 < MINVAL else 1.0))
                if g1["solref"][0] > 0 and g2["solref"][0] > 0:
                    solref = mix * g1["solref"] + (1 - mix) * g2["solref"]
                else:
                    solref = np.minimum(g1["solref"], g2["solref"])
                solimp = mix * g1["solimp"] + (1 - mix) * g2["solimp"]
                fri = np.maximum(g1["friction"], g2["friction"])
            add_pair(i1, i2, max(g1["condim"], g2["condim"]), np.array([fri[0], fri[0], fri[1], fri[2], fri[2]]),
                     max(g1["margin"], g2["margin"]), max(g1["gap"], g2["gap"]), solref, solimp)
    gname = {g["name"]: i for i, g in enumerate(F.geoms)}
    for pr in F.pairs:
        i1, i2 = gname[pr["geom1"]], gname[pr["geom2"]]
        g1, g2 = F.geoms[i1], F.geoms[i2]
        # an explicit pair replaces the dynamic one for the same geoms
        for k in range(len(P1) - 1, -1, -1):
            if {P1[k], P2[k]} == {gidx[i1], gidx[i2]}:
                for L in (P1, P2, PC, PF, PM, PG, PSR, PSI, PIW):
                    L.pop(k)
        fri = floats(pr.get("friction"), 5, None) if pr.get("friction") else None
        if fri is None:
            f3 = np.maximum(g1["friction"], g2["friction"])
            fri = np.array([f3[0], f3[0], f3[1], f3[2], f3[2]])
        add_pair(i1, i2, int(pr.get("condim", max(g1["condim"], g2["condim"]))), fri,
                 float(pr.get("margin", max(g1["margin"], g2["margin"]))), float(pr.get("gap", max(g1["gap"], g2["gap"]))),
                 floats(pr.get("solref"), 2, None) if pr.get("solref") else 0.5 * (g1["solref"] + g2["solref"]),
                 floats(pr.get("solimp"), 5, [0.9, 0.95, 0.001, 0.5, 2]) if pr.get("solimp") else 0.5 * (g1["solimp"] + g2["solimp"]))
    m.pair_geom1, m.pair_geom2, m.pair_condim = (np.array(x, dtype=np.int32) for x in (P1, P2, PC))
    gnames = [F.geoms[g]["name"] for g in gkeep]
    m.pair_grid, m.grid_dims, m.grid_walls, m.grid_param = _grid_tables(grid, [gnames[b] for b in P2])
    m.pair_friction = np.array(PF).reshape(-1, 5)
    m.pair_margin, m.pair_gap = np.array(PM), np.array(PG)
    m.pair_solref, m.pair_solimp, m.pair_invweight = np.array(PSR).reshape(-1, 2), np.array(PSI).reshape(-1, 5), np.array(PIW).reshape(-1, 2)

    # sites (+ one synthetic site per MJCF body so env code can read any body frame)
    sb, sp, sq, sn = [], [], [], []
    for s in F.sites:
        b = s["body"]
        sb.append(rt_of[b]); sp.append(rel_pos[b] + qrot(rel_quat[b], s["pos"])); sq.append(qmul(rel_quat[b], s["quat"])); sn.append(s["name"])
    for b in range(1, nb):
        sb.append(rt_of[b]); sp.append(rel_pos[b]); sq.append(rel_quat[b]); sn.append("bodyframe:" + F.bodies[b]["name"])
    m.site_body, m.site_pos, m.site_quat = np.array(sb, dtype=np.int32), np.array(sp).reshape(-1, 3), np.array(sq).reshape(-1, 4)

    # actuators
    jname = {J["name"]: i for i, J in enumerate(F.joints)}
    A = F.actuators
    m.act_trnid = np.array([jname[a["joint"]] for a in A], dtype=np.int32)
    m.act_ctrllimited = np.array([int(a["ctrllimited"]) for a in A], dtype=np.int32)
    m.act_forcelimited = np.array([int(a["forcelimited"]) for a in A], dtype=np.int32)
    m.act_gear = np.array([a["gear"] for a in A])
    m.act_gainprm = np.array([a["gainprm"] for a in A]).reshape(-1, 3)
    m.act_biasprm = np.array([a["biasprm"] for a in A]).reshape(-1, 3)
    m.act_ctrlrange = np.array([a["ctrlrange"] for a in A]).reshape(-1, 2)
    m.act_forcerange = np.array([a["forcerange"] for a in A]).reshape(-1, 2)

    # equalities
    et, e1, e2, ea, ed, esr, esi, eiw = [], [], [], [], [], [], [], []
    for E in F.equalities:
        a = E["attrs"]
        data = np.zeros(11)
        if E["kind"] == "weld":
            b1, b2 = name2body[a["body1"]], name2body[a.get("body2", "world")]
            anchor = floats(a.get("anchor"), 3, [0, 0, 0])
            if "relpose" in a and np.any(floats(a["relpose"]) != 0):
                rp = floats(a["relpose"])
                relpos, relquat = rp[:3], qnorm(rp[3:])
            else:
                # pose of body2 in the frame of body1 at qpos0
                relpos = xmat[b1].T @ (xpos[b2] + xmat[b2] @ anchor - xpos[b1])
                relquat = qmul(qconj(xquat[b1]), xquat[b2])
            # data layout [anchor(3) relpos(3) relquat(4) torquescale]; MuJoCo applies data[3:6] on body1 and
            # data[0:3] on body2 -- we additionally fold the offset of the MJCF body inside its runtime body.
            data[0:3], data[3:6], data[6:10], data[10] = anchor, relpos, relquat, float(a.get("torquescale", 1))
            et.append(EQ_WELD); e1.append(b1); e2.append(b2)
            eiw.append(body_invw[b1] + body_invw[b2])
        elif E["kind"] == "joint":
            j1 = jname[a["joint1"]]
            j2 = jname[a["joint2"]] if "joint2" in a else -1
            data[0:5] = floats(a.get("polycoef"), 5, [0, 1, 0, 0, 0])
            et.append(EQ_JOINT); e1.append(j1); e2.append(j2)
            w = dof_invw[F.joints[j1]["dofadr"]] + (dof_invw[F.joints[j2]["dofadr"]] if j2 >= 0 else 0)
            eiw.append([w, 0])
        else:
            raise NotImplementedError("connect equality")
        ea.append(int(E["active"])); ed.append(data); esr.append(E["solref"]); esi.append(E["solimp"])
    m.eq_type, m.eq_active = np.array(et, dtype=np.int32), np.array(ea, dtype=np.int32)
    # weld objects refer to synthetic body-frame sites so that fused bodies keep their own frames
    m.eq_obj1 = np.array([(len(F.sites) + b - 1 if t == EQ_WELD and b > 0 else (-1 if t == EQ_WELD else b)) for t, b in zip(et, e1)], dtype=np.int32)
    m.eq_obj2 = np.array([(len(F.sites) + b - 1 if t == EQ_WELD and b > 0 else (-1 if t == EQ_WELD else b)) for t, b in zip(et, e2)], dtype=np.int32)
    m.eq_data, m.eq_solref, m.eq_solimp, m.eq_invweight = (np.array(ed).reshape(-1, 11), np.array(esr).reshape(-1, 2),
                                                           np.array(esi).reshape(-1, 5), np.array(eiw).reshape(-1, 2))

    # fixed tendons
    ta, tn, tl, tr, tm, tsr, tsi, tiw, wd, wc = [], [], [], [], [], [], [], [], [], []
    for T in F.tendons:
        ta.append(len(wd)); tn.append(len(T["joints"]))
        row = np.zeros(nv)
        for jn, c in T["joints"]:
            d = F.joints[jname[jn]]["dofadr"]
            wd.append(d); wc.append(c); row[d] += c
        lim = T.get("limited", "auto")
        tl.append(int(lim == "true" or (lim == "auto" and P.compiler["autolimits"] == "true" and "range" in T)))
        tr.append(floats(T.get("range"), 2, [0, 0])); tm.append(float(T.get("margin", 0)))
        tsr.append(floats(T.get("solreflimit"), 2, [0.02, 1])); tsi.append(floats(T.get("solimplimit"), 5, [0.9, 0.95, 0.001, 0.5, 2]))
        tiw.append(float(row @ Minv @ row))
    m.ten_adr, m.ten_num, m.ten_limited = (np.array(x, dtype=np.int32) for x in (ta, tn, tl))
    m.ten_range, m.ten_margin = np.array(tr).reshape(-1, 2), np.array(tm)
    m.ten_solref, m.ten_solimp, m.ten_invweight0 = np.array(tsr).reshape(-1, 2), np.array(tsi).reshape(-1, 5), np.array(tiw)
    m.wrap_dof, m.wrap_coef = np.array(wd, dtype=np.int32), np.array(wc)

    # touch sensors (site volume + body), others ignored
    ss, sbod, ssz, sty = [], [], [], []
    sname = {s["name"]: i for i, s in enumerate(F.sites)}
    sensor_prefix = (overrides or {}).get("sensor_prefix")   # keep only the sensors an env reads (e.g. "robot0:TS_")
    for S in F.sensors:
        if S["type"] == "touch" and (sensor_prefix is None or S.get("name", "").startswith(sensor_prefix)):
            si = sname[S["site"]]
            ss.append(si); sbod.append(rt_of[F.sites[si]["body"]]); ssz.append(F.sites[si]["size"])
            sty.append(GEOM_NAMES[F.sites[si]["type"]])
            if sty[-1] not in (GEOM_NAMES["sphere"], GEOM_NAMES["box"], GEOM_NAMES["cylinder"]):
                raise NotImplementedError("touch sensor sites must be spheres, boxes or cylinders")
    m.sensor_site, m.sensor_body, m.sensor_size = np.array(ss, dtype=np.int32), np.array(sbod, dtype=np.int32), np.array(ssz).reshape(-1, 3)
    m.sensor_type = np.array(sty, dtype=np.int32)
    m.key_qpos = np.zeros(0)

    o = F.opt
    m.opt = np.array([o["timestep"], *o["gravity"], o["tolerance"], o["impratio"], meaninertia, o["ls_tolerance"]])
    m.opt_int = np.array([o["iterations"], o["ls_iterations"], o["integrator"], o["noslip_iterations"], o["warmstart"]], dtype=np.int32)
    m.sizes = np.array([nrb, len(F.joints), nq, nv, len(A), len(gkeep), len(sb), len(mocap_body), len(et), len(P1),
                        len(F.tendons), len(wd), len(ss), nM], dtype=np.int32)
    m.names = {
        "joint": [J["name"] for J in F.joints], "site": sn, "actuator": [a["name"] for a in A],
        "geom": [F.geoms[g]["name"] for g in gkeep], "body_map": {B["name"]: rt_of[i] for i, B in enumerate(F.bodies)},
        "source": os.path.basename(path),
    }
    m._reshape()
    m._full = F  # kept for tests / debugging (not serialised)
    m._full_arrays = dict(parent=parent, bpos=bpos, bquat=bquat, ipos=ipos, iquat=iquat, mass=mass, inertia=inertia,
                          M0=M0, body_invw=body_invw, weld=weld, xpos=xpos, xquat=xquat)
    return m
