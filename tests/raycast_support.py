"""TEST INFRASTRUCTURE for the raycast tests: builds and loads
  * tests/raycast/ora_raycast.cpp -- the CPU restatement of the world raycast (brute force, include/b2d.h semantics),
    self-contained, g++ only;
  * tests/raycast/ref_raycast.cpp -- the reference's own shape_raycast / edyn::raycast, linked with the reference's object
    files in oracle/_ref/edyn_obj; None where those were not built (they need /root/reference at build time).
Both are compiled once per source version into a directory under the system temporary directory, so the repository tree
is never written."""
import ctypes as C
import glob
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests", "raycast")
REF = "/root/reference"
REF_OBJ = os.path.join(ROOT, "oracle", "_ref", "edyn_obj")
FLAGS = ["-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"]
MISS = 0xFFFFFFFF


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(x, shape=None):
    a = np.ascontiguousarray(np.asarray(x, np.float32))
    return a.reshape(shape) if shape is not None else a


def _u32(x, shape=None):
    a = np.ascontiguousarray(np.asarray(x, np.uint32))
    return a.reshape(shape) if shape is not None else a


def _build(name, srcs, cmd_tail, extra_deps=()):
    h = hashlib.sha1()
    for p in list(srcs) + list(extra_deps):
        h.update(p.encode())
        h.update(open(p, "rb").read() if os.path.getsize(p) < (1 << 22) else str(os.path.getmtime(p)).encode())
    h.update(" ".join(cmd_tail).encode())
    out_dir = os.path.join(tempfile.gettempdir(), f"edyn_b200_raycast_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    lib = os.path.join(out_dir, f"{name}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(lib):
        tmp = lib + f".{os.getpid()}.tmp"
        subprocess.run([os.environ.get("CXX", "g++")] + FLAGS + ["-o", tmp] + list(srcs) + list(cmd_tail), check=True)
        os.replace(tmp, lib)
    return lib


_ora = None
_ref = None


def ora():
    global _ora
    if _ora is None:
        src = os.path.join(HERE, "ora_raycast.cpp")
        _ora = C.CDLL(_build("ora_raycast", [src], ["-O2"], [os.path.join(ROOT, "oracle", "ora_math.hpp")]))
    return _ora


def ref():
    """The reference's raycast, or None where its object files are not available."""
    global _ref
    if _ref is None:
        objs = sorted(glob.glob(os.path.join(REF_OBJ, "**", "*.o"), recursive=True))
        if not objs or not os.path.isdir(os.path.join(REF, "include", "edyn")):
            return None
        src = os.path.join(HERE, "ref_raycast.cpp")
        flags = ["-O2", "-w", "-DEDYN_DISABLE_ASSERT", "-DNDEBUG", "-pthread", "-fvisibility=hidden", "-ffunction-sections",
                 "-fdata-sections", "-Wl,--gc-sections", "-I" + os.path.join(ROOT, "oracle", "entt_lite"),
                 "-I" + os.path.join(REF, "include")] + objs
        _ref = C.CDLL(_build("ref_raycast", [src], flags, [os.path.join(REF_OBJ, "collision", "raycast.o")]), mode=os.RTLD_NOW)
        _ref.rr_create.restype = C.c_void_p
    return _ref


def shape_raycast(lib, prefix, kind, p, pos, orn, p0, p1):
    """(hit, fraction, normal(3), feature) of one shape; hit = the reference reported a result (fraction < FLT_MAX)."""
    out, feat = np.zeros(4, np.float32), np.zeros(1, np.uint32)
    args = [_f32(x) for x in (p, pos, orn, p0, p1)]
    getattr(lib, prefix + "shape_raycast")(C.c_uint32(int(kind)), *[_ptr(a) for a in args], _ptr(out), _ptr(feat))
    return bool(out[0] != np.finfo(np.float32).max), out[0], out[1:4].copy(), int(feat[0])


def world_raycast(pos, orn, shape_kind, shape_params, p0, p1, ignore=(), ignore_body=None):
    """Brute-force world raycast over the given bodies (shape kind 255 = no shape / removed): dict of body, fraction,
    normal, feature per segment, as World.raycast returns them."""
    pos, orn, sk, sp = _f32(pos, (-1, 3)), _f32(orn, (-1, 4)), _u32(shape_kind), _f32(shape_params, (-1, 4))
    a, b = _f32(p0, (-1, 3)), _f32(p1, (-1, 3))
    n = len(a)
    ign = _u32(list(ignore)).reshape(-1)
    ib = _u32(ignore_body, (n,)) if ignore_body is not None else None
    out = dict(body=np.zeros(n, np.uint32), fraction=np.zeros(n, np.float32), normal=np.zeros((n, 3), np.float32),
               feature=np.zeros(n, np.uint32))
    ora().ora_world_raycast(C.c_uint32(len(sk)), _ptr(pos), _ptr(orn), _ptr(sk), _ptr(sp), C.c_uint32(n), _ptr(a), _ptr(b),
                            _ptr(ib), _ptr(ign) if len(ign) else None, C.c_uint32(len(ign)), _ptr(out["body"]),
                            _ptr(out["fraction"]), _ptr(out["normal"]), _ptr(out["feature"]))
    return out


class RefWorld:
    """Static bodies in a reference registry, queried with the reference's own edyn::raycast."""

    def __init__(self, pos, orn, shape_kind, shape_params):
        self.l = ref()
        pos, orn, sk, sp = _f32(pos, (-1, 3)), _f32(orn, (-1, 4)), _u32(shape_kind), _f32(shape_params, (-1, 4))
        self.h = C.c_void_p(self.l.rr_create(C.c_uint32(len(sk)), _ptr(pos), _ptr(orn), _ptr(sk), _ptr(sp)))

    def raycast(self, p0, p1, ignore=()):
        body, out, feat = np.zeros(1, np.uint32), np.zeros(4, np.float32), np.zeros(1, np.uint32)
        ign = _u32(list(ignore)).reshape(-1)
        self.l.rr_raycast(self.h, _ptr(_f32(p0)), _ptr(_f32(p1)), _ptr(ign) if len(ign) else None, C.c_uint32(len(ign)),
                          _ptr(body), _ptr(out), _ptr(feat))
        return int(body[0]), out[0], out[1:4].copy(), int(feat[0])

    def close(self):
        if self.h:
            self.l.rr_destroy(self.h)
            self.h = None


class BruteWorld:
    """Bodies (as edyn_b200 scene / World.add_bodies dicts) for the brute-force world raycast: positions and
    orientations follow set_state, removed bodies lose their shape."""

    def __init__(self):
        self.pos, self.orn = np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32)
        self.kind, self.params = np.zeros(0, np.uint32), np.zeros((0, 4), np.float32)

    def add_bodies(self, b):
        self.pos = np.vstack([self.pos, _f32(b["pos"], (-1, 3))])
        self.orn = np.vstack([self.orn, _f32(b["orn"], (-1, 4))])
        self.kind = np.concatenate([self.kind, _u32(b["shape_kind"]).reshape(-1)])
        self.params = np.vstack([self.params, _f32(b["shape_params"], (-1, 4))])

    def set_state(self, pos, orn, linvel=None, angvel=None):
        self.pos, self.orn = _f32(pos, (-1, 3)).copy(), _f32(orn, (-1, 4)).copy()

    def remove_bodies(self, ids):
        self.kind[np.asarray(ids, np.int64)] = 255

    def raycast(self, p0, p1, ignore=(), ignore_body=None):
        return world_raycast(self.pos, self.orn, self.kind, self.params, p0, p1, ignore, ignore_body)
