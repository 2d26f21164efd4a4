"""TEST INFRASTRUCTURE.  Sensors and the material mixing table on top of the CPU oracle and the reference's real stepper.

MaterialOracle drives an unmodified oracle (oracle.OracleWorld) so that it follows the reference's material rules:
  * a new contact point (lifetime 0 after the narrowphase) gets the friction and restitution of collision_util.cpp:282-317:
    the table entry of the two bodies' material ids, else sqrt(fA fB) and min(rA, rB) in float32 -- and (0, 0) when either
    body is a sensor, whose points have no contact_point_material (collision_util.cpp:358-384);
  * a sensor's manifolds keep their points through the islands but have no rows: their points are taken out of the oracle
    for the solve and put back unchanged afterwards, so neither the velocity / position iterations nor the restitution
    solver's groups see them, while they stay edges of the entity graph;
  * the restitution solver tags the manifolds whose pair material has restitution > EPSILON (constraint_util.cpp:90-101).
    The oracle filters the tagged list it is given by its bodies' mixed restitution, so its bodies are created with
    restitution 1 (their materials live here) and the tagged list is always handed over: the reference's own
    (set_graph_order) or, by default, every such manifold in pair-key order with the adjacency the oracle would build.
RefMaterials adds material ids, sensors and the table to the reference's real stepper (tests/materials/refm.hpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "materials", "_build")
NONE, UNASSIGNED = 0xFFFFFFFF, 0xFFFF
EPS = np.float32(1.1920928955078125e-07)        # EDYN_EPSILON (float)
f32, u32 = np.float32, np.uint32


def build():
    """(Re)build tests/materials where the reference is present; elsewhere the shipped libraries are used as they are."""
    if os.path.isdir("/root/reference/include/edyn") and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "edyn_obj")):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "materials")], check=True)


def library(O, name):
    """tests/materials/_build/lib<name>.so loaded like the other refs_* libraries, or None where it is absent."""
    path = os.path.join(BUILD, f"lib{name}.so")
    if not os.path.exists(path):
        return None
    lib = O.load_refs_library(path)
    lib.refm_get_contacts.restype = C.c_uint32
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class MixingTable:
    """material_mix_table: unordered id pairs -> (friction, restitution), float32."""

    def __init__(self):
        self.entries = {}

    def set(self, id0, id1, friction, restitution):
        for a, b, f, r in zip(np.ravel(id0), np.ravel(id1), np.ravel(friction), np.ravel(restitution)):
            self.entries[(min(int(a), int(b)), max(int(a), int(b)))] = (f32(f), f32(r))

    def remove(self, id0, id1):
        for a, b in zip(np.ravel(id0), np.ravel(id1)):
            self.entries.pop((min(int(a), int(b)), max(int(a), int(b))), None)


class MaterialOracle:
    """An OracleWorld holding `scene` (its bodies' `material` column: ids, UNASSIGNED or NONE for a sensor) that follows
    the material rules above.  Everything else is the oracle's own (attribute access falls through to it)."""

    def __init__(self, O, scene, vel_iters=None, pos_iters=None, restitution=False, sleeping=False):
        from tests.parity import oracle_for
        b = scene["bodies"]
        n = len(b["kind"])
        self.O, self.restitution = O, restitution
        self.friction, self.rest = np.asarray(b["friction"], f32).copy(), np.asarray(b["restitution"], f32).copy()
        mid = b.get("material")
        self.mid = np.full(n, UNASSIGNED, u32) if mid is None else np.asarray(mid, u32).copy()
        self.sensor = self.mid == NONE
        self.table = MixingTable()
        self.graph = None
        self.hinges = scene["hinges"]
        ones = dict(scene, bodies=dict(b, restitution=np.ones(n, f32)))
        self.o = oracle_for(O, ones, vel_iters=vel_iters, pos_iters=pos_iters, restitution=restitution, sleeping=sleeping)

    def __getattr__(self, k):
        return getattr(self.o, k)

    def set_material_mixing(self, id0, id1, friction, restitution):
        self.table.set(id0, id1, friction, restitution)

    def remove_material_mixing(self, id0, id1):
        self.table.remove(id0, id1)

    def set_graph_order(self, adj_off, adj_nbr, tagged_pairs):
        """The reference's adjacency and tagged manifolds for the coming solve (see OracleWorld.set_graph_order)."""
        self.graph = (adj_off, adj_nbr, tagged_pairs)

    def pair_material(self, a, b):
        """(friction, restitution) arrays of new points between bodies a[i] and b[i]."""
        a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
        fr = np.sqrt(self.friction[a] * self.friction[b]).astype(f32)
        re = np.minimum(self.rest[a], self.rest[b]).astype(f32)
        ia, ib = self.mid[a], self.mid[b]
        for k in range(len(a)):
            if ia[k] != UNASSIGNED and ib[k] != UNASSIGNED and ia[k] != NONE and ib[k] != NONE:
                e = self.table.entries.get((min(int(ia[k]), int(ib[k])), max(int(ia[k]), int(ib[k]))))
                if e is not None:
                    fr[k], re[k] = e
        sens = self.sensor[a] | self.sensor[b]
        fr[sens] = 0
        re[sens] = 0
        return fr, re

    def run_phases(self, mask):
        O = self.O
        if mask & (O.PH_BROAD | O.PH_NARROW):
            self.o.run_phases(mask & (O.PH_BROAD | O.PH_NARROW))
            if mask & O.PH_NARROW:
                self._new_points()
        if mask & O.PH_ISLANDS:
            self.o.run_phases(O.PH_ISLANDS)
        if mask & O.PH_SOLVE:
            self._solve()

    def step(self, n=1):
        for _ in range(n):
            self.run_phases(self.O.PH_BROAD | self.O.PH_NARROW | self.O.PH_ISLANDS | self.O.PH_SOLVE)

    def _new_points(self):
        c = self.o.contacts()
        new = (np.arange(4)[None, :] < c["num"][:, None]) & (c["lifetime"] == 0)
        if not new.any():
            return
        m, s = np.nonzero(new)
        fr, re = self.pair_material(c["pairs"][m, 0], c["pairs"][m, 1])
        c["pts"][m, s, 13], c["pts"][m, s, 14] = fr, re
        self.o.set_contacts(c["pairs"], c["num"], c["pts"], c["att"], c["lifetime"])

    def _default_graph(self, c):
        """The adjacency the oracle builds when none is given (ascending neighbour id, a manifold before a joint to the same
        neighbour) and the manifolds with restitution in pair-key order (the device's tie rule)."""
        n = len(self.friction)
        nbrs = [[] for _ in range(n)]
        for a, b in c["pairs"].tolist():
            nbrs[a].append(b | 0x80000000); nbrs[b].append(a | 0x80000000)
        h = self.hinges
        for a, b in (zip(np.asarray(h["a"]).tolist(), np.asarray(h["b"]).tolist()) if h else ()):
            if a != b:
                nbrs[a].append(b); nbrs[b].append(a)
        off, flat = [0], []
        for v in nbrs:
            seen = {}
            for x in sorted(v, key=lambda x: (x & 0x7FFFFFFF, -(x >> 31))):
                seen.setdefault(x & 0x7FFFFFFF, x)
            flat += list(seen.values())
            off.append(len(flat))
        _, re = self.pair_material(c["pairs"][:, 0], c["pairs"][:, 1])
        tagged = c["pairs"][re > EPS]
        if len(tagged):
            keys = (np.minimum(tagged[:, 0], tagged[:, 1]).astype(np.uint64) << np.uint64(32)) | np.maximum(tagged[:, 0], tagged[:, 1])
            tagged = tagged[np.argsort(keys, kind="stable")]
        return np.array(off, u32), np.array(flat, u32), tagged.reshape(-1, 2)

    def _solve(self):
        c = self.o.contacts()
        sens = self.sensor[c["pairs"][:, 0]] | self.sensor[c["pairs"][:, 1]] if len(c["pairs"]) else np.zeros(0, bool)
        hide = sens & (c["num"] > 0)
        if self.restitution:
            self.o.set_graph_order(*(self.graph if self.graph is not None else self._default_graph(c)))
        self.graph = None
        if hide.any():
            num = c["num"].copy()
            num[hide] = 0
            self.o.set_contacts(c["pairs"], num, c["pts"], c["att"], c["lifetime"])
        self.o.run_phases(self.O.PH_SOLVE)
        if hide.any():
            d = self.o.contacts()
            for k in ("num", "pts", "att", "lifetime"):
                d[k][hide] = c[k][hide]
            self.o.set_contacts(d["pairs"], d["num"], d["pts"], d["att"], d["lifetime"])


class RefMaterials:
    """The refm_* entry points of a library built from tests/materials (the real stepper or the binding harness), for one
    O.RefWorld made with library=lib."""

    def __init__(self, lib, world):
        self.l, self.r = lib, world

    def add_bodies(self, b, sleeping_disabled=True):
        n = len(b["kind"])
        arr = lambda x, dt, shape: np.ascontiguousarray(np.asarray(x, dt).reshape(shape))      # noqa: E731
        a = [arr(b["pos"], f32, (n, 3)), arr(b["orn"], f32, (n, 4)), arr(b["linvel"], f32, (n, 3)), arr(b["angvel"], f32, (n, 3)),
             arr(b["inv_mass"], f32, (n,)), arr(b["gravity"], f32, (n, 3)), arr(b["kind"], u32, (n,)), arr(b["shape_kind"], u32, (n,)),
             arr(b["shape_params"], f32, (n, 4)), arr(b["friction"], f32, (n,)), arr(b["restitution"], f32, (n,))]
        grp = arr(b["group"], np.uint64, (n,)) if b.get("group") is not None else None
        msk = arr(b["mask"], np.uint64, (n,)) if b.get("mask") is not None else None
        mat = arr(b["material"] if b.get("material") is not None else np.full(n, UNASSIGNED), u32, (n,))
        rc = self.l.refm_add_bodies(self.r.h, C.c_uint32(n), *[_ptr(x) for x in a], _ptr(grp), _ptr(msk),
                                    C.c_int(1 if sleeping_disabled else 0), _ptr(mat))
        assert rc == 0, "refm_add_bodies: unsupported shape kind"

    def populate(self, scene, sleeping_disabled=True):
        self.add_bodies(scene["bodies"], sleeping_disabled)
        if scene["hinges"]:
            h = scene["hinges"]
            self.r.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
        if scene["exclusions"] is not None:
            self.r.add_exclusions(*scene["exclusions"])

    def set_material_mixing(self, id0, id1, friction, restitution):
        a, b = np.ascontiguousarray(np.ravel(id0), u32), np.ascontiguousarray(np.ravel(id1), u32)
        f, r = np.ascontiguousarray(np.ravel(friction), f32), np.ascontiguousarray(np.ravel(restitution), f32)
        self.l.refm_set_material_mixing(self.r.h, C.c_uint32(len(a)), _ptr(a), _ptr(b), _ptr(f), _ptr(r), C.c_int(0))

    def remove_material_mixing(self, id0, id1):
        a, b = np.ascontiguousarray(np.ravel(id0), u32), np.ascontiguousarray(np.ravel(id1), u32)
        self.l.refm_set_material_mixing(self.r.h, C.c_uint32(len(a)), _ptr(a), _ptr(b), None, None, C.c_int(1))

    def contacts(self):
        """pairs, num, pts (m, 4, 14) as RefWorld.contacts, and mat (m, 4, 4): friction, restitution (0 without a
        contact_point_material), 1 with a contact_constraint, 1 with a contact_point_impulse."""
        m = int(self.l.refs_num_manifolds(self.r.h))
        k = max(m, 1)
        pairs, num, pts, mat = np.zeros((k, 2), u32), np.zeros(k, u32), np.zeros((k, 4, 14), f32), np.zeros((k, 4, 4), f32)
        got = int(self.l.refm_get_contacts(self.r.h, C.c_uint32(m), _ptr(pairs), _ptr(num), _ptr(pts), _ptr(mat)))
        return dict(pairs=pairs[:got], num=num[:got], pts=pts[:got], mat=mat[:got])
