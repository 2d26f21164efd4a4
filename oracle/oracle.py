"""TEST INFRASTRUCTURE -- ctypes front-end of the CPU oracle (oracle/liboracle.so) and, when it
was built, of the real reference functions (oracle/_ref/libedyn_ref.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product package (edyn_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle.so")
REF_SO = os.path.join(HERE, "_ref", "libedyn_ref.so")
STEPPER_SO = os.path.join(HERE, "_ref", "libedyn_stepper.so")

SH_SPHERE, SH_CAPSULE, SH_BOX, SH_PLANE, SH_NONE = 0, 2, 3, 6, 255
DYNAMIC, KINEMATIC, STATIC = 0, 1, 2
PH_BROAD, PH_NARROW, PH_ISLANDS, PH_SOLVE = 1, 2, 4, 8
# process_collision's branches in the order of merge_branch (ora_world.hpp): bit positions of OracleWorld.merge_trace()
MERGE_BRANCHES = (
    "settled", "early_return", "empty_keep", "empty_remove", "nearest_a", "nearest_b", "roll_a", "roll_b", "roll_both",
    "taken", "remove_normal", "remove_tangent", "remove_first", "remove_middle", "remove_last", "remove_gap", "remove_all4",
    "kept", "ins1_append", "ins1_similar", "ins2_append", "ins2_similar", "ins2_replace0", "ins2_replace1", "ins2_none",
    "ins3_none", "ins3_append", "ins3_col1", "ins3_col0", "ins3_col2", "ins3_shortest", "ins4_similar", "ins4_replace0",
    "ins4_replace1", "ins4_replace2", "ins4_replace3", "ins4_none", "pivot_b", "similar_inplace", "similar_moved",
    "similar_created", "replace_persisted", "replace_after_gap", "replace_then_similar", "similar_then_replace", "full4",
    "move_up", "move_down", "move_both")

_f = np.float32
_u = np.uint32


def build(force=False):
    """Compile the restatement (always) and oracle/_ref (only where /root/reference exists)."""
    if force or not os.path.exists(ORACLE_SO) or os.path.isdir("/root/reference/src/edyn"):
        subprocess.run(["make", "-s", "-C", HERE], check=True)
    # the reference's whole sequential stepper (about a minute on 8 cores the first time, a no-op make afterwards)
    if os.path.isdir("/root/reference/src/edyn"):
        subprocess.run(["make", "-s", "-j", str(os.cpu_count() or 4), "-C", HERE, "stepper"], check=True)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _arr(x, dt, shape=None):
    a = np.ascontiguousarray(np.asarray(x, dtype=dt))
    if shape is not None:
        a = a.reshape(shape)
    return a


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_SO):
            build()
        _lib = C.CDLL(ORACLE_SO)
        _lib.ora_create.restype = C.c_void_p
        _lib.ora_create.argtypes = [C.c_float, C.c_int, C.c_int, C.c_int]
        _lib.ora_solve_row.restype = C.c_float
        for name in ("ora_num_bodies", "ora_num_manifolds", "ora_get_merge_trace"):
            getattr(_lib, name).restype = C.c_uint32
    return _lib


def ref():
    """The real reference functions, or None when oracle/_ref was not built/shipped."""
    global _ref
    if _ref is None and os.path.exists(REF_SO):
        _ref = C.CDLL(REF_SO)
        _ref.ref_solve_row.restype = C.c_float
    return _ref


class PureFns:
    """Pure-function surface shared by the restatement (prefix 'ora_') and the reference ('ref_')."""

    def __init__(self, dll, prefix):
        self.dll, self.p = dll, prefix

    def _fn(self, name):
        return getattr(self.dll, self.p + name)

    def collide(self, kindA, pA, kindB, pB, posA, ornA, posB, ornB):
        out = np.zeros((4, 10), _f)
        att = np.zeros(4, _u)
        args = [_arr(x, _f) for x in (pA, pB, posA, ornA, posB, ornB)]
        n = self._fn("collide")(C.c_uint32(kindA), _ptr(args[0]), C.c_uint32(kindB), _ptr(args[1]), _ptr(args[2]),
                                _ptr(args[3]), _ptr(args[4]), _ptr(args[5]), _ptr(out), _ptr(att))
        return out[:n].copy(), att[:n].copy()

    def shape_aabb(self, kind, p, pos, orn):
        out = np.zeros(6, _f)
        a = [_arr(x, _f) for x in (p, pos, orn)]
        self._fn("shape_aabb")(C.c_uint32(kind), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(out))
        return out

    def integrate(self, q, w, dt):
        out = np.zeros(4, _f)
        a = [_arr(q, _f), _arr(w, _f)]
        self._fn("integrate")(_ptr(a[0]), _ptr(a[1]), C.c_float(dt), _ptr(out))
        return out

    def plane_space(self, n):
        p, q = np.zeros(3, _f), np.zeros(3, _f)
        a = _arr(n, _f)
        self._fn("plane_space")(_ptr(a), _ptr(p), _ptr(q))
        return p, q

    def intersect_line_aabb(self, p0, p1, mn, mx):
        s = np.zeros(2, _f)
        a = [_arr(x, _f) for x in (p0, p1, mn, mx)]
        fn = self._fn("intersect_line_aabb")
        fn.restype = C.c_int
        n = fn(_ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), _ptr(s))
        return n, s

    def closest_segment_segment(self, p1, q1, p2, q2):
        out = np.zeros(16, _f)
        d = C.c_float(0)
        a = [_arr(x, _f) for x in (p1, q1, p2, q2)]
        fn = self._fn("closest_segment_segment")
        fn.restype = C.c_int
        n = fn(_ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), _ptr(out), C.byref(d))
        return n, out, d.value

    def maybe_add_points(self, pivA, pivB):
        pivA, pivB = _arr(pivA, _f, (-1, 3)), _arr(pivB, _f, (-1, 3))
        oa, ob = np.zeros((4, 3), _f), np.zeros((4, 3), _f)
        fn = self._fn("maybe_add_points")
        fn.restype = C.c_int
        n = fn(C.c_uint32(len(pivA)), _ptr(pivA), _ptr(pivB), _ptr(oa), _ptr(ob))
        return oa[:n].copy(), ob[:n].copy()

    def moment_of_inertia(self, kind, p, mass):
        out = np.zeros(9, _f)
        a = _arr(p, _f)
        self._fn("moment_of_inertia")(C.c_uint32(kind), _ptr(a), C.c_float(mass), _ptr(out))
        return out.reshape(3, 3)

    def inverse_symmetric(self, m):
        out = np.zeros(9, _f)
        a = _arr(m, _f)
        self._fn("inverse_symmetric")(_ptr(a), _ptr(out))
        return out.reshape(3, 3)

    def world_inertia(self, orn, inv_I):
        out = np.zeros(9, _f)
        a = [_arr(orn, _f), _arr(inv_I, _f)]
        self._fn("world_inertia")(_ptr(a[0]), _ptr(a[1]), _ptr(out))
        return out.reshape(3, 3)

    def prepare_row(self, J, inv_mA, inv_IA, inv_mB, inv_IB, error, erp, restitution, vels):
        out = np.zeros(2, _f)
        a = [_arr(J, _f), _arr(inv_IA, _f), _arr(inv_IB, _f), _arr(vels, _f)]
        self._fn("prepare_row")(_ptr(a[0]), C.c_float(inv_mA), _ptr(a[1]), C.c_float(inv_mB), _ptr(a[2]),
                                C.c_float(error), C.c_float(erp), C.c_float(restitution), _ptr(a[3]), _ptr(out))
        return out

    def solve_row(self, J, row5, dv12):
        r = _arr(row5, _f).copy()
        a = [_arr(J, _f), _arr(dv12, _f)]
        fn = self._fn("solve_row")
        fn.restype = C.c_float
        d = fn(_ptr(a[0]), _ptr(r), _ptr(a[1]))
        return np.float32(d), r


    def solve_friction(self, J24, fr6, mu, normal_impulse, masses20, dv12, warm=False):
        """solve_friction / warm_start of a constraint_row_friction; returns (impulse[2], dv12) after the call."""
        fr, dv = _arr(fr6, _f).copy(), _arr(dv12, _f).copy()
        a = [_arr(J24, _f), _arr(masses20, _f)]
        self._fn("solve_friction")(_ptr(a[0]), _ptr(fr), C.c_float(mu), C.c_float(normal_impulse), _ptr(a[1]), _ptr(dv), C.c_int(int(warm)))
        return fr[4:6].copy(), dv


    def contact_prepare(self, cp15, dt, bodyA23, bodyB23):
        """contact_constraint::prepare -> dict(nJ, n5 = lower upper impulse error restitution, fJ, fr6, mu)."""
        nJ, n5, fJ, fr6, mu = np.zeros(12, _f), np.zeros(5, _f), np.zeros(24, _f), np.zeros(6, _f), C.c_float(0)
        a = [_arr(cp15, _f), _arr(bodyA23, _f), _arr(bodyB23, _f)]
        self._fn("contact_prepare")(_ptr(a[0]), C.c_float(dt), _ptr(a[1]), _ptr(a[2]), _ptr(nJ), _ptr(n5), _ptr(fJ), _ptr(fr6), C.byref(mu))
        return dict(nJ=nJ, n5=n5, fJ=fJ, fr6=fr6, mu=np.float32(mu.value))

    def contact_solve_position(self, cp13, bodyA26, bodyB26):
        """contact_constraint::solve_position + position_solver::solve -> (solved, bodyA26', bodyB26', out5 = normal distance max_error)."""
        a, b, out = _arr(bodyA26, _f).copy(), _arr(bodyB26, _f).copy(), np.zeros(5, _f)
        cp = _arr(cp13, _f)
        fn = self._fn("contact_solve_position")
        fn.restype = C.c_int
        solved = fn(_ptr(cp), _ptr(a), _ptr(b), _ptr(out))
        return int(solved), a, b, out


    def find_nearest_contact(self, cpA, cpB, resA, resB):
        resA, resB = _arr(resA, _f, (-1, 3)), _arr(resB, _f, (-1, 3))
        fn = self._fn("find_nearest_contact"); fn.restype = C.c_uint32
        return int(fn(_ptr(_arr(cpA, _f)), _ptr(_arr(cpB, _f)), C.c_uint32(len(resA)), _ptr(resA), _ptr(resB)))

    def find_nearest_contact_rolling(self, resA, cp_pivot, origin, orn, angvel, dt):
        resA = _arr(resA, _f, (-1, 3))
        fn = self._fn("find_nearest_contact_rolling"); fn.restype = C.c_uint32
        a = [_arr(cp_pivot, _f), _arr(origin, _f), _arr(orn, _f), _arr(angvel, _f)]
        return int(fn(C.c_uint32(len(resA)), _ptr(resA), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), C.c_float(dt)))

    def should_remove_point(self, pivotA, pivotB, normal, posA, ornA, posB, ornB):
        fn = self._fn("should_remove_point"); fn.restype = C.c_int
        a = [_arr(x, _f) for x in (pivotA, pivotB, normal, posA, ornA, posB, ornB)]
        return bool(fn(*[_ptr(x) for x in a]))


    def hinge_solve_position(self, hinge12, bodyA26, bodyB26):
        a, b = _arr(bodyA26, _f).copy(), _arr(bodyB26, _f).copy()
        fn = self._fn("hinge_solve_position"); fn.restype = C.c_float
        err = fn(_ptr(_arr(hinge12, _f)), _ptr(a), _ptr(b))
        return np.float32(err), a, b

    def material_mix(self, fa, fb, ra, rb):
        out = np.zeros(2, _f)
        self._fn("material_mix")(C.c_float(fa), C.c_float(fb), C.c_float(ra), C.c_float(rb), _ptr(out))
        return out

    def intersect_aabb(self, a6, b6):
        fn = self._fn("intersect_aabb"); fn.restype = C.c_int
        return bool(fn(_ptr(_arr(a6, _f)), _ptr(_arr(b6, _f))))


def ref_connected_components(non_connecting, edges):
    """entity_graph::connected_components of the reference (None when oracle/_ref is absent): label per node."""
    r = ref()
    if r is None:
        return None
    nc = _arr(non_connecting, np.uint8)
    e = _arr(edges, _u, (-1, 2))
    out = np.zeros(len(nc), _u)
    r.ref_connected_components.restype = C.c_uint32
    r.ref_connected_components(C.c_uint32(len(nc)), _ptr(nc), C.c_uint32(len(e)), _ptr(e), _ptr(out))
    return out


def ref_broadphase_pairs(aabb0, aabb1, procedural, cap=1 << 16):
    """Pair search of broadphase::update around the reference's real dynamic AABB trees (oracle/ref_glue.cpp); ordered
    (querying body, other) pairs, or None when oracle/_ref is absent."""
    r = ref()
    if r is None:
        return None
    a0, a1 = _arr(aabb0, _f, (-1, 6)), _arr(aabb1, _f, (-1, 6))
    pr = _arr(procedural, np.uint8)
    out = np.zeros((cap, 2), _u)
    r.ref_broadphase_pairs.restype = C.c_uint32
    k = r.ref_broadphase_pairs(C.c_uint32(len(pr)), _ptr(a0), _ptr(a1), _ptr(pr), C.c_uint32(cap), _ptr(out))
    assert k <= cap
    return out[:k].copy()


def ora_fns():
    return PureFns(lib(), "ora_")


def ref_fns():
    r = ref()
    return PureFns(r, "ref_") if r is not None else None


def hinge_rows(which, pivotA, pivotB, axisA, axisB, posA, ornA, posB, ornB):
    """which = 'ora' (restatement) or 'ref' (real reference): the 5 hinge Jacobians as (5, 4, 3)."""
    dll = lib() if which == "ora" else ref()
    fn = getattr(dll, which + "_hinge_rows")
    J = np.zeros(60, _f)
    a = [_arr(x, _f) for x in (pivotA, pivotB, axisA, axisB, posA, ornA, posB, ornB)]
    fn.restype = C.c_int
    n = fn(*[_ptr(x) for x in a], _ptr(J))
    return n, J.reshape(5, 4, 3)


class OracleWorld:
    """CPU restatement of one edyn registry stepped by stepper_sequential (see ora_world.hpp)."""

    def __init__(self, dt=1.0 / 60, vel_iters=8, pos_iters=3, threads=1):
        self.l = lib()
        self.h = C.c_void_p(self.l.ora_create(C.c_float(dt), vel_iters, pos_iters, threads))
        self.dt = dt
        self.num_hinges = 0

    def __del__(self):
        try:
            if self.h:
                self.l.ora_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def add_bodies(self, b):
        """b: dict of arrays as produced by edyn_b200.scenes / edyn_b200.bodies_soa()."""
        n = len(b["kind"])
        a = dict(pos=_arr(b["pos"], _f, (n, 3)), orn=_arr(b["orn"], _f, (n, 4)), linvel=_arr(b["linvel"], _f, (n, 3)),
                 angvel=_arr(b["angvel"], _f, (n, 3)), inv_mass=_arr(b["inv_mass"], _f, (n,)),
                 inv_inertia=_arr(b["inv_inertia"], _f, (n, 9)), gravity=_arr(b["gravity"], _f, (n, 3)),
                 kind=_arr(b["kind"], _u, (n,)), shape_kind=_arr(b["shape_kind"], _u, (n,)),
                 shape_params=_arr(b["shape_params"], _f, (n, 4)), friction=_arr(b["friction"], _f, (n,)),
                 restitution=_arr(b["restitution"], _f, (n,)))
        grp = _arr(b["group"], np.uint64, (n,)) if "group" in b and b["group"] is not None else None
        msk = _arr(b["mask"], np.uint64, (n,)) if "mask" in b and b["mask"] is not None else None
        self.l.ora_add_bodies.restype = C.c_int
        return self.l.ora_add_bodies(self.h, C.c_uint32(n), _ptr(a["pos"]), _ptr(a["orn"]), _ptr(a["linvel"]),
                                     _ptr(a["angvel"]), _ptr(a["inv_mass"]), _ptr(a["inv_inertia"]), _ptr(a["gravity"]),
                                     _ptr(a["kind"]), _ptr(a["shape_kind"]), _ptr(a["shape_params"]),
                                     _ptr(a["friction"]), _ptr(a["restitution"]), _ptr(grp), _ptr(msk))

    def add_hinges(self, a, b, pivotA, pivotB, axisA, axisB):
        n = len(a)
        arrs = [_arr(a, _u), _arr(b, _u), _arr(pivotA, _f, (n, 3)), _arr(pivotB, _f, (n, 3)), _arr(axisA, _f, (n, 3)),
                _arr(axisB, _f, (n, 3))]
        self.num_hinges += n
        return self.l.ora_add_hinges(self.h, C.c_uint32(n), *[_ptr(x) for x in arrs])

    def remove_bodies(self, ids):
        ids = _arr(ids, _u)
        self.l.ora_remove_bodies(self.h, C.c_uint32(len(ids)), _ptr(ids))

    def set_sleeping(self, enabled=True):
        self.l.ora_set_sleeping(self.h, int(bool(enabled)))

    def wake_bodies(self, ids):
        ids = _arr(ids, _u)
        self.l.ora_wake_bodies(self.h, C.c_uint32(len(ids)), _ptr(ids))

    def sleeping(self):
        out = np.zeros(self.num_bodies, _u)
        self.l.ora_get_sleeping(self.h, _ptr(out))
        return out.astype(bool)

    def add_exclusions(self, a, b):
        a, b = _arr(a, _u), _arr(b, _u)
        self.l.ora_add_exclusions(self.h, C.c_uint32(len(a)), _ptr(a), _ptr(b))

    def remove_exclusions(self, a, b):
        a, b = _arr(a, _u), _arr(b, _u)
        self.l.ora_remove_exclusions(self.h, C.c_uint32(len(a)), _ptr(a), _ptr(b))

    def step(self, n=1):
        self.l.ora_step(self.h, int(n))

    def run_phases(self, mask):
        self.l.ora_run_phases(self.h, C.c_uint32(mask))

    @property
    def num_bodies(self):
        return int(self.l.ora_num_bodies(self.h))

    def state(self):
        n = self.num_bodies
        out = dict(pos=np.zeros((n, 3), _f), orn=np.zeros((n, 4), _f), linvel=np.zeros((n, 3), _f),
                   angvel=np.zeros((n, 3), _f), aabb=np.zeros((n, 6), _f), inv_IW=np.zeros((n, 9), _f))
        self.l.ora_get_state(self.h, _ptr(out["pos"]), _ptr(out["orn"]), _ptr(out["linvel"]), _ptr(out["angvel"]),
                             _ptr(out["aabb"]), _ptr(out["inv_IW"]))
        return out

    def set_state(self, pos, orn, linvel, angvel):
        a = [_arr(pos, _f), _arr(orn, _f), _arr(linvel, _f), _arr(angvel, _f)]
        self.l.ora_set_state(self.h, *[_ptr(x) for x in a])

    def pairs(self):
        m = int(self.l.ora_num_manifolds(self.h))
        p = np.zeros((m, 2), _u)
        if m:
            self.l.ora_get_pairs(self.h, _ptr(p))
        return p

    def contacts(self):
        m = int(self.l.ora_num_manifolds(self.h))
        num = np.zeros(m, _u)
        pts = np.zeros((m, 4, 18), _f)
        u = np.zeros((m, 4, 2), _u)
        if m:
            self.l.ora_get_contacts(self.h, _ptr(num), _ptr(pts), _ptr(u))
        return dict(pairs=self.pairs(), num=num, pts=pts, att=u[:, :, 0].copy(), lifetime=u[:, :, 1].copy())

    def set_contacts(self, pairs, num, pts, att, lifetime=None):
        pairs = _arr(pairs, _u, (-1, 2))
        m = len(pairs)
        num = _arr(num, _u, (m,))
        pts = _arr(pts, _f, (m, 4, 18))
        u = np.zeros((m, 4, 2), _u)
        u[:, :, 0] = _arr(att, _u, (m, 4))
        if lifetime is not None:
            u[:, :, 1] = _arr(lifetime, _u, (m, 4))
        self.l.ora_set_contacts(self.h, C.c_uint32(m), _ptr(pairs), _ptr(num), _ptr(pts), _ptr(u))

    def set_merge_trace(self, on=True):
        """Record, in every following narrowphase, which branches of process_collision each manifold took."""
        self.l.ora_set_merge_trace(self.h, C.c_int(1 if on else 0))

    def merge_trace(self):
        """One uint64 per manifold from the last narrowphase: bit b = branch b of MERGE_BRANCHES was taken."""
        m = int(self.l.ora_num_manifolds(self.h))
        out = np.zeros(max(m, 1), np.uint64)
        self.l.ora_get_merge_trace(self.h, _ptr(out))
        return out[:m]

    def islands(self):
        lab = np.zeros(self.num_bodies, _u)
        self.l.ora_get_islands(self.h, _ptr(lab))
        return lab

    def set_islands(self, labels):
        """Partition used by the next PH_SOLVE instead of the connected components computed by PH_ISLANDS."""
        lab = _arr(labels, _u, (self.num_bodies,))
        self.l.ora_set_islands(self.h, _ptr(lab))

    def should_collide(self, a, b):
        self.l.ora_should_collide.restype = C.c_int
        return bool(self.l.ora_should_collide(self.h, C.c_uint32(a), C.c_uint32(b)))

    def hinge_impulses(self):
        imp = np.zeros((max(1, self.num_hinges), 5), _f)
        self.l.ora_get_hinge_impulses(self.h, _ptr(imp))
        return imp[:self.num_hinges]

    def set_hinge_impulses(self, imp5):
        imp = _arr(imp5, _f, (self.num_hinges, 5))
        if self.num_hinges:
            self.l.ora_set_hinge_impulses(self.h, _ptr(imp))

    def set_order(self, hinge_idx, pairs):
        h = _arr(hinge_idx, _u)
        p = _arr(pairs, _u, (-1, 2))
        self.l.ora_set_order(self.h, C.c_uint32(len(h)), _ptr(h), C.c_uint32(len(p)), _ptr(p))

    def set_point_order(self, hinge_idx, contact3):
        """Row order with one entry per contact ROW: (body0, body1, index of the point in the manifold's list)."""
        hinge_idx = _arr(hinge_idx, _u)
        contact3 = _arr(contact3, _u, (-1, 3))
        self.l.ora_set_point_order(self.h, C.c_uint32(len(hinge_idx)), _ptr(hinge_idx), C.c_uint32(len(contact3)), _ptr(contact3))

    def set_position_type_order(self, contacts_first):
        """Position iterations sweep the constraint types in the compiler's argument evaluation order
        (island_solver.cpp:340): tuple order (joints, then contacts; default) or GCC's (contacts first)."""
        self.l.ora_set_position_type_order(self.h, C.c_int(1 if contacts_first else 0))

    def set_position_renormalize_all(self, on):
        """Process-wide: position_solver::solve's in-place normalisation of NON-procedural bodies' orientation too
        (position_solver.hpp:26-32); only matters for static bodies whose quaternion is an ulp off unit length."""
        self.l.ora_set_position_renormalize_all(C.c_int(1 if on else 0))

    def set_pool_order(self, on):
        """Broadphase queries in the procedural_tag pool's order, swap-and-pop on removal included (which body of a new
        pair is body[0] after bodies were destroyed); off = descending index, the device's rule."""
        self.l.ora_set_pool_order(self.h, C.c_int(1 if on else 0))

    def set_restitution_iterations(self, iterations, individual=3):
        """settings.num_restitution_iterations / num_individual_restitution_iterations (reference defaults 8 / 3; 0 = the
        restitution solver is off and restitution goes through the row rhs)."""
        self.l.ora_set_restitution_iterations(self.h, C.c_int(iterations), C.c_int(individual))

    def set_graph_order(self, adj_off, adj_nbr, tagged_pairs):
        off, nbr, tag = _arr(adj_off, _u), _arr(adj_nbr, _u), _arr(tagged_pairs, _u, (-1, 2))
        self.l.ora_set_graph_order(self.h, _ptr(off), _ptr(nbr), C.c_uint32(len(tag)), _ptr(tag))

    def clear_order(self):
        self.l.ora_clear_order(self.h)


# ---------------------------------------------------------------------------------------------------------------------
# The reference itself: edyn::attach / make_rigidbody / make_constraint<hinge_constraint> / exclude_collision /
# step_simulation compiled in place from /root/reference against oracle/entt_lite (oracle/ref_stepper.cpp, `make stepper`).

_stepper = None


def load_refs_library(path):
    """dlopen a library exporting the refs_* interface of oracle/ref_stepper.cpp and declare the non-int signatures."""
    l = C.CDLL(path, mode=os.RTLD_NOW)
    l.refs_create.restype = C.c_void_p
    l.refs_create.argtypes = [C.c_float, C.c_int, C.c_int, C.c_int, C.c_int]
    for name in ("refs_num_bodies", "refs_num_manifolds", "refs_get_contacts"):
        getattr(l, name).restype = C.c_uint32
    return l


def ref_stepper():
    """The library, or None where it was neither built here nor shipped (it needs /root/reference at build time)."""
    global _stepper
    if _stepper is None and os.path.exists(STEPPER_SO):
        _stepper = load_refs_library(STEPPER_SO)
    return _stepper


class RefWorld:
    """One registry stepped by the reference's own stepper_sequential.  threads = 0: execution_mode::sequential;
    threads > 0: sequential_multithreaded with that many workers (edyn.cpp:85-89)."""

    def __init__(self, dt=1.0 / 60, vel_iters=8, pos_iters=3, restitution_iters=0, threads=0, library=None):
        self.l = library if library is not None else ref_stepper()
        if self.l is None:
            raise RuntimeError("oracle/_ref/libedyn_stepper.so is not available")
        self.h = C.c_void_p(self.l.refs_create(C.c_float(dt), vel_iters, pos_iters, restitution_iters, threads))
        self.num_hinges = 0

    def __del__(self):
        try:
            if self.h:
                self.l.refs_destroy(self.h)
                self.h = None
        except Exception:
            pass

    @property
    def num_bodies(self):
        return int(self.l.refs_num_bodies(self.h))

    def add_bodies(self, b, sleeping_disabled=True):
        n = len(b["kind"])
        a = [_arr(b["pos"], _f, (n, 3)), _arr(b["orn"], _f, (n, 4)), _arr(b["linvel"], _f, (n, 3)), _arr(b["angvel"], _f, (n, 3)),
             _arr(b["inv_mass"], _f, (n,)), _arr(b["gravity"], _f, (n, 3)), _arr(b["kind"], _u, (n,)), _arr(b["shape_kind"], _u, (n,)),
             _arr(b["shape_params"], _f, (n, 4)), _arr(b["friction"], _f, (n,)), _arr(b["restitution"], _f, (n,))]
        grp = _arr(b["group"], np.uint64, (n,)) if b.get("group") is not None else None
        msk = _arr(b["mask"], np.uint64, (n,)) if b.get("mask") is not None else None
        rc = self.l.refs_add_bodies(self.h, C.c_uint32(n), *[_ptr(x) for x in a], _ptr(grp), _ptr(msk), C.c_int(1 if sleeping_disabled else 0))
        if rc:
            raise RuntimeError("refs_add_bodies: unsupported shape kind")

    def add_hinges(self, a, b, pivotA, pivotB, axisA, axisB):
        n = len(a)
        arrs = [_arr(a, _u), _arr(b, _u), _arr(pivotA, _f, (n, 3)), _arr(pivotB, _f, (n, 3)), _arr(axisA, _f, (n, 3)), _arr(axisB, _f, (n, 3))]
        self.num_hinges += n
        return self.l.refs_add_hinges(self.h, C.c_uint32(n), *[_ptr(x) for x in arrs])

    def add_exclusions(self, a, b):
        a, b = _arr(a, _u), _arr(b, _u)
        self.l.refs_add_exclusions(self.h, C.c_uint32(len(a)), _ptr(a), _ptr(b))

    def step(self, n=1):
        self.l.refs_step(self.h, C.c_uint32(n))

    def state(self):
        n = self.num_bodies
        pos, orn, lv, av, bb = np.zeros((n, 3), _f), np.zeros((n, 4), _f), np.zeros((n, 3), _f), np.zeros((n, 3), _f), np.zeros((n, 6), _f)
        self.l.refs_get_state(self.h, _ptr(pos), _ptr(orn), _ptr(lv), _ptr(av), _ptr(bb))
        return dict(pos=pos, orn=orn, linvel=lv, angvel=av, aabb=bb)

    def destroy_body(self, body):
        self.l.refs_destroy_body(self.h, C.c_uint32(body))

    def remove_exclusion(self, a, b):
        self.l.refs_remove_exclusion(self.h, C.c_uint32(a), C.c_uint32(b))

    def set_velocity(self, body, linvel, angvel):
        lv, av = _arr(linvel, _f), _arr(angvel, _f)
        self.l.refs_set_velocity(self.h, C.c_uint32(body), _ptr(lv), _ptr(av))

    def step_begin(self):
        """First half of step_simulation: broadphase, narrowphase, island manager (see refs_step_begin)."""
        self.l.refs_step_begin(self.h)

    def step_end(self):
        self.l.refs_step_end(self.h)

    def graph_order(self, max_adjacencies=None, max_tagged=None):
        """(adj_off, adj_nbr, tagged_pairs) as the restitution solver will walk them in the coming solver.update."""
        n = self.num_bodies
        cap_a = max_adjacencies or max(64, 32 * n)
        cap_t = max_tagged or max(64, 16 * n)
        off, nbr, tag, nt = np.zeros(n + 1, _u), np.zeros(cap_a, _u), np.zeros((cap_t, 2), _u), C.c_uint32(0)
        rc = self.l.refs_get_graph_order(self.h, _ptr(off), C.c_uint32(cap_a), _ptr(nbr), C.c_uint32(cap_t), _ptr(tag), C.byref(nt))
        if rc:
            raise RuntimeError("refs_get_graph_order: capacity")
        return off, nbr[:off[n]].copy(), tag[:nt.value].copy()

    def sleeping(self):
        out = np.zeros(self.num_bodies, _u)
        self.l.refs_get_sleeping(self.h, _ptr(out))
        return out.astype(bool)

    def inertia_inv(self):
        inv = np.zeros((self.num_bodies, 9), _f)
        self.l.refs_get_inertia_inv(self.h, _ptr(inv))
        return inv

    def contacts(self):
        """pairs (ordered: body[0], body[1]), num, pts (m, 4, 14): pivotA pivotB normal distance impulse_n impulse_t0 impulse_t1 lifetime."""
        m = int(self.l.refs_num_manifolds(self.h))
        pairs, num, pts = np.zeros((max(m, 1), 2), _u), np.zeros(max(m, 1), _u), np.zeros((max(m, 1), 4, 14), _f)
        got = int(self.l.refs_get_contacts(self.h, C.c_uint32(m), _ptr(pairs), _ptr(num), _ptr(pts)))
        return dict(pairs=pairs[:got], num=num[:got], pts=pts[:got])

    def islands(self):
        lab = np.zeros(self.num_bodies, _u)
        self.l.refs_get_islands(self.h, _ptr(lab))
        return lab

    def seed_manifolds(self, pairs, num, pts, att, lifetime):
        """Manifolds with given points (layout of World.upload_contacts: pts (m, 4, 18), slot 0 = list head), made by the
        reference's make_contact_manifold / create_contact_point and patched to the given values (refs_seed_manifolds)."""
        pairs = _arr(pairs, _u, (-1, 2))
        m = len(pairs)
        u = np.zeros((m, 4, 2), _u)
        u[:, :, 0], u[:, :, 1] = _arr(att, _u, (m, 4)), _arr(lifetime, _u, (m, 4))
        num, pts = _arr(num, _u, (m,)), _arr(pts, _f, (m, 4, 18))
        if self.l.refs_seed_manifolds(self.h, C.c_uint32(m), _ptr(pairs), _ptr(num), _ptr(pts), _ptr(u)):
            raise RuntimeError("refs_seed_manifolds: bad body index or point count")
        self.num_seeded = getattr(self, "num_seeded", 0) + m

    def narrowphase(self):
        """The reference's narrowphase::update(false) alone: contact distances, detect_collision, process_collision."""
        self.l.refs_narrowphase(self.h)

    def seeded(self):
        """The seeded manifolds in seeding order: dict(num, pts (m, 4, 18), att, lifetime), as World.contacts()."""
        m = getattr(self, "num_seeded", 0)
        num, pts, u = np.zeros(max(m, 1), _u), np.zeros((max(m, 1), 4, 18), _f), np.zeros((max(m, 1), 4, 2), _u)
        rc = self.l.refs_get_seeded(self.h, C.c_uint32(m), _ptr(num), _ptr(pts), _ptr(u))
        if rc:
            raise RuntimeError(f"refs_get_seeded: {rc}")
        return dict(num=num[:m], pts=pts[:m], att=u[:m, :, 0].copy(), lifetime=u[:m, :, 1].copy())

    def solver_order(self, max_contacts=None):
        """(hinge indices, (n, 3) contact rows as body0, body1, point index) of the last step, in the reference's row order."""
        cap_c = int(max_contacts or 4 * max(1, int(self.l.refs_num_manifolds(self.h))))
        cap_h = max(1, self.num_hinges)
        hi, ct = np.zeros(cap_h, _u), np.zeros((cap_c, 3), _u)
        nh, nc = C.c_uint32(0), C.c_uint32(0)
        if self.l.refs_get_solver_order(self.h, C.c_uint32(cap_h), _ptr(hi), C.byref(nh), C.c_uint32(cap_c), _ptr(ct), C.byref(nc)):
            raise RuntimeError("refs_get_solver_order: buffer too small")
        return hi[:nh.value].copy(), ct[:nc.value].copy()
