"""Python host adapter over the C ABI (include/b2d.h).

Mirrors the reference's lifecycle surface for the sequential stepper
(include/edyn/edyn.hpp:66-186, src/edyn/edyn.cpp:73-301):
    attach(config) -> World           edyn::attach(registry, config)
    make_rigidbody(world, def)        edyn::make_rigidbody(registry, def)
    make_hinge(world, a, b, ...)      edyn::make_constraint<hinge_constraint>(...) + set_axes
    exclude_collision(world, a, b)    edyn::exclude_collision
    insert_material_mixing(world, id0, id1, material)   edyn::insert_material_mixing
    step_simulation(world)            edyn::step_simulation(registry, t)   (one fixed step)
    update(world, dt_elapsed)         edyn::update(registry, time)         (accumulator, <= max_steps, presentation)
    set_paused(world, paused)         edyn::set_paused
    set_solver_velocity_iterations... edyn::set_solver_velocity_iterations
All compute happens in libb2d.so on the GPU; nothing here touches oracle/.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import B2DError, Bodies, BodyPatch, Config, Stats
from .rigidbody import MATERIAL_UNASSIGNED, Material, RigidBodyDef, bodies_soa

f32, u32 = np.float32, np.uint32

PH_BROAD, PH_NARROW, PH_ISLANDS, PH_SOLVE, PH_ALL = 1, 2, 4, 8, 15
FLAG_RECOLOR_EACH_STEP = 1
FLAG_RESTITUTION_SOLVER = 4     # the reference's default restitution solver (8 x 3 iterations) instead of restitution through the row rhs
FLAG_SLEEPING = 2                # island sleeping; off = every body is sleeping_disabled (benchmark configurations)
RAY_MISS = 0xFFFFFFFF            # B2D_RAY_MISS
RAY_FEATURE_NONE = 0xFFFFFFFF    # B2D_RAY_FEATURE_NONE
RAY_CAPSULE_SIDE = 2             # B2D_RAY_CAPSULE_SIDE


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(x, dt, shape=None):
    a = np.ascontiguousarray(np.asarray(x, dtype=dt))
    return a.reshape(shape) if shape is not None else a


class World:
    """One device-resident world (one entt::registry's worth of rigid bodies)."""

    def __init__(self, max_bodies, max_manifolds=None, max_hinges=0, device=0, fixed_dt=1.0 / 60,
                 velocity_iterations=8, position_iterations=3, flags=0, gravity=(0.0, -9.8, 0.0)):
        self.l = _lib.lib()
        if max_manifolds is None:
            max_manifolds = max(1024, 8 * max_bodies)
        self.cfg = Config(device, max_bodies, max_manifolds, max_hinges, fixed_dt, velocity_iterations,
                          position_iterations, flags)
        h = self.l.b2d_create(C.byref(self.cfg))
        if not h:
            raise B2DError(self.l.b2d_last_error(None).decode())
        self.h = C.c_void_p(h)
        self.gravity = tuple(gravity)
        self.fixed_dt = fixed_dt
        self.num_bodies = 0
        self.num_hinges = 0
        self._defs, self._hinges = [], []
        self._excl_set, self._excl_log = set(), []          # collision_exclusion, as unordered pairs (see `exclusions`)
        self.removed = np.zeros(max_bodies, bool)
        self.hinge_alive = np.zeros(0, bool)
        self.max_manifolds = max_manifolds
        self._accum = 0.0
        self.max_steps_per_update = 10          # settings.max_steps_per_update
        self.paused = False                     # settings.paused

    # -- lifecycle
    def close(self):
        if getattr(self, "h", None):
            self.l.b2d_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise B2DError(f"b2d error {rc}: {self.l.b2d_last_error(self.h).decode()}")

    # -- construction
    def add_bodies(self, soa: dict) -> int:
        n = len(soa["kind"])
        keep = dict(pos=_c(soa["pos"], f32, (n, 3)), orn=_c(soa["orn"], f32, (n, 4)), linvel=_c(soa["linvel"], f32, (n, 3)),
                    angvel=_c(soa["angvel"], f32, (n, 3)), inv_mass=_c(soa["inv_mass"], f32, (n,)),
                    inv_inertia=_c(soa["inv_inertia"], f32, (n, 9)), gravity=_c(soa["gravity"], f32, (n, 3)),
                    kind=_c(soa["kind"], u32, (n,)), shape_kind=_c(soa["shape_kind"], u32, (n,)),
                    shape_params=_c(soa["shape_params"], f32, (n, 4)), friction=_c(soa["friction"], f32, (n,)),
                    restitution=_c(soa["restitution"], f32, (n,)))
        grp = _c(soa["group"], np.uint64, (n,)) if soa.get("group") is not None else None
        msk = _c(soa["mask"], np.uint64, (n,)) if soa.get("mask") is not None else None
        mat = _c(soa["material"], u32, (n,)) if soa.get("material") is not None else None     # absent: all unassigned
        pre = _c(soa["presentation"], u32, (n,)) if soa.get("presentation") is not None else None     # absent: none
        b = Bodies(n, *[_p(keep[k]) for k in ("pos", "orn", "linvel", "angvel", "inv_mass", "inv_inertia", "gravity",
                                               "kind", "shape_kind", "shape_params", "friction", "restitution")],
                   _p(grp), _p(msk), _p(mat), _p(pre))
        first = C.c_uint32(0)
        self._check(self.l.b2d_add_bodies(self.h, C.byref(b), C.byref(first)))
        self.num_bodies += n
        # host copy of the immutable definition (mass, shape, material, filter): what island migration ships to a peer
        keep["group"] = grp if grp is not None else np.full(n, ~np.uint64(0), np.uint64)
        keep["mask"] = msk if msk is not None else np.full(n, ~np.uint64(0), np.uint64)
        keep["has_filter"] = np.full(n, grp is not None and msk is not None, bool)
        keep["material"] = mat if mat is not None else np.full(n, MATERIAL_UNASSIGNED, u32)
        keep["presentation"] = pre if pre is not None else np.zeros(n, u32)
        self._defs.append(keep)
        return first.value

    def wake_bodies(self, ids=None):
        """edyn::wake_up_entity; ids=None wakes everything."""
        if ids is None:
            self._check(self.l.b2d_wake_bodies(self.h, None, C.c_uint32(0)))
        else:
            ids = _c(ids, u32)
            self._check(self.l.b2d_wake_bodies(self.h, _p(ids), C.c_uint32(len(ids))))

    def sleeping(self):
        out = np.zeros(max(1, self.num_bodies), u32)
        self._check(self.l.b2d_download_sleeping(self.h, _p(out)))
        return out[:self.num_bodies].astype(bool)

    def body_defs(self, ids):
        """Definition arrays (as passed to add_bodies) of bodies `ids`; state fields are the creation-time ones."""
        ids = np.asarray(ids, np.int64)
        if len(self._defs) > 1:
            self._defs = [{k: np.concatenate([d[k] for d in self._defs]) for k in self._defs[0]}]
        d = self._defs[0]
        return {k: v[ids].copy() for k, v in d.items()}

    def remove_bodies(self, ids):
        """registry.destroy(body): the bodies, their manifolds and their joints leave the simulation; ids are not reused."""
        ids = _c(ids, u32)
        self._check(self.l.b2d_remove_bodies(self.h, _p(ids), C.c_uint32(len(ids))))
        self.removed[ids] = True
        if self._hinges:
            h = self.hinge_defs()
            self.hinge_alive &= ~(self.removed[h["a"]] | self.removed[h["b"]])

    def add_hinges(self, a, b, pivot_a, pivot_b, axis_a, axis_b):
        n = len(a)
        arr = [_c(a, u32), _c(b, u32), _c(pivot_a, f32, (n, 3)), _c(pivot_b, f32, (n, 3)), _c(axis_a, f32, (n, 3)), _c(axis_b, f32, (n, 3))]
        self._check(self.l.b2d_add_hinges(self.h, C.c_uint32(n), *[_p(x) for x in arr]))
        self.num_hinges += n
        self._hinges.append(dict(zip(("a", "b", "pivot_a", "pivot_b", "axis_a", "axis_b"), arr)))
        self.hinge_alive = np.concatenate([self.hinge_alive, np.ones(n, bool)])

    def hinge_defs(self):
        if len(self._hinges) > 1:
            self._hinges = [{k: np.concatenate([h[k] for h in self._hinges]) for k in self._hinges[0]}]
        return self._hinges[0] if self._hinges else None

    def add_exclusions(self, a, b):
        a, b = _c(a, u32), _c(b, u32)
        self._check(self.l.b2d_add_exclusions(self.h, C.c_uint32(len(a)), _p(a), _p(b)))
        self._excl_log.append((True, np.minimum(a, b), np.maximum(a, b)))

    def remove_exclusions(self, a, b):
        a, b = _c(a, u32), _c(b, u32)
        self._check(self.l.b2d_remove_exclusions(self.h, C.c_uint32(len(a)), _p(a), _p(b)))
        self._excl_log.append((False, np.minimum(a, b), np.maximum(a, b)))

    @property
    def exclusions(self):
        """collision_exclusion as a set of unordered (lo, hi) pairs; materialised only when somebody asks (a million-link
        scene registers ~800 k exclusions that nobody on the host ever reads)."""
        for add, lo, hi in self._excl_log:
            pairs = set(zip(lo.tolist(), hi.tolist()))
            if add:
                self._excl_set |= pairs
            else:
                self._excl_set -= pairs
        self._excl_log = []
        return self._excl_set

    # -- stepping
    def step(self, n=1):
        self._check(self.l.b2d_step(self.h, C.c_uint32(n)))

    def run_phases(self, mask):
        self._check(self.l.b2d_run_phases(self.h, C.c_uint32(mask)))

    def sync(self):
        self._check(self.l.b2d_sync(self.h))

    @property
    def stream(self):
        return self.l.b2d_stream(self.h)

    # -- state
    def upload_state(self, pos, orn, linvel, angvel):
        n = self.num_bodies
        a = [_c(pos, f32, (n, 3)), _c(orn, f32, (n, 4)), _c(linvel, f32, (n, 3)), _c(angvel, f32, (n, 3))]
        self._check(self.l.b2d_upload_state(self.h, *[_p(x) for x in a]))
        self._keep = a

    def upload_bodies(self, ids, **comp):
        """registry.patch on a subset of bodies (b2d_upload_bodies): comp = pos / orn / linvel / angvel / inv_mass /
        inv_inertia / gravity / friction / restitution / kind / material, each packed per listed body; the rest stays
        untouched.  material: ids (MATERIAL_NONE for a sensor; a body cannot change between sensor and non-sensor)."""
        ids = _c(ids, u32)
        n = len(ids)
        shapes = dict(pos=(n, 3), orn=(n, 4), linvel=(n, 3), angvel=(n, 3), inv_mass=(n,), inv_inertia=(n, 9),
                      gravity=(n, 3), friction=(n,), restitution=(n,))
        unknown = set(comp) - set(shapes) - {"kind", "material"}
        if unknown:
            raise B2DError(f"upload_bodies: unknown components {sorted(unknown)}")
        keep = {k: _c(v, f32, shapes[k]) for k, v in comp.items() if k in shapes}
        for k in ("kind", "material"):
            if k in comp:
                keep[k] = _c(comp[k], u32, (n,))
        patch = BodyPatch(*[_p(keep.get(k)) for k in ("pos", "orn", "linvel", "angvel", "inv_mass", "inv_inertia", "gravity",
                                                      "friction", "restitution", "kind", "material")])
        self._check(self.l.b2d_upload_bodies(self.h, C.c_uint32(n), _p(ids), C.byref(patch)))

    def set_material_mixing(self, id0, id1, friction, restitution):
        """material_mix_table::insert for the unordered id pairs (id0[i], id1[i]); applies to contact points created later."""
        a, b = _c(id0, u32).reshape(-1), _c(id1, u32).reshape(-1)
        f, r = _c(friction, f32, (len(a),)), _c(restitution, f32, (len(a),))
        self._check(self.l.b2d_set_material_mixing(self.h, C.c_uint32(len(a)), _p(a), _p(b), _p(f), _p(r)))

    def remove_material_mixing(self, id0, id1):
        """material_mix_table::remove for the unordered id pairs (id0[i], id1[i]); absent pairs are ignored."""
        a, b = _c(id0, u32).reshape(-1), _c(id1, u32).reshape(-1)
        self._check(self.l.b2d_remove_material_mixing(self.h, C.c_uint32(len(a)), _p(a), _p(b)))

    def download_state(self, aabb=True, inv_IW=False, out=None):
        n = self.num_bodies
        o = out or dict(pos=np.zeros((n, 3), f32), orn=np.zeros((n, 4), f32), linvel=np.zeros((n, 3), f32), angvel=np.zeros((n, 3), f32))
        if aabb and "aabb" not in o:
            o["aabb"] = np.zeros((n, 6), f32)
        if inv_IW and "inv_IW" not in o:
            o["inv_IW"] = np.zeros((n, 9), f32)
        self._check(self.l.b2d_download_state(self.h, _p(o["pos"]), _p(o["orn"]), _p(o["linvel"]), _p(o["angvel"]),
                                              _p(o.get("aabb")), _p(o.get("inv_IW"))))
        return o

    def pairs(self):
        cap = self.max_manifolds
        p = np.zeros((cap, 2), u32)
        n = C.c_uint32(0)
        self._check(self.l.b2d_download_pairs(self.h, C.c_uint32(cap), _p(p), C.byref(n)))
        return p[:n.value].copy()

    def contacts(self):
        m = C.c_uint32(0)
        self._check(self.l.b2d_num_manifolds(self.h, C.byref(m)))
        cap = max(1, m.value)
        pairs, num = np.zeros((cap, 2), u32), np.zeros(cap, u32)
        pts, u = np.zeros((cap, 4, 18), f32), np.zeros((cap, 4, 2), u32)
        n = C.c_uint32(0)
        self._check(self.l.b2d_download_contacts(self.h, C.c_uint32(cap), _p(pairs), _p(num), _p(pts), _p(u), C.byref(n)))
        k = n.value
        return dict(pairs=pairs[:k], num=num[:k], pts=pts[:k], att=u[:k, :, 0].copy(), lifetime=u[:k, :, 1].copy())

    def upload_contacts(self, pairs, num, pts, att, lifetime=None):
        pairs = _c(pairs, u32, (-1, 2))
        m = len(pairs)
        num, pts = _c(num, u32, (m,)), _c(pts, f32, (m, 4, 18))
        u = np.zeros((m, 4, 2), u32)
        u[:, :, 0] = _c(att, u32, (m, 4))
        if lifetime is not None:
            u[:, :, 1] = _c(lifetime, u32, (m, 4))
        self._check(self.l.b2d_upload_contacts(self.h, C.c_uint32(m), _p(pairs), _p(num), _p(pts), _p(u)))

    def islands(self):
        lab = np.zeros(self.num_bodies, u32)
        self._check(self.l.b2d_download_islands(self.h, _p(lab)))
        return lab

    def solver_order(self):
        hi = np.zeros(max(1, self.num_hinges), u32)
        pr = np.zeros((self.max_manifolds, 2), u32)
        nh, nm = C.c_uint32(len(hi)), C.c_uint32(len(pr))
        self._check(self.l.b2d_download_solver_order(self.h, _p(hi), C.byref(nh), _p(pr), C.byref(nm)))
        return hi[:nh.value].copy(), pr[:nm.value].copy()

    def hinge_impulses(self):
        imp = np.zeros((max(1, self.num_hinges), 5), f32)
        self._check(self.l.b2d_download_hinge_impulses(self.h, _p(imp)))
        return imp[:self.num_hinges]

    # -- presentation transforms (include/b2d.h, b2d_update_presentation: semantics)
    def update_presentation(self, interpolation_dt):
        """update_presentation: present transforms of the awake dynamic bodies with presentation = state extrapolated
        by interpolation_dt seconds (enqueued on the world's stream)."""
        self._check(self.l.b2d_update_presentation(self.h, C.c_float(interpolation_dt)))

    def snap_presentation(self):
        """snap_presentation: present transforms = position / orientation for every body with presentation."""
        self._check(self.l.b2d_snap_presentation(self.h))

    def presentation(self):
        """(present_position (n, 3), present_orientation (n, 4)) float32; bodies without presentation report their
        position / orientation."""
        n = self.num_bodies
        pos, orn = np.zeros((max(1, n), 3), f32), np.zeros((max(1, n), 4), f32)
        self._check(self.l.b2d_download_presentation(self.h, _p(pos), _p(orn)))
        return pos[:n], orn[:n]

    def presentation_device(self, pos_ptr, orn_ptr):
        """Enqueue the copy of presentation() into integer DEVICE addresses (n x 3 and n x 4 float32; 0 = skip that one)."""
        v = lambda x: C.c_void_p(x or None)       # noqa: E731
        self._check(self.l.b2d_download_presentation_device(self.h, v(pos_ptr), v(orn_ptr)))

    # -- queries (include/b2d.h, b2d_raycast: semantics)
    def raycast(self, p0, p1, ignore=None, ignore_body=None) -> dict:
        """edyn::raycast for n segments at once: p0, p1 are (n, 3).  ignore: body ids no segment may hit; ignore_body: one id
        per segment (B2D_RAY_MISS for none).  Returns body (n,) uint32 (RAY_MISS on a miss), fraction (n,) float32 (FLT_MAX on a
        miss), normal (n, 3) float32 and feature (n,) uint32."""
        a, b = _c(p0, f32), _c(p1, f32)
        a, b = a.reshape(-1, 3), b.reshape(-1, 3)
        n = len(a)
        if b.shape != a.shape:
            raise ValueError("raycast: p0 and p1 must have the same (n, 3) shape")
        ign = _c(ignore if ignore is not None else [], u32).reshape(-1)
        ib = _c(ignore_body, u32, (n,)) if ignore_body is not None else None
        out = dict(body=np.empty(n, u32), fraction=np.empty(n, f32), normal=np.empty((n, 3), f32), feature=np.empty(n, u32))
        self._check(self.l.b2d_raycast(self.h, C.c_uint32(n), _p(a), _p(b), _p(ib), _p(ign) if len(ign) else None,
                                       C.c_uint32(len(ign)), _p(out["body"]), _p(out["fraction"]), _p(out["normal"]), _p(out["feature"])))
        return out

    def raycast_device(self, n, p0_ptr, p1_ptr, body_ptr=0, fraction_ptr=0, normal_ptr=0, feature_ptr=0, ignore=None,
                       ignore_body_ptr=0):
        """Enqueue a raycast of n segments on the world's stream: every argument but `ignore` (host body ids) is an integer
        DEVICE address (0 = none; p0 / p1 are n x 3 float32, normal n x 3 float32, the rest n words)."""
        ign = _c(ignore if ignore is not None else [], u32).reshape(-1)
        v = lambda x: C.c_void_p(x or None)       # noqa: E731
        self._check(self.l.b2d_raycast_device(self.h, C.c_uint32(n), v(p0_ptr), v(p1_ptr), v(ignore_body_ptr),
                                              _p(ign) if len(ign) else None, C.c_uint32(len(ign)), v(body_ptr),
                                              v(fraction_ptr), v(normal_ptr), v(feature_ptr)))

    def device_bounds(self, device_ptr):
        """Enqueue the dynamic-AABB bounds reduction into 8 floats (min, max, speed, 0) at `device_ptr` (an int device address)."""
        self._check(self.l.b2d_device_bounds(self.h, C.c_void_p(device_ptr)))

    # -- multi-GPU hand-over (device buffers are passed as integer addresses; the transport belongs to the caller)
    def set_halo_margin(self, margin):
        self._check(self.l.b2d_set_halo_margin(self.h, C.c_float(margin)))

    def set_entities(self, first, entity):
        e = _c(entity, u32)
        self._check(self.l.b2d_set_entities(self.h, C.c_uint32(first), C.c_uint32(len(e)), _p(e)))

    def entities(self):
        e = np.zeros(max(1, self.num_bodies), u32)
        self._check(self.l.b2d_download_entities(self.h, _p(e)))
        return e[:self.num_bodies]

    def island_halo(self, boxes_ptr, nboxes, self_rank, peer_mask, records_ptr, capacity, count_ptr):
        self._check(self.l.b2d_island_halo(self.h, C.c_void_p(boxes_ptr), C.c_uint32(nboxes), C.c_uint32(self_rank),
                                           C.c_uint64(peer_mask), C.c_void_p(records_ptr), C.c_uint32(capacity), C.c_void_p(count_ptr)))

    def handover_plan(self, records_ptr, my_begin, my_end, nranks):
        counts = np.zeros((nranks, 4), u32)
        self._check(self.l.b2d_handover_plan(self.h, C.c_void_p(records_ptr), C.c_uint32(my_begin), C.c_uint32(my_end),
                                             C.c_uint32(nranks), _p(counts)))
        return counts

    def handover_bytes(self, counts4):
        c = _c(counts4, u32, (4,))
        return int(self.l.b2d_handover_bytes(_p(c)))

    def handover_pack(self, dst, blob_ptr, capacity):
        self._check(self.l.b2d_handover_pack(self.h, C.c_uint32(dst), C.c_void_p(blob_ptr), C.c_uint64(capacity)))

    def handover_unpack(self, blob_ptr, nbytes):
        c = np.zeros(4, u32)
        self._check(self.l.b2d_handover_unpack(self.h, C.c_void_p(blob_ptr), C.c_uint64(nbytes), _p(c)))
        self.num_bodies += int(c[0])
        self.num_hinges += int(c[2])
        self.hinge_alive = np.concatenate([self.hinge_alive, np.ones(int(c[2]), bool)])
        return c

    def set_timing(self, enabled=True):
        self._check(self.l.b2d_set_timing(self.h, C.c_int(1 if enabled else 0)))

    def reset_timers(self):
        self._check(self.l.b2d_reset_timers(self.h))

    def debug_tiles(self):
        """Development aid: island tiles of the last step."""
        out = np.zeros(6, np.uint32)
        self._check(self.l.b2d_debug_tiles(self.h, _p(out)))
        return dict(zip(("tiles", "tiled_manifolds", "tiled_hinges", "active_manifolds", "active_hinges", "max_bodies_per_tile"), out.tolist()))

    def debug_newcount(self):
        """Development aid: the new pairs the last broadphase counted per body (b2d_debug_newcount)."""
        out = np.zeros(max(1, self.num_bodies), np.uint32)
        self._check(self.l.b2d_debug_newcount(self.h, _p(out)))
        return out[:self.num_bodies]

    def debug_tile_map(self):
        """Development aid: the island-tile packing of the last rebuild (b2d_debug_tile_map).  Per body its tile and record
        slot (0xFFFFFFFF / 0xFFFF: not tiled); per tile its body count and its [c0, c1) / [h0, h1) ranges into
        `pairs` (the body pairs of the tiled manifolds) and `hinges` (the tiled hinge ids)."""
        cnt = np.zeros(5, u32)
        self._check(self.l.b2d_debug_tile_map(self.h, _p(cnt), None, None, None, None, None))
        nt, nt2, nc, nh, cap = (int(x) for x in cnt)
        n = max(1, self.cfg.max_bodies)
        btile, bslot = np.zeros(n, u32), np.zeros(n, u32)
        tiles, pairs, hinges = np.zeros((5, max(1, nt)), u32), np.zeros((max(1, nc), 2), u32), np.zeros(max(1, nh), u32)
        self._check(self.l.b2d_debug_tile_map(self.h, _p(cnt), _p(btile), _p(bslot), _p(tiles), _p(pairs), _p(hinges)))
        return dict(ntiles=nt, ntiles2=nt2, ntiled=nc, nhtiled=nh, max_tiles=cap, btile=btile[:self.num_bodies],
                    bslot=bslot[:self.num_bodies], tile_nb=tiles[0, :nt].copy(), tile_c0=tiles[1, :nt].copy(),
                    tile_c1=tiles[2, :nt].copy(), tile_h0=tiles[3, :nt].copy(), tile_h1=tiles[4, :nt].copy(),
                    pairs=pairs[:nc], hinges=hinges[:nh])

    def stats(self) -> dict:
        s = Stats()
        self._check(self.l.b2d_get_stats(self.h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in Stats._fields_}


# ----------------------------------------------------------------------------- edyn-style free functions

def attach(max_bodies, **kw) -> World:
    """edyn::attach(registry, init_config) for execution_mode::sequential (src/edyn/edyn.cpp:73-141)."""
    return World(max_bodies, **kw)


def detach(world: World):
    world.close()


def make_rigidbody(world: World, definition) -> int:
    """edyn::make_rigidbody (src/edyn/util/rigidbody.cpp:47-185).  Accepts one def or a list (batch_rigidbodies)."""
    defs = [definition] if isinstance(definition, RigidBodyDef) else list(definition)
    return world.add_bodies(bodies_soa(defs, world.gravity))


def make_hinge(world: World, body_a, body_b, pivot_a, pivot_b, axis_a, axis_b):
    """edyn::make_constraint<hinge_constraint> + pivot + set_axes (src/edyn/constraints/hinge_constraint.cpp:11-17)."""
    world.add_hinges([body_a], [body_b], [pivot_a], [pivot_b], [axis_a], [axis_b])
    return world.num_hinges - 1


def exclude_collision(world: World, a, b):
    """edyn::exclude_collision (src/edyn/util/exclude_collision.cpp)."""
    world.add_exclusions([a], [b])


def insert_material_mixing(world: World, id0: int, id1: int, material: Material):
    """edyn::insert_material_mixing (src/edyn/util/insert_material_mixing.cpp:9-22): friction and restitution of the contact
    points created from now on between bodies of material ids id0 and id1 (either order)."""
    world.set_material_mixing([id0], [id1], [material.friction], [material.restitution])


def remove_collision_exclusion(world: World, a, b):
    """edyn::remove_collision_exclusion."""
    world.remove_exclusions([a], [b])


def clear_collision_exclusion(world: World, e):
    """edyn::clear_collision_exclusion: drops every exclusion body `e` takes part in."""
    mine = [p for p in world.exclusions if e in p]
    if mine:
        world.remove_exclusions([p[0] for p in mine], [p[1] for p in mine])


class RaycastResult:
    """edyn::raycast_result (include/edyn/collision/raycast.hpp:103-136): entity is the body id (None on a miss), info the
    feature (box face, capsule hemisphere index or RAY_CAPSULE_SIDE; None for spheres, planes and misses)."""

    def __init__(self, entity, fraction, normal, info):
        self.entity, self.fraction, self.normal, self.info = entity, fraction, normal, info

    def __repr__(self):
        return f"RaycastResult(entity={self.entity}, fraction={self.fraction}, normal={self.normal}, info={self.info})"


def raycast(world: World, p0, p1, ignore_entities=()) -> RaycastResult:
    """edyn::raycast(registry, p0, p1, ignore_entities) (src/edyn/collision/raycast.cpp:20-56) for one segment."""
    r = world.raycast(np.asarray(p0, f32).reshape(1, 3), np.asarray(p1, f32).reshape(1, 3), ignore=list(ignore_entities))
    body, feat = int(r["body"][0]), int(r["feature"][0])
    return RaycastResult(None if body == RAY_MISS else body, float(r["fraction"][0]), r["normal"][0].copy(),
                         None if feat == RAY_FEATURE_NONE else feat)


def step_simulation(world: World):
    """edyn::step_simulation(registry, t): exactly one fixed step (stepper_sequential.cpp:121-147)."""
    world.step(1)


def set_paused(world: World, paused: bool):
    """edyn::set_paused (stepper_sequential.cpp:148-151): the accumulator restarts from zero."""
    world.paused = bool(paused)
    world._accum = 0.0


def update(world: World, elapsed: float) -> int:
    """edyn::update(registry, time): accumulate wall time, run floor(acc / fixed_dt) steps capped by
    max_steps_per_update (stepper_sequential.cpp:45-65), then update_presentation (:104-105).  While paused it only snaps
    the presentation (:37-43).  Returns the number of steps taken.

    The reference's interpolation_dt = min(float(time - fixed_dt - sim_time), fixed_dt) with sim_time = time - acc;
    with elapsed times instead of timestamps that is min(float(acc - fixed_dt), fixed_dt): the present transforms lag
    one fixed step behind the wall clock, so that frames between two steps move smoothly."""
    if world.paused:
        world.snap_presentation()
        return 0
    world._accum += elapsed
    n = int(world._accum / world.fixed_dt)
    world._accum -= n * world.fixed_dt
    n = min(n, world.max_steps_per_update)
    if n:
        world.step(n)
    fixed_dt = f32(world.fixed_dt)
    world.update_presentation(min(f32(world._accum - float(fixed_dt)), fixed_dt))
    return n
