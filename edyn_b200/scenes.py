"""Synthetic scenes of BASELINE.json's configs (concrete inputs: SURVEY.md section 8d), as component arrays.

Every generator returns a dict:
    bodies      b2d_bodies-style SoA (see rigidbody.bodies_soa)
    hinges      None or dict(a, b, pivot_a, pivot_b, axis_a, axis_b)
    exclusions  None or (a, b)
    settings    dict(velocity_iterations, position_iterations)
    name, dynamic (number of dynamic bodies)
Deterministic: the only randomness is numpy's default_rng(1234) for orientations / jitter.
"""
import numpy as np

from .rigidbody import (DYNAMIC, STATIC, SHAPE_BOX, SHAPE_CAPSULE, SHAPE_PLANE, SHAPE_SPHERE, Shape,
                        inverse_matrix_symmetric, moment_of_inertia)

f32 = np.float32
GRAVITY = (0.0, -9.8, 0.0)


def _assemble(pos, orn, shape_kind, shape_params, kind, mass=1.0, friction=0.5, restitution=0.0):
    n = len(kind)
    pos = np.asarray(pos, f32).reshape(n, 3)
    orn = np.asarray(orn, f32).reshape(n, 4)
    shape_kind = np.asarray(shape_kind, np.uint32)
    shape_params = np.asarray(shape_params, f32).reshape(n, 4)
    kind = np.asarray(kind, np.uint32)
    mass = np.broadcast_to(np.asarray(mass, f32), (n,)).copy()
    dyn = kind == DYNAMIC
    inv_mass = np.zeros(n, f32)
    inv_mass[dyn] = f32(1) / mass[dyn]
    inv_inertia = np.zeros((n, 9), f32)
    # one inertia per distinct (shape, mass)
    keys = np.concatenate([shape_kind[:, None].astype(f32), shape_params, mass[:, None]], axis=1)
    uniq, inverse = np.unique(keys[dyn], axis=0, return_inverse=True)
    table = np.zeros((len(uniq), 9), f32)
    for i, k in enumerate(uniq):
        table[i] = inverse_matrix_symmetric(moment_of_inertia(Shape(int(k[0]), tuple(float(x) for x in k[1:5])), k[5])).reshape(9)
    inv_inertia[dyn] = table[inverse.reshape(-1)]
    gravity = np.zeros((n, 3), f32)
    gravity[dyn] = GRAVITY
    return dict(pos=pos, orn=orn, linvel=np.zeros((n, 3), f32), angvel=np.zeros((n, 3), f32), inv_mass=inv_mass,
                inv_inertia=inv_inertia, gravity=gravity, kind=kind, shape_kind=shape_kind, shape_params=shape_params,
                friction=np.broadcast_to(np.asarray(friction, f32), (n,)).copy(),
                restitution=np.broadcast_to(np.asarray(restitution, f32), (n,)).copy(),
                group=np.full(n, 0xFFFFFFFFFFFFFFFF, np.uint64), mask=np.full(n, 0xFFFFFFFFFFFFFFFF, np.uint64))


def _planes(specs):
    """specs: list of (normal, constant)."""
    n = len(specs)
    pos = np.zeros((n, 3), f32)
    orn = np.tile(np.array([0, 0, 0, 1], f32), (n, 1))
    params = np.array([[s[0][0], s[0][1], s[0][2], s[1]] for s in specs], f32)
    return pos, orn, np.full(n, SHAPE_PLANE, np.uint32), params, np.full(n, STATIC, np.uint32)


def _join(dyn, planes):
    return [np.concatenate([np.asarray(a), np.asarray(b)]) for a, b in zip(dyn, planes)]


def _identity(n):
    return np.tile(np.array([0, 0, 0, 1], f32), (n, 1))


def _random_quats(n, rng):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q.astype(f32)


def hello_world():
    """Config 1: one dynamic box dropped on a static plane (hello_world.cpp:17-39 restated with a box + plane)."""
    a = 0.7 * np.pi
    orn = np.array([[0, 0, np.sin(a / 2), np.cos(a / 2)]], f32)        # quaternion_axis_angle(z, 0.7 pi)
    dyn = (np.array([[0, 3, 0]], f32), orn, np.array([SHAPE_BOX], np.uint32), np.array([[0.5, 0.5, 0.5, 0]], f32),
           np.array([DYNAMIC], np.uint32))
    arrs = _join(dyn, _planes([((0, 1, 0), 0.0)]))
    b = _assemble(*arrs, mass=np.array([10, 1], f32), friction=0.8)
    return dict(name="hello_world", bodies=b, hinges=None, exclusions=None, dynamic=1,
                settings=dict(velocity_iterations=8, position_iterations=3))


def boxes_on_plane(side=16, jitter=0.0):
    """Config 2: side^3 unit boxes dropped on a plane (4 096 at side = 16), 10 velocity iterations."""
    i, k, j = np.meshgrid(np.arange(side), np.arange(side), np.arange(side), indexing="ij")
    pos = np.stack([1.1 * i.ravel(), 0.6 + 1.1 * k.ravel(), 1.1 * j.ravel()], axis=1).astype(f32)
    n = len(pos)
    if jitter:
        pos += np.random.default_rng(1234).uniform(-jitter, jitter, size=pos.shape).astype(f32)
    dyn = (pos, _identity(n), np.full(n, SHAPE_BOX, np.uint32), np.tile(np.array([0.5, 0.5, 0.5, 0], f32), (n, 1)),
           np.full(n, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _planes([((0, 1, 0), 0.0)])))
    return dict(name=f"boxes_{n}", bodies=b, hinges=None, exclusions=None, dynamic=n,
                settings=dict(velocity_iterations=10, position_iterations=3))


def approaching_stacks(height=2, gap=0.6, speed=3.0):
    """Two stacks of unit boxes sliding towards each other on a plane: two islands that merge into one after a few
    steps.  Exercises the cross-GPU case of SURVEY 8e (an island changes rank) and manifold / warm-start transfer."""
    ys = 0.5 + np.arange(height, dtype=f32)
    left = np.stack([np.zeros(height, f32), ys, np.zeros(height, f32)], axis=1)
    right = left + np.array([1.0 + gap, 0, 0], f32)
    pos = np.concatenate([left, right]).astype(f32)
    n = len(pos)
    dyn = (pos, _identity(n), np.full(n, SHAPE_BOX, np.uint32), np.tile(np.array([0.5, 0.5, 0.5, 0], f32), (n, 1)),
           np.full(n, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _planes([((0, 1, 0), 0.0)])))
    b["linvel"][:height, 0] = speed
    b["linvel"][height:n, 0] = -speed
    return dict(name=f"approaching_stacks_{height}", bodies=b, hinges=None, exclusions=None, dynamic=n,
                settings=dict(velocity_iterations=10, position_iterations=3))


def sleep_and_wake(drop_height=55.0):
    """A box resting on a plane (asleep after 2 s) and a second one dropped from `drop_height` that lands on it ~1.3 s
    later and wakes it; both then fall asleep together.  Exercises island sleeping (island_manager.cpp:541-623)."""
    pos = np.array([[0, 0.5, 0], [0.2, drop_height, 0.1]], f32)
    dyn = (pos, _identity(2), np.full(2, SHAPE_BOX, np.uint32), np.tile(np.array([0.5, 0.5, 0.5, 0], f32), (2, 1)),
           np.full(2, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _planes([((0, 1, 0), 0.0)])))
    return dict(name="sleep_and_wake", bodies=b, hinges=None, exclusions=None, dynamic=2,
                settings=dict(velocity_iterations=10, position_iterations=3))


def _box_walls(x1, z1, height):
    """Floor plane y = 0 plus four static wall slabs around [-0.5, x1] x [-0.5, z1].

    SURVEY.md section 8d asks for five planes.  The walls are static BOXES instead because the reference's sphere-plane
    routine computes pivotB as `d - normal * l - center` with d already relative to `center`
    (src/edyn/collision/collide/collide_sphere_plane.cpp:8-17), i.e. off by 2 * normal * constant: fine for the floor
    (constant 0), but for an offset wall the position solver then sees metres of penetration and teleports the
    sphere.  Both the oracle and the device path reproduce that arithmetic bit for bit, so the benchmark scenes simply
    do not contain offset planes."""
    t = 1.0                                             # wall half thickness
    hy = 0.5 * height + 1.0
    cx, cz = 0.5 * (x1 - 0.5), 0.5 * (z1 - 0.5)
    hx, hz = 0.5 * (x1 + 0.5) + 2 * t, 0.5 * (z1 + 0.5) + 2 * t
    pos = np.array([[0, 0, 0], [-0.5 - t, hy, cz], [x1 + t, hy, cz], [cx, hy, -0.5 - t], [cx, hy, z1 + t]], f32)
    params = np.array([[0, 1, 0, 0], [t, hy, hz, 0], [t, hy, hz, 0], [hx, hy, t, 0], [hx, hy, t, 0]], f32)
    kinds = np.array([SHAPE_PLANE, SHAPE_BOX, SHAPE_BOX, SHAPE_BOX, SHAPE_BOX], np.uint32)
    return pos, _identity(5), kinds, params, np.full(5, STATIC, np.uint32)


def spheres_in_box(nx=64, ny=16, nz=64, jitter=0.01):
    """Config 3: nx*ny*nz spheres (65 536 default) of radius 0.25 inside a floor plane + four static walls, 10 iterations."""
    i, k, j = np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij")
    pos = np.stack([0.55 * i.ravel(), 0.3 + 0.55 * k.ravel(), 0.55 * j.ravel()], axis=1).astype(f32)
    n = len(pos)
    if jitter:
        pos += np.random.default_rng(1234).uniform(-jitter, jitter, size=pos.shape).astype(f32)
    dyn = (pos, _identity(n), np.full(n, SHAPE_SPHERE, np.uint32), np.tile(np.array([0.25, 0, 0, 0], f32), (n, 1)),
           np.full(n, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _box_walls(0.55 * (nx - 1) + 0.85, 0.55 * (nz - 1) + 0.85, 0.55 * ny + 1.0)))
    return dict(name=f"spheres_{n}", bodies=b, hinges=None, exclusions=None, dynamic=n,
                settings=dict(velocity_iterations=10, position_iterations=3))


def mixed_pile(side=64, jitter=0.01):
    """Config 4: side^3 (262 144 default) boxes / spheres / capsules with random orientations, friction 0.5,
    restitution 0.2 (through the row rhs: restitution iterations = 0 on both sides), 20 velocity iterations."""
    rng = np.random.default_rng(1234)
    i, k, j = np.meshgrid(np.arange(side), np.arange(side), np.arange(side), indexing="ij")
    pos = np.stack([0.6 * i.ravel(), 0.4 + 0.6 * k.ravel(), 0.6 * j.ravel()], axis=1).astype(f32)
    n = len(pos)
    orn = _random_quats(n, rng)
    if jitter:
        pos += rng.uniform(-jitter, jitter, size=pos.shape).astype(f32)
    which = np.arange(n) % 3
    sk = np.where(which == 0, SHAPE_BOX, np.where(which == 1, SHAPE_SPHERE, SHAPE_CAPSULE)).astype(np.uint32)
    params = np.zeros((n, 4), f32)
    params[which == 0] = (0.25, 0.25, 0.25, 0)
    params[which == 1] = (0.25, 0, 0, 0)
    params[which == 2] = (0.15, 0.2, 0, 0)
    dyn = (pos, orn, sk, params, np.full(n, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _box_walls(0.6 * (side - 1) + 0.9, 0.6 * (side - 1) + 0.9, 0.6 * side + 1.0)), friction=0.5, restitution=0.2)
    return dict(name=f"mixed_{n}", bodies=b, hinges=None, exclusions=None, dynamic=n,
                settings=dict(velocity_iterations=20, position_iterations=3))


def hinge_chains(chains_x=512, chains_z=512, links=4):
    """Config 5: chains of `links` capsules joined by hinges (1 048 576 bodies at 512 x 512 x 4), resting 0.05 above
    a plane; adjacent links never collide (exclude_collision); 10 velocity iterations."""
    nc = chains_x * chains_z
    cx, cz = np.meshgrid(np.arange(chains_x), np.arange(chains_z), indexing="ij")
    base = np.stack([cx.ravel() * (0.7 * links + 0.7), np.full(nc, 0.15), cz.ravel() * 0.5], axis=1)
    pos = (base[:, None, :] + np.stack([0.7 * np.arange(links), np.zeros(links), np.zeros(links)], axis=1)[None]).reshape(-1, 3).astype(f32)
    n = nc * links
    dyn = (pos, _identity(n), np.full(n, SHAPE_CAPSULE, np.uint32), np.tile(np.array([0.1, 0.25, 0, 0], f32), (n, 1)),
           np.full(n, DYNAMIC, np.uint32))
    b = _assemble(*_join(dyn, _planes([((0, 1, 0), 0.0)])))
    first = (np.arange(nc)[:, None] * links + np.arange(links - 1)[None]).ravel().astype(np.uint32)
    nh = len(first)
    hinges = dict(a=first, b=first + 1, pivot_a=np.tile(np.array([0.35, 0, 0], f32), (nh, 1)),
                  pivot_b=np.tile(np.array([-0.35, 0, 0], f32), (nh, 1)), axis_a=np.tile(np.array([0, 0, 1], f32), (nh, 1)),
                  axis_b=np.tile(np.array([0, 0, 1], f32), (nh, 1)))
    return dict(name=f"chains_{n}", bodies=b, hinges=hinges, exclusions=(first, first + 1), dynamic=n,
                settings=dict(velocity_iterations=10, position_iterations=3))


def build_world(scene, device=0, max_manifolds=None, flags=0, max_bodies=None, max_hinges=None, **override):
    """Create a device world holding `scene` (edyn_b200.World).  max_bodies / max_hinges reserve room for bodies that
    arrive later (island migration)."""
    from .world import World
    b = scene["bodies"]
    n = max(len(b["kind"]), max_bodies or 0)
    st = dict(scene["settings"])
    st.update(override)
    nh = max(len(scene["hinges"]["a"]) if scene["hinges"] else 0, max_hinges or 0)
    w = World(n, max_manifolds=max_manifolds or max(4096, 10 * n), max_hinges=nh, device=device,
              velocity_iterations=st["velocity_iterations"], position_iterations=st["position_iterations"], flags=flags)
    w.add_bodies(b)
    if scene["hinges"]:
        h = scene["hinges"]
        w.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    if scene["exclusions"] is not None:
        w.add_exclusions(*scene["exclusions"])
    return w


def raycast_segments(lo, hi, n, kind="mixed", seed=0):
    """Segments over a scene whose bodies lie in the box [lo, hi] (3 floats each): "down" = probes from 1 m above the box
    to 1 m below it at uniform (x, z), as ground / line-of-sight probes; "across" = horizontal segments at uniform height
    and heading that cross the whole box; "mixed" = half of each.  Returns p0, p1 as (n, 3) float32."""
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    nd = n if kind == "down" else (0 if kind == "across" else n // 2)
    p0, p1 = np.empty((n, 3)), np.empty((n, 3))
    xz = rng.uniform(lo[[0, 2]], hi[[0, 2]], (nd, 2))
    p0[:nd] = np.stack([xz[:, 0], np.full(nd, hi[1] + 1.0), xz[:, 1]], 1)
    p1[:nd] = np.stack([xz[:, 0], np.full(nd, lo[1] - 1.0), xz[:, 1]], 1)
    na = n - nd
    c, half = (lo + hi) / 2, np.linalg.norm((hi - lo)[[0, 2]]) / 2 + 1.0
    ang = rng.uniform(0, 2 * np.pi, na)
    d = np.stack([np.cos(ang), np.zeros(na), np.sin(ang)], 1)
    off = rng.uniform(lo[[0, 2]], hi[[0, 2]], (na, 2)) - c[[0, 2]]
    mid = np.stack([c[0] + off[:, 0] * 0.5, rng.uniform(lo[1], hi[1], na), c[2] + off[:, 1] * 0.5], 1)
    p0[nd:], p1[nd:] = mid - d * half, mid + d * half
    return p0.astype(f32), p1.astype(f32)
