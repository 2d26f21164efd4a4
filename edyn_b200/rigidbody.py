"""Host-side mirror of edyn::rigidbody_def / make_rigidbody (reference include/edyn/util/rigidbody.hpp,
src/edyn/util/rigidbody.cpp:47-185): turns body definitions into the component arrays the device world stages.

All arithmetic is float32 and follows the reference's expression order (moment_of_inertia.cpp:11-91,
matrix3x3.hpp:177-204) so that the staged inertia_inv matches what make_rigidbody would have emplaced.
"""
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

f32 = np.float32

SHAPE_SPHERE, SHAPE_CAPSULE, SHAPE_BOX, SHAPE_PLANE, SHAPE_NONE = 0, 2, 3, 6, 255
DYNAMIC, KINEMATIC, STATIC = 0, 1, 2


@dataclass
class Shape:
    kind: int
    params: Sequence[float]            # sphere (r); capsule (r, half_length, axis); box (hx, hy, hz); plane (nx, ny, nz, c)


def sphere_shape(radius):
    return Shape(SHAPE_SPHERE, (radius, 0, 0, 0))


def capsule_shape(radius, half_length, axis=0):
    return Shape(SHAPE_CAPSULE, (radius, half_length, float(axis), 0))


def box_shape(half_extents):
    return Shape(SHAPE_BOX, (half_extents[0], half_extents[1], half_extents[2], 0))


def plane_shape(normal, constant):
    return Shape(SHAPE_PLANE, (normal[0], normal[1], normal[2], constant))


MATERIAL_UNASSIGNED = 0xFFFF           # material::UnassignedID
MATERIAL_NONE = 0xFFFFFFFF             # B2D_MATERIAL_NONE: no material component, the body is a sensor


@dataclass
class Material:                        # include/edyn/comp/material.hpp (friction default 0.5, restitution 0)
    restitution: float = 0.0
    friction: float = 0.5
    id: int = MATERIAL_UNASSIGNED      # material::id, the key of the mixing table (edyn.insert_material_mixing)


@dataclass
class RigidBodyDef:                    # include/edyn/util/rigidbody.hpp rigidbody_def
    kind: int = DYNAMIC
    position: Sequence[float] = (0.0, 0.0, 0.0)
    orientation: Sequence[float] = (0.0, 0.0, 0.0, 1.0)
    mass: float = 1.0
    inertia: Optional[np.ndarray] = None
    linvel: Sequence[float] = (0.0, 0.0, 0.0)
    angvel: Sequence[float] = (0.0, 0.0, 0.0)
    gravity: Optional[Sequence[float]] = None      # None -> world default (settings.gravity)
    shape: Optional[Shape] = None
    material: Optional[Material] = field(default_factory=Material)     # None: a sensor (collides, is never pushed)
    collision_group: int = 0xFFFFFFFFFFFFFFFF
    collision_mask: int = 0xFFFFFFFFFFFFFFFF
    presentation: bool = True          # present_position / present_orientation; make_rigidbody emplaces them on dynamic bodies only


def moment_of_inertia(shape: Shape, mass) -> np.ndarray:
    """dynamics/moment_of_inertia.cpp:11-91,159-181 for the in-scope shapes (float32)."""
    m = f32(mass)
    p = [f32(x) for x in shape.params]
    if shape.kind == SHAPE_SPHERE:
        i = f32(0.4) * m * p[0] * p[0]
        return np.diag([i, i, i]).astype(f32)
    if shape.kind == SHAPE_BOX:
        e = [p[0] * f32(2), p[1] * f32(2), p[2] * f32(2)]
        k = f32(1) / f32(12) * m
        return np.diag([k * (e[1] * e[1] + e[2] * e[2]), k * (e[2] * e[2] + e[0] * e[0]), k * (e[0] * e[0] + e[1] * e[1])]).astype(f32)
    if shape.kind == SHAPE_CAPSULE:
        pi = f32(3.1415926535897932384626433832795029)
        r, length, axis = p[0], p[1] * f32(2), int(p[2])
        cyl_vol = pi * r * r * length
        sph_vol = pi * r * r * r * f32(4) / f32(3)
        total = cyl_vol + sph_vol
        cyl_mass = m * cyl_vol / total
        sph_mass = m * sph_vol / total
        cxx = f32(0.5) * cyl_mass * r * r
        cyz = f32(1) / f32(12) * cyl_mass * (f32(3) * r * r + length * length)
        sph_i = f32(0.4) * sph_mass * r * r
        # the reference reads .x / .y of the cylinder inertia AFTER its own axis permutation
        # (moment_of_inertia.cpp:27-44, :76-77); mirrored so the staged inertia_inv matches make_rigidbody
        cyl = [cyz, cyz, cyz]
        cyl[axis] = cxx
        xx = sph_i + cyl[0]
        t = f32(4) * length + f32(3) * r
        yy = sph_i + sph_mass * (t * t) / f32(64) + cyl[1]
        d = [yy, yy, yy]
        d[axis] = xx
        return np.diag(d).astype(f32)
    raise ValueError("moment_of_inertia: shape outside the hot-path scope")


def inverse_matrix_symmetric(mat: np.ndarray) -> np.ndarray:
    """math/matrix3x3.hpp:177-204, float32."""
    a = mat.astype(f32)
    r0, r1, r2 = a[0], a[1], a[2]
    c = np.array([r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0]], f32)
    det = f32(r0[0] * c[0] + r0[1] * c[1] + r0[2] * c[2])
    di = f32(1) / det
    a11, a12, a13, a22, a23, a33 = a[0, 0], a[0, 1], a[0, 2], a[1, 1], a[1, 2], a[2, 2]
    o = np.zeros((3, 3), f32)
    o[0, 0] = di * (a22 * a33 - a23 * a23)
    o[0, 1] = di * (a13 * a23 - a12 * a33)
    o[0, 2] = di * (a12 * a23 - a13 * a22)
    o[1, 0] = o[0, 1]
    o[1, 1] = di * (a11 * a33 - a13 * a13)
    o[1, 2] = di * (a12 * a13 - a11 * a23)
    o[2, 0] = o[0, 2]
    o[2, 1] = o[1, 2]
    o[2, 2] = di * (a11 * a22 - a12 * a12)
    return o


def bodies_soa(defs: Sequence[RigidBodyDef], default_gravity=(0.0, -9.8, 0.0)) -> dict:
    """Component arrays for a list of definitions, laid out as include/b2d.h's b2d_bodies expects."""
    n = len(defs)
    out = dict(pos=np.zeros((n, 3), f32), orn=np.zeros((n, 4), f32), linvel=np.zeros((n, 3), f32),
               angvel=np.zeros((n, 3), f32), inv_mass=np.zeros(n, f32), inv_inertia=np.zeros((n, 9), f32),
               gravity=np.zeros((n, 3), f32), kind=np.zeros(n, np.uint32), shape_kind=np.full(n, SHAPE_NONE, np.uint32),
               shape_params=np.zeros((n, 4), f32), friction=np.zeros(n, f32), restitution=np.zeros(n, f32),
               group=np.full(n, 0xFFFFFFFFFFFFFFFF, np.uint64), mask=np.full(n, 0xFFFFFFFFFFFFFFFF, np.uint64),
               material=np.full(n, MATERIAL_UNASSIGNED, np.uint32), presentation=np.zeros(n, np.uint32))
    cache = {}
    for i, d in enumerate(defs):
        out["pos"][i] = d.position
        out["orn"][i] = d.orientation
        out["kind"][i] = d.kind
        if d.kind != STATIC:
            out["linvel"][i] = d.linvel
            out["angvel"][i] = d.angvel
        if d.kind == DYNAMIC:
            out["inv_mass"][i] = f32(1) / f32(d.mass)
            if d.inertia is not None:
                inv = inverse_matrix_symmetric(np.asarray(d.inertia, f32))
            else:
                key = (d.shape.kind, tuple(d.shape.params), float(d.mass))
                if key not in cache:
                    cache[key] = inverse_matrix_symmetric(moment_of_inertia(d.shape, d.mass))
                inv = cache[key]
            out["inv_inertia"][i] = inv.reshape(9)
            g = default_gravity if d.gravity is None else d.gravity
            out["gravity"][i] = g
        if d.shape is not None:
            out["shape_kind"][i] = d.shape.kind
            out["shape_params"][i] = d.shape.params
        if d.material is not None:
            out["friction"][i] = d.material.friction
            out["restitution"][i] = d.material.restitution
            out["material"][i] = d.material.id
        else:
            out["material"][i] = MATERIAL_NONE
        out["group"][i] = d.collision_group
        out["mask"][i] = d.collision_mask
        out["presentation"][i] = 1 if d.presentation and d.kind == DYNAMIC else 0
    return out
