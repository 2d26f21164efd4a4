"""Sensors and the material mixing table: the oracle (driven by tests/material_oracle.py) against the reference's REAL
stepper (oracle/ref_stepper.cpp with the material entry points of tests/materials/refm.hpp), bit for bit every step -- state, ordered pair sets, point counts, each point's friction and restitution, which points
carry a contact_constraint (a sensor's carry a null_constraint and no contact_point_material / _impulse), island
partitions and, where sleeping is on, the sleeping flags.

A body made without a material (rigidbody_def::material = std::nullopt) is a sensor; material ids select entries of
registry.ctx().get<material_mix_table>() when a point is created (collision_util.cpp:282-317) and, for the restitution
solver, when a manifold is created (constraint_util.cpp:90-101).  The restitution solver would read a material a sensor's
points lack (restitution_solver.cpp:225): the restatement skips such manifolds, so the restitution-solver scenes here
have no sensors."""
import numpy as np
import pytest

from tests import material_oracle as M
from tests.test_gpu_materials import FLOOR, ICE, NONE, RUBBER, STONE, TABLE, UNASSIGNED, _scene
from tests.test_ref_stepper import _keys, _refines

f32 = np.float32


@pytest.fixture(scope="module")
def refstep(O):
    """O with O.refm = tests/materials/_build/libref_materials.so (built where the reference is, else skipped)."""
    if O.ref_stepper() is None:
        pytest.skip("oracle/_ref/libedyn_stepper.so not available (needs /root/reference at build time)")
    M.build()
    O.refm = M.library(O, "ref_materials")
    if O.refm is None:
        pytest.skip("tests/materials/_build/libref_materials.so not available")
    return O


def ref_world(O, scene, sleeping=False, **kw):
    """The real stepper holding `scene` with its materials: (RefWorld, RefMaterials)."""
    r = O.RefWorld(vel_iters=scene["settings"]["velocity_iterations"], pos_iters=scene["settings"]["position_iterations"],
                   library=O.refm, **kw)
    rm = M.RefMaterials(O.refm, r)
    rm.populate(scene, sleeping_disabled=not sleeping)
    return r, rm


def _join(scene, extra, material):
    """scene with the bodies `extra` (a b2d_bodies-style dict) appended, their material column `material`."""
    b = dict(scene["bodies"])
    if b.get("material") is None:
        b["material"] = np.full(len(b["kind"]), UNASSIGNED, np.uint32)
    extra = dict(extra, material=np.asarray(material, np.uint32))
    return dict(scene, bodies={k: np.concatenate([b[k], extra[k]]) for k in b})


def _bodies(E, pos, shape, params, kind, gravity=None, linvel=None):
    n = len(pos)
    b = E.scenes._assemble(np.asarray(pos, f32), np.tile(np.array([0, 0, 0, 1], f32), (n, 1)), np.full(n, shape, np.uint32),
                           np.tile(np.asarray(params, f32), (n, 1)), np.full(n, kind, np.uint32))
    if gravity is not None:
        b["gravity"][:] = gravity
    if linvel is not None:
        b["linvel"][:] = linvel
    return b


def lockstep(O, scene, steps, table=(), edits=None, restitution_iterations=0, sleeping=False):
    """Free-running lock step of the real stepper and the oracle with the mixing entries `table` set before the first step;
    edits: {step: [(id0, id1, friction, restitution) or (id0, id1) to remove]} applied to both before that step.  Asserts
    on the first difference; returns (sensor points seen, points seen, steps whose partition the reference had coarser)."""
    r, rm = ref_world(O, scene, sleeping, restitution_iters=restitution_iterations)
    o = M.MaterialOracle(O, scene, restitution=restitution_iterations > 0, sleeping=sleeping)
    o.set_position_type_order(contacts_first=True)
    o.set_restitution_iterations(restitution_iterations)

    def apply(entries):
        ins = [e for e in entries if len(e) == 4]
        rem = [e for e in entries if len(e) == 2]
        if ins:
            a, b, f, e = (np.array(c) for c in zip(*ins))
            rm.set_material_mixing(a, b, f, e); o.set_material_mixing(a, b, f, e)
        if rem:
            a, b = (np.array(c) for c in zip(*rem))
            rm.remove_material_mixing(a, b); o.remove_material_mixing(a, b)
    apply(list(table))
    sensor = np.asarray(scene["bodies"]["material"]) == NONE
    dyn = np.asarray(scene["bodies"]["kind"]) == 0
    sensor_points = points = coarser = 0
    for s in range(steps):
        if edits and s in edits:
            apply(edits[s])
        if restitution_iterations:
            r.step_begin()
            graph = r.graph_order()
            r.step_end()
        else:
            r.step(1)
        hi, ct = r.solver_order()
        o.run_phases(O.PH_BROAD | O.PH_NARROW | O.PH_ISLANDS)
        ref_islands = r.islands()
        refines, equal = _refines(o.islands()[dyn], ref_islands[dyn])
        assert refines, f"step {s}: the oracle's islands are not a refinement of the reference's"
        coarser += not equal
        o.set_islands(ref_islands)
        o.set_point_order(hi, ct)
        if restitution_iterations:
            o.set_graph_order(*graph)
        o.run_phases(O.PH_SOLVE)
        a, b = r.state(), o.state()
        for k in ("pos", "orn", "linvel", "angvel", "aabb"):
            assert np.array_equal(a[k], b[k]), f"step {s}: {k} differs"
        if sleeping:
            assert np.array_equal(r.sleeping(), o.sleeping().astype(bool)), f"step {s}: sleeping flags differ"
        rc, oc = rm.contacts(), o.contacts()
        rk, ok = _keys(rc["pairs"]), _keys(oc["pairs"])
        ri, oi = np.argsort(rk), np.argsort(ok)
        assert np.array_equal(rk[ri], ok[oi]), f"step {s}: ordered pair sets differ"
        assert np.array_equal(rc["num"][ri], oc["num"][oi]), f"step {s}: point counts differ"
        for x, y in zip(ri, oi):
            nm = int(rc["num"][x])
            if not nm:
                continue
            pa, pb = (int(v) for v in rc["pairs"][x])
            is_sensor = bool(sensor[pa] or sensor[pb])
            got, want = rc["mat"][x, :nm], oc["pts"][y, :nm]
            assert np.array_equal(got[:, 0], want[:, 13]) and np.array_equal(got[:, 1], want[:, 14]), \
                f"step {s}: friction / restitution of {(pa, pb)} differ: {got[:, :2]} against {want[:, 13:15]}"
            assert np.all(got[:, 2] == (0 if is_sensor else 1)) and np.all(got[:, 3] == got[:, 2]), \
                f"step {s}: {(pa, pb)}: contact_constraint / impulse on a {'sensor' if is_sensor else 'material'} pair's points"
            sensor_points += nm * is_sensor
            points += nm
    return sensor_points, points, coarser


def _sensors(E):
    """A dynamic sensor box falling through the pile, a static sensor box around a column and a kinematic sensor sphere
    sweeping through (ids: NONE)."""
    from edyn_b200.rigidbody import DYNAMIC, KINEMATIC, SHAPE_BOX, SHAPE_SPHERE, STATIC
    parts = [_bodies(E, [[1.0, 4.0, 1.0]], SHAPE_BOX, (0.4, 0.4, 0.4, 0), DYNAMIC),
             _bodies(E, [[0.0, 1.0, 1.0]], SHAPE_BOX, (0.8, 1.2, 1.6, 0), STATIC),
             _bodies(E, [[-1.5, 0.35, 1.0]], SHAPE_SPHERE, (0.3, 0, 0, 0), KINEMATIC, linvel=(3.0, 0, 0))]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def test_sensors_over_piles_match_real_stepper(refstep, E):
    """Dynamic, kinematic and static sensors in a pile with material ids and table entries, spheres and boxes."""
    for shape in ("box", "sphere"):
        scene, n = _scene(E, shape, 3)
        sp, pts, _ = lockstep(refstep, scene, 150, TABLE)
        assert sp > 0 and pts > sp, (shape, sp, pts)


def test_sensors_over_hinge_chains_match_real_stepper(refstep, E):
    scene = _join(E.scenes.hinge_chains(3, 3, 4), _sensors(E), [NONE] * 3)
    sp, pts, _ = lockstep(refstep, scene, 150)
    assert sp > 0 and pts > sp


def test_zero_point_sensor_manifold_joins_islands(refstep, E):
    """A weightless dynamic sensor sphere floating 0.015 from two resting boxes: inside the broadphase margin, outside the
    contact threshold, so its two manifolds never get a point, yet they join the boxes into one island."""
    from edyn_b200.rigidbody import DYNAMIC, SHAPE_SPHERE
    scene = E.scenes.boxes_on_plane(1)
    b = scene["bodies"]
    two = {k: np.concatenate([b[k][:1], b[k][:1]]) for k in b}
    two["pos"] = np.array([[0.0, 0.5, 0.0], [1.63, 0.5, 0.0]], f32)
    floor = {k: b[k][1:] for k in b}
    s = _bodies(E, [[0.815, 0.5, 0.0]], SHAPE_SPHERE, (0.3, 0, 0, 0), DYNAMIC, gravity=(0, 0, 0))
    scene = dict(scene, bodies={k: np.concatenate([two[k], floor[k]]) for k in b})
    scene["bodies"]["material"] = np.full(3, UNASSIGNED, np.uint32)
    scene = _join(scene, s, [NONE])
    O = refstep
    sp, pts, _ = lockstep(O, scene, 60)
    assert sp == 0 and pts > 0
    r, rm = ref_world(O, scene)
    r.step(30)
    lab = r.islands()
    assert lab[0] == lab[1] == lab[3] != 0xFFFFFFFF, lab
    c = rm.contacts()
    sensor_pairs = [k for k, p in enumerate(c["pairs"].tolist()) if 3 in p]
    assert len(sensor_pairs) == 2 and not c["num"][sensor_pairs].any()


def test_sensor_keeps_island_awake(refstep, E):
    """Island sleeping on: a slow weightless dynamic sensor passing through a resting box keeps the box's island awake
    while they touch; both sides agree on every sleeping flag."""
    from edyn_b200.rigidbody import DYNAMIC, SHAPE_SPHERE
    scene = E.scenes.boxes_on_plane(1)
    scene["bodies"]["material"] = np.full(2, UNASSIGNED, np.uint32)
    s = _bodies(E, [[-4.0, 0.5, 0.0]], SHAPE_SPHERE, (0.3, 0, 0, 0), DYNAMIC, gravity=(0, 0, 0), linvel=(0.5, 0, 0))
    scene = _join(scene, s, [NONE])
    sp, _, _ = lockstep(refstep, scene, 600, sleeping=True)
    assert sp > 0


def test_mixing_table_matches_real_stepper(refstep, E):
    """Entries that override friction, turn restitution on for a pair whose mix is 0 and off for one whose mix is > 0, an
    entry for ids no body has, unassigned ids; then entries inserted, overwritten and removed between steps."""
    scene, _ = _scene(E, "box", 3, sensors=False)
    lockstep(refstep, scene, 150, TABLE)
    edits = {20: [(RUBBER, FLOOR, 0.2, 0.9), (ICE, STONE, 0.7, 0.0)], 40: [(FLOOR, RUBBER)], 60: [(STONE, STONE, 1.0, 0.5)],
             80: [(STONE, FLOOR), (ICE, ICE)]}
    lockstep(refstep, scene, 150, TABLE, edits=edits)
    sphere, _ = _scene(E, "sphere", 3, sensors=False)
    lockstep(refstep, sphere, 150, TABLE, edits=edits)


def test_restitution_solver_with_mixing_matches_real_stepper(refstep, E):
    """The restitution solver with table-driven restitution (no sensors: see the module docstring)."""
    for shape in ("box", "sphere"):
        scene, _ = _scene(E, shape, 3, sensors=False)
        lockstep(refstep, scene, 120, TABLE, restitution_iterations=8)


def test_bodies_soa_material_column(E):
    """RigidBodyDef(material=None) stages B2D_MATERIAL_NONE; a Material's id is staged as it is, unassigned by default."""
    R = E.rigidbody
    defs = [R.RigidBodyDef(shape=R.sphere_shape(0.5)), R.RigidBodyDef(shape=R.sphere_shape(0.5), material=None),
            R.RigidBodyDef(shape=R.sphere_shape(0.5), material=R.Material(friction=0.2, id=7))]
    soa = R.bodies_soa(defs)
    assert soa["material"].tolist() == [UNASSIGNED, NONE, 7]
    assert soa["friction"].tolist() == [f32(0.5), 0.0, f32(0.2)]
