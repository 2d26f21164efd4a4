"""Sensors (bodies without a material) and the material mixing table on the device, in lock step with the oracle
(tests/parity.py) in every solver mode, with the restitution solver off and on.

A sensor's pairs get manifolds and contact points like any other pair and join islands, but no rows: nothing pushes a
sensor, a sensor pushes nothing, and the solver order never names a sensor's manifold.  Mixing-table entries replace the
mixed friction and restitution of points created after the entry was set; existing points keep theirs.

The scenes are sized so that sensors sit in two-point tiles (spheres), generic tiles (small box piles) and on the dataflow
path (a pile of more bodies than a tile holds, and the dataflow mode).  Also runs against the CPU emulation (B2D_EMU=1),
without the CUDA-graph mode."""
import os

import numpy as np
import pytest

from tests.material_oracle import MaterialOracle
from tests.parity import lockstep

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
STEPS = 40 if EMU else 120
NONE, UNASSIGNED = 0xFFFFFFFF, 0xFFFF
f32 = np.float32

# material ids of the scenes below and the mixing entries set before the first step: (id0, id1, friction, restitution)
FLOOR, RUBBER, ICE, STONE = 1, 2, 3, 4
TABLE = [(FLOOR, RUBBER, 1.2, 0.6),      # restitution on for a pair whose mix is 0
         (STONE, FLOOR, 0.05, 0.0),      # restitution off and friction down for a pair whose mix is > 0
         (ICE, ICE, 0.01, 0.0),
         (40, 41, 0.3, 0.3)]             # ids no body has


def _scene(E, shape="box", side=3, sensors=True):
    """A side x side x 2 pile (one island: more bodies than a tile holds at side 9) of dynamic boxes (or spheres) on a floor plane, with material ids cycling through RUBBER,
    ICE, STONE and unassigned; the floor is FLOOR with restitution 0.  With sensors: a dynamic sensor box dropped onto the
    pile (it falls through everything), a static sensor box enclosing the pile's first column and a kinematic sensor
    sphere sweeping through the pile."""
    from edyn_b200.rigidbody import DYNAMIC, KINEMATIC, SHAPE_BOX, SHAPE_SPHERE, STATIC
    i, k, j = np.meshgrid(np.arange(side), np.arange(2), np.arange(side), indexing="ij")
    pos = np.stack([i.ravel(), 0.55 + 1.05 * k.ravel(), j.ravel()], axis=1).astype(f32)          # side by side: one island
    n = len(pos)
    sk = SHAPE_BOX if shape == "box" else SHAPE_SPHERE
    params = (0.5, 0.5, 0.5, 0) if shape == "box" else (0.5, 0, 0, 0)
    parts = [(pos, np.full(n, sk, np.uint32), np.tile(np.array(params, f32), (n, 1)), np.full(n, DYNAMIC, np.uint32))]
    ids = [np.array([RUBBER, ICE, STONE, UNASSIGNED], np.uint32)[np.arange(n) % 4]]
    rest = [np.where(np.arange(n) % 4 == 2, f32(0.4), f32(0.0)).astype(f32)]       # STONE bounces on its own
    if sensors:
        c = 0.5 * (side - 1)
        spos = np.array([[c, 4.0, c], [0.0, 1.0, c], [-1.5, 0.6, c]], f32)
        parts.append((spos, np.array([SHAPE_BOX, SHAPE_BOX, SHAPE_SPHERE], np.uint32),
                      np.array([[0.4, 0.4, 0.4, 0], [0.8, 1.2, 0.55 * side, 0], [0.3, 0, 0, 0]], f32),
                      np.array([DYNAMIC, STATIC, KINEMATIC], np.uint32)))
        ids.append(np.full(3, NONE, np.uint32))
        rest.append(np.zeros(3, f32))
    pos, sk, params, kind = (np.concatenate([p[q] for p in parts]) for q in range(4))
    m = len(kind)
    pos = np.concatenate([pos, np.zeros((1, 3), f32)])
    orn = np.tile(np.array([0, 0, 0, 1], f32), (m + 1, 1))
    from edyn_b200.rigidbody import SHAPE_PLANE
    b = E.scenes._assemble(pos, orn, np.concatenate([sk, [SHAPE_PLANE]]).astype(np.uint32),
                           np.concatenate([params, [[0, 1, 0, 0]]]).astype(f32),
                           np.concatenate([kind, [STATIC]]).astype(np.uint32), friction=0.5,
                           restitution=np.concatenate(rest + [np.zeros(1, f32)]))
    b["material"] = np.concatenate(ids + [np.array([FLOOR], np.uint32)])
    if sensors:
        b["linvel"][n + 2] = (3.0, 0, 0)          # the kinematic sensor sweeps through the pile
    return dict(name=f"materials_{shape}_{side}", bodies=b, hinges=None, exclusions=None, dynamic=n,
                settings=dict(velocity_iterations=10, position_iterations=3)), n


def _set_table(w, o, table=TABLE):
    a, b, f, r = (np.array(c) for c in zip(*table))
    w.set_material_mixing(a, b, f, r)
    o.set_material_mixing(a, b, f, r)


class SensorCheck:
    """lockstep hook: no sensor manifold in the solver order, and the figures the tests assert on."""

    def __init__(self, sensors):
        self.sensors = np.asarray(sensors, np.uint32)
        self.fell_with_points = False       # the dynamic sensor below the floor's surface, its floor manifold holding points
        self.inside = set()                 # bodies the static sensor had points with

    def __call__(self, step, w):
        _, order = w.solver_order()
        assert not np.isin(order, self.sensors).any(), f"step {step}: a sensor's manifold is in the solver order"
        c = w.contacts()
        dyn, stat = int(self.sensors[0]), int(self.sensors[1])
        floor = w.num_bodies - 1
        for k, p in enumerate(c["pairs"].tolist()):
            if c["num"][k] and stat in p:
                self.inside.add(p[0] if p[1] == stat else p[1])
            if c["num"][k] and set(p) == {dyn, floor} and w.download_state(aabb=False)["pos"][dyn, 1] < 0.0:
                self.fell_with_points = True
            if c["num"][k] and (dyn in p or stat in p or int(self.sensors[2]) in p):
                pts = c["pts"][k, :c["num"][k]]
                assert not pts[:, 13:18].any(), f"step {step}: a sensor's point has friction, restitution or impulses"


@pytest.mark.parametrize("restitution", [False, True], ids=["rows", "restitution_solver"])
@pytest.mark.parametrize("shape,side", [("sphere", 3), ("box", 3), ("box", 9)], ids=["two_point_tiles", "tiles", "dataflow_pile"])
def test_sensors_lockstep(gpu, E, O, shape, side, restitution):
    scene, n = _scene(E, shape, side)
    sensors = [n, n + 1, n + 2]
    for mode in MODES:
        hook = SensorCheck(sensors)

        def before(s, w, o):
            if s == 0:                                  # the oracle that knows the materials, and the table on both sides
                o = MaterialOracle(O, scene, restitution=restitution)
                _set_table(w, o)
            return o
        res = lockstep(E, O, scene, STEPS, restitution_solver=restitution, mode=mode, hook=hook, before=before)
        assert res["ok"], (scene["name"], mode, res)
        assert hook.fell_with_points or EMU, (scene["name"], mode)       # the dynamic sensor fell through the floor
        first_column = set(range(0, 2 * side))                           # i = 0: bodies 0 .. 2 side - 1
        assert first_column <= hook.inside, (scene["name"], mode, sorted(hook.inside))


def test_sensor_falls_through(gpu, E):
    """A dynamic sensor dropped on the pile passes through it and the floor and keeps falling freely."""
    scene, n = _scene(E, "box", 3)
    w = E.scenes.build_world(scene)
    steps, dt = 90, 1.0 / 60
    w.step(steps)
    st = w.download_state(aabb=False)
    y = 4.0 - 9.8 * dt * dt * steps * (steps + 1) / 2                                         # semi-implicit Euler free fall
    assert abs(float(st["pos"][n, 1]) - y) < 1e-3, st["pos"][n]                               # no contact ever pushed it
    assert float(st["pos"][0, 1]) > 0.4                                                        # the pile still rests on the floor
    assert w.stats()["error_flags"] == 0


def test_mixing_applies_to_new_points_only(gpu, E):
    """A table entry set while points exist leaves them as they are; points created afterwards carry the entry.  Removing it
    brings the mix back for later points."""
    scene, _ = _scene(E, "box", 2, sensors=False)
    floor = scene["bodies"]["kind"].shape[0] - 1

    def floor_points(w, body):
        c = w.contacts()
        k = [i for i, p in enumerate(c["pairs"].tolist()) if set(p) == {body, floor}]
        return c["pts"][k[0], :c["num"][k[0]]] if k else np.zeros((0, 18), f32)

    rubber, settle = 0, 30                              # body 0: material RUBBER, restitution 0, resting on FLOOR
    mixed = f32(np.sqrt(f32(0.5) * f32(0.5)))
    w = E.scenes.build_world(scene)
    w.step(settle)
    before = floor_points(w, rubber)
    assert len(before) and np.all(before[:, 13] == mixed) and np.all(before[:, 14] == 0)
    w.set_material_mixing([RUBBER], [FLOOR], [1.2], [0.0])
    w.step(1)
    after = floor_points(w, rubber)
    assert np.all(after[:, 13] == mixed) and np.all(after[:, 14] == 0), after[:, 13:15]     # the settled points keep theirs
    # the entry set before the first contact: the points take it, in either id order
    w2 = E.scenes.build_world(scene)
    w2.set_material_mixing([FLOOR], [RUBBER], [1.2], [0.0])
    w2.step(settle)
    got = floor_points(w2, rubber)
    assert len(got) and np.all(got[:, 13] == f32(1.2)) and np.all(got[:, 14] == 0)
    # an entry removed before the first contact: the mix again
    w3 = E.scenes.build_world(scene)
    w3.set_material_mixing([FLOOR], [RUBBER], [1.2], [0.0])
    w3.remove_material_mixing([FLOOR], [RUBBER])
    w3.step(settle)
    got = floor_points(w3, rubber)
    assert len(got) and np.all(got[:, 13] == mixed) and np.all(got[:, 14] == 0)


def test_table_edits_between_steps_lockstep(gpu, E, O):
    """Table entries inserted, overwritten and removed between steps, the restitution through the rows, and a table that
    outgrows its first allocation: the device follows the oracle in every mode."""
    scene, n = _scene(E, "box", 3)
    big = [(100 + k, 200 + k, 0.1, 0.1) for k in range(200)]          # more entries than the first allocation holds

    def before(s, w, o):
        if s == 0:
            o = MaterialOracle(O, scene)
            _set_table(w, o)
        elif s == 10:
            _set_table(w, o, [(RUBBER, FLOOR, 0.2, 0.9), (ICE, STONE, 0.7, 0.0)])
        elif s == 20:
            w.remove_material_mixing([FLOOR], [RUBBER]); o.remove_material_mixing([FLOOR], [RUBBER])
        elif s == 25:
            _set_table(w, o, big)
        return o
    for mode in MODES:
        res = lockstep(E, O, scene, STEPS, mode=mode, hook=SensorCheck([n, n + 1, n + 2]), before=before)
        assert res["ok"], (mode, res)


def test_abi_checks(gpu, E):
    """Bad ids are argument errors, a sensor toggle is unsupported, and a NULL material column is all-unassigned."""
    scene, n = _scene(E, "box", 2)
    w = E.scenes.build_world(scene)
    with pytest.raises(E.B2DError, match="error -4"):
        w.set_material_mixing([0xFFFF], [1], [0.5], [0.0])
    with pytest.raises(E.B2DError, match="error -4"):
        w.remove_material_mixing([1], [0x10000])
    with pytest.raises(E.B2DError, match="error -3"):
        w.upload_bodies([0], material=[NONE])                     # a body with a material becomes a sensor
    with pytest.raises(E.B2DError, match="error -3"):
        w.upload_bodies([n], material=[RUBBER])                   # a sensor gets a material
    with pytest.raises(E.B2DError, match="error -4"):
        w.upload_bodies([0], material=[0x10000])
    w.upload_bodies([0, n], material=[ICE, NONE])                 # id changes and a sensor staying one are fine
    bad = dict(scene["bodies"]); bad["material"] = bad["material"].copy(); bad["material"][0] = 0x12345
    with pytest.raises(E.B2DError, match="error -4"):
        E.scenes.build_world(dict(scene, bodies=bad))
    # NULL material == every body unassigned
    plain = {k: v for k, v in scene["bodies"].items() if k != "material"}
    unassigned = dict(plain, material=np.full(len(plain["kind"]), UNASSIGNED, np.uint32))
    a, b = E.scenes.build_world(dict(scene, bodies=plain)), E.scenes.build_world(dict(scene, bodies=unassigned))
    for x in (a, b):
        x.set_material_mixing([RUBBER], [FLOOR], [1.5], [0.5])    # no body has an id: nothing to look up
        x.step(40)
    sa, sb = a.download_state(), b.download_state()
    for k in ("pos", "orn", "linvel", "angvel", "aabb"):
        assert np.array_equal(sa[k], sb[k]), k


def _handover_scene(E):
    """Two stacks of three boxes sliding into each other (left RUBBER, right STONE, floor FLOOR) and a weightless dynamic
    sensor sphere riding on the right stack's top box: its manifold joins it to the right stack's island, so it moves
    with that island from rank 1 to rank 0."""
    from edyn_b200.rigidbody import DYNAMIC, SHAPE_SPHERE
    scene = E.scenes.approaching_stacks(height=3, gap=0.6, speed=3.0)
    b = scene["bodies"]
    s = E.scenes._assemble(np.array([[b["pos"][5, 0], 3.1, 0.0]], f32), np.array([[0, 0, 0, 1]], f32),
                           np.array([SHAPE_SPHERE], np.uint32), np.array([[0.3, 0, 0, 0]], f32), np.array([DYNAMIC], np.uint32))
    s["gravity"][:] = 0
    s["linvel"][:] = (-3.0, 0, 0)
    bodies = {k: np.concatenate([b[k], s[k]]) for k in b}
    bodies["material"] = np.array([RUBBER] * 3 + [STONE] * 3 + [FLOOR, NONE], np.uint32)
    return dict(scene, bodies=bodies, dynamic=7)


def test_handover_carries_sensors_and_ids(gpu, E):
    """The island hand-over moves the sensor bit and the material ids with the bodies: after the right stack and its
    sensor moved to rank 0, the sensor passes through the left stack untouched, and the points created there between
    RUBBER and STONE boxes take the table's entry, which both ranks hold."""
    if EMU:
        pytest.skip("the hand-over payloads live in torch CUDA tensors")
    import threading
    import torch
    from edyn_b200 import dist
    shared, out, errs = dist.ThreadComm.Shared(2), [], []
    steps = 60

    def body(rank):
        try:
            torch.cuda.set_device(0)
            scene = _handover_scene(E)
            owner = [0, 0, 0, 1, 1, 1, -1, 1]               # the sensor's island starts on rank 1; the floor is on both
            sw = dist.DeviceShardedWorld(scene, rank, 2, dist.ThreadComm(shared, rank), device=0, owner=owner, slack=1.0)
            sw.world.set_material_mixing([RUBBER], [STONE], [0.05], [0.0])
            for _ in range(steps):
                sw.step(1)
            w = sw.world
            out.append(dict(rank=rank, migrated_in=sw.migrated_in, entities=w.entities().copy(), state=w.download_state(),
                            contacts=w.contacts(), err=w.stats()["error_flags"]))
            sw.close()
        except BaseException as e:              # noqa: BLE001  (a dead rank must not leave its peer in the barrier)
            errs.append(e)
            shared.barrier.abort()
    ts = [threading.Thread(target=body, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=300)
    assert not errs, errs
    r0 = next(r for r in out if r["rank"] == 0)
    assert r0["migrated_in"] >= 4 and r0["err"] == 0, r0["migrated_in"]
    ent = r0["entities"]
    slot = {int(e): int(np.where(ent == e)[0][-1]) for e in range(8)}
    sensor = r0["state"]
    x0 = _handover_scene(E)["bodies"]["pos"][7, 0]
    assert np.array_equal(sensor["linvel"][slot[7]], np.array([-3.0, 0, 0], f32))            # never pushed, before or after the move
    assert abs(float(sensor["pos"][slot[7], 0]) - (x0 - 3.0 * steps / 60)) < 1e-3
    c, left, right = r0["contacts"], {slot[e] for e in range(3)}, {slot[e] for e in range(3, 6)}
    hit = [k for k, (a, b) in enumerate(c["pairs"].tolist()) if c["num"][k] and {a, b} & left and {a, b} & right]
    assert hit, "the stacks met on rank 0"
    for k in hit:
        pts = c["pts"][k, :c["num"][k]]
        assert np.all(pts[:, 13] == f32(0.05)) and np.all(pts[:, 14] == 0.0), pts[:, 13:15]
