"""The island tiles at their capacity edges, in lock step with the oracle.  An island is tiled when it has at most 128
dynamic bodies, manifolds with points and joints; tiles hold at most 256 of each (tests/tile_packing.py restates the
packing).  These scenes put islands at 127 / 128 / 129 on each count, fill a two-point tile and a generic tile to all 256
lanes (bodies, manifolds, the points-3/4 block, the joint rows), hang a chain from a static anchor (joints only, the
static-partner path of the position iterations), rest a chain on a moving kinematic platform, run an island that needs
several position iterations next to one that stops after the first in the same tile, and alternate two-point and
generic islands in root order.

Every step of every scene, in three modes (plain launches, CUDA graphs with rebuild reuse, dataflow only) and at three
iteration settings ((1, 0): the tile kernel without position iterations): the packing against the restatement, the oracle lock step of
tests/parity.py, and the three modes bit-identical to each other.  Also runs against the CPU emulation
(B2D_EMU=1), which has no graphs and runs fewer steps."""
import os

import numpy as np
import pytest

from tests import tile_packing as TP
from tests.parity import lockstep, report, same_digests

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
STEPS = 40 if EMU else 100
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
ITERS = [(10, 3), (1, 0)] if EMU else [(10, 3), (1, 0), (20, 6)]
f32 = np.float32
CAPSULE = (0.1, 0.25, 0.0, 0.0)         # the chains workload's links: 0.7 m long along x, hinged at the tips
BOX = (0.2, 0.2, 0.2, 0.0)


class _Scene:
    """Bodies, hinges and exclusions, appended part by part."""

    def __init__(self):
        self.rows, self.hinges, self.excl, self.roots = [], [], [], {}

    def body(self, pos, shape_kind, params, kind=0, linvel=(0, 0, 0), angvel=(0, 0, 0)):
        self.rows.append((pos, shape_kind, params, kind, linvel, angvel))
        return len(self.rows) - 1

    def hinge(self, a, b, pa, pb, axis=(0, 0, 1)):
        self.hinges.append((a, b, pa, pb, axis))

    def chain(self, name, x0, y, z, links, shape_kind, params, spacing, joints=None, vz=0.5):
        """A straight chain along x, links hinged tip to tip about z, neighbours excluded from colliding.  joints: hinge
        count (default links - 1; more doubles hinges from the first one on).  Each link gets its own sideways velocity."""
        from edyn_b200.rigidbody import DYNAMIC
        ids = [self.body((x0 + spacing * k, y, z), shape_kind, params, DYNAMIC, linvel=(0.2, 0, vz * np.sin(0.37 * k)),
                         angvel=(0, 0.3 * np.cos(0.23 * k), 0)) for k in range(links)]
        pairs = [(ids[k], ids[k + 1]) for k in range(links - 1)]
        joints = links - 1 if joints is None else joints
        for j in range(joints):
            a, b = pairs[j % len(pairs)]
            self.hinge(a, b, (spacing / 2, 0, 0), (-spacing / 2, 0, 0))
        self.excl += pairs
        self.roots[name] = ids[0]
        return ids

    def capsule_chain(self, name, x0, links, y=0.5, z=0.0, **kw):
        from edyn_b200.rigidbody import SHAPE_CAPSULE
        return self.chain(name, x0, y, z, links, SHAPE_CAPSULE, CAPSULE, 0.7, **kw)

    def box_train(self, name, x0, links, y=0.5, z=0.0, vz=0.2, **kw):
        from edyn_b200.rigidbody import SHAPE_BOX
        return self.chain(name, x0, y, z, links, SHAPE_BOX, BOX, 0.5, vz=vz, **kw)

    def build(self, E, name, plane=True):
        from edyn_b200.rigidbody import SHAPE_PLANE, STATIC
        if plane:
            self.body((0, 0, 0), SHAPE_PLANE, (0, 1, 0, 0), STATIC)
        pos, sk, par, kind, lv, av = (np.array([r[i] for r in self.rows]) for i in range(6))
        n = len(pos)
        b = E.scenes._assemble(pos.astype(f32), np.tile(np.array([0, 0, 0, 1], f32), (n, 1)), sk.astype(np.uint32), par.astype(f32), kind.astype(np.uint32))
        b["linvel"][:] = lv.astype(f32)
        b["angvel"][:] = av.astype(f32)
        h = self.hinges
        hinges = dict(a=np.array([x[0] for x in h], np.uint32), b=np.array([x[1] for x in h], np.uint32),
                      pivot_a=np.array([x[2] for x in h], f32), pivot_b=np.array([x[3] for x in h], f32),
                      axis_a=np.array([x[4] for x in h], f32), axis_b=np.array([x[4] for x in h], f32)) if h else None
        ex = (np.array([p[0] for p in self.excl], np.uint32), np.array([p[1] for p in self.excl], np.uint32)) if self.excl else None
        return dict(name=name, bodies=b, hinges=hinges, exclusions=ex, dynamic=int((kind == 0).sum()),
                    settings=dict(velocity_iterations=10, position_iterations=3), roots=dict(self.roots))


def two_point_scene(E):
    """Capsule chains dropped onto the plane.  A lone capsule, then three 128-link chains: the lone capsule and the first
    chain share tile 0 (129), the next two fill tile 1 to 256 bodies and 256 two-point manifolds (the prefix sum reaches
    the second chain at 129 = g).  A 127-link chain is tiled; a 129-link chain, and a 128-link chain with a static box
    against one link (129 manifolds), go to the dataflow path."""
    from edyn_b200.rigidbody import SHAPE_BOX, SHAPE_CAPSULE, STATIC
    s = _Scene()
    s.roots["lone"] = s.body((-3.0, 0.5, 0.0), SHAPE_CAPSULE, CAPSULE, linvel=(0.3, 0, 0.4))
    for i, (name, links) in enumerate((("full_a", 128), ("full_b", 128), ("full_c", 128), ("c127", 127), ("c129", 129), ("boxed", 128))):
        s.capsule_chain(name, 0.0, links, z=2.0 * (i + 1))
    # a static slab beside link 40 of the last chain, touching it once the chain lies on the plane
    s.body((0.7 * 40, 0.1, 12.0 + 0.1 + 0.2 - 0.004), SHAPE_BOX, (0.3, 0.1, 0.2, 0), STATIC)
    return s.build(E, "two_point_edges")


def generic_and_joint_scene(E):
    """Two-point and generic islands alternate in root order: a 128-box train (4-point manifolds), a 65-link capsule chain
    with every hinge doubled (128 joints), a second box train, a second doubled chain, then a doubled chain with one more
    hinge (129 joints: dataflow).  The trains fill a generic tile (256 bodies, manifolds and points-3/4 rows, 254 joints),
    the doubled chains a two-point tile's 256 joint lanes."""
    s = _Scene()
    s.box_train("train_a", 0.0, 128, y=0.35)
    s.capsule_chain("joints_a", 0.0, 65, z=2.0, joints=128)
    s.box_train("train_b", 0.0, 128, y=0.35, z=4.0)
    s.capsule_chain("joints_b", 0.0, 65, z=6.0, joints=128)
    s.capsule_chain("joints_129", 0.0, 65, z=8.0, joints=129)
    return s.build(E, "generic_and_joint_edges")


def partner_scene(E):
    """A capsule chain hinged to a static anchor, swinging in the air (a tile of joints only, whose position iterations
    read the anchor's pose), a chain resting on a moving, turning kinematic platform, and two box trains in one generic
    tile: one starting 4 cm into the plane (several position iterations), one resting on it (done after the first)."""
    from edyn_b200.rigidbody import KINEMATIC, SHAPE_BOX, SHAPE_SPHERE, STATIC
    s = _Scene()
    anchor = s.body((20.0, 10.0, 3.0), SHAPE_SPHERE, (0.1, 0, 0, 0), STATIC)
    ids = s.capsule_chain("swing", 20.35, 12, y=10.0, z=3.0, vz=0.0)
    s.hinge(anchor, ids[0], (0, 0, 0), (-0.35, 0, 0))
    s.excl.append((anchor, ids[0]))
    s.body((30.0, 0.3, 0.0), SHAPE_BOX, (3.0, 0.1, 1.0, 0), KINEMATIC, linvel=(0.6, 0, 0.2), angvel=(0, 0.25, 0))
    s.capsule_chain("riding", 28.6, 5, y=0.52, z=0.0, vz=0.0)
    s.box_train("sunk", 0.0, 6, y=0.16, z=10.0, vz=0.0)
    s.box_train("resting", 0.0, 6, y=0.2, z=12.0, vz=0.0)
    return s.build(E, "partner_edges")


SCENES = {"two_point": two_point_scene, "generic_joints": generic_and_joint_scene, "partners": partner_scene}


def _placement(name, pc, roots):
    """The scene reaches the edges it was built for (once everything has landed)."""
    last = pc.history[-1]
    tile, n2 = last["tile"], last["ntiles2"]
    fill = np.stack([h["fill"].max(axis=0) if len(h["fill"]) else np.zeros(3, np.int64) for h in pc.history]).max(axis=0)

    def cls(r):
        t = tile[roots[r]]
        return "none" if t == TP.TILE_NONE else ("two" if t < n2 else "generic")
    if name == "two_point":
        assert [cls(r) for r in ("lone", "full_a", "full_b", "full_c", "c127", "c129")] == ["two"] * 5 + ["none"]
        assert tile[roots["full_b"]] == tile[roots["full_c"]] != tile[roots["full_a"]]
        assert tuple(fill[:2]) == (256, 256), fill
        boxed = [(h["weight"][roots["boxed"]], h["tile"][roots["boxed"]]) for h in pc.history]
        assert (0, TP.TILE_NONE) in boxed and (128, TP.TILE_NONE) not in boxed, boxed
    elif name == "generic_joints":
        assert [cls(r) for r in ("train_a", "joints_a", "train_b", "joints_b", "joints_129")] == ["generic", "two", "generic", "two", "none"]
        assert tile[roots["train_a"]] == tile[roots["train_b"]] and tile[roots["joints_a"]] == tile[roots["joints_b"]]
        full = [h["fill"][tile[roots["train_a"]]] for h in pc.history]
        assert max(tuple(f) for f in full) == (256, 256, 254), full[-1]
        assert max(h["fill"][tile[roots["joints_a"]]][2] for h in pc.history) == 256
    else:
        assert [cls(r) for r in ("swing", "riding", "sunk", "resting")] == ["two", "two", "generic", "generic"]
        assert tile[roots["sunk"]] == tile[roots["resting"]]


def _run(E, O, scene, mode, vi, pi):
    pc = TP.PackingCheck(scene)
    res = lockstep(E, O, scene, STEPS, mode=mode, hook=pc, vel_iters=vi, pos_iters=pi)
    return res, pc


@pytest.mark.parametrize("iters", ITERS, ids=lambda it: f"v{it[0]}p{it[1]}")
@pytest.mark.parametrize("name", list(SCENES))
def test_tile_edges_lockstep(gpu, E, O, name, iters):
    scene = SCENES[name](E)
    vi, pi = iters
    digests = {}
    for mode in MODES:
        res, pc = _run(E, O, scene, mode, vi, pi)
        assert res["ok"], (mode, res)
        # the two-point and generic-joint scenes keep most bodies spinning, so most of their poses are in the trig set of
        # tests/parity.py (the report line gives the split); their velocities, contacts and impulses are held to bits
        report(f"{name} v{vi}p{pi} {mode}", res)
        assert pc.rebuilt + pc.reused == STEPS
        if mode == "plain":
            _placement(name, pc, scene["roots"])
            assert pc.tiled_steps == STEPS
        if mode == "graph":
            assert res["reused"] > 0 and pc.reused > 0, (res["reused"], pc.reused)
        if mode == "dataflow":
            assert pc.tiled_steps == 0
        digests[mode] = res["digests"]
    same_digests(digests)
