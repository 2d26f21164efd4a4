"""Point-count transitions of live manifolds, which only the contact merge (np_merge) reports to the island rebuild through
Counters::graph_changed: a manifold that gains its first points (0 -> n), one that loses its last while it lives on
(n -> 0), one without an island tile whose count changes, and one that grows past 2 points inside a two-point tile,
which has no room for a third.  Nothing else flags them: the broadphase flags new manifolds only, and an upload of poses
does not flag at all.

The scene: boxes dropped onto the plane turned about a horizontal axis land on an edge (two points, a two-point tile) and
tip flat (3 or 4 points); a box rises slowly off a kinematic platform until its points are gone and, a few steps later,
its manifold; a box hops on a box resting on a kinematic platform, so that its manifold loses its points and regains them
while the island keeps its tile through the other manifold.

Every step, in three modes (plain launches, CUDA graphs that skip the rebuild while graph_changed is clear, dataflow only):
the oracle lock step of tests/emu/lockstep.py, the packing against its restatement (tests/tile_packing.py; in the graph
mode a skipped rebuild whose inputs changed fails there), and the modes bit-identical to each other.  Also, with the
step split after the narrowphase, graph_changed must be set on every step where one of those transitions happened: the
CPU emulation has no CUDA graphs, and that check is what it can see of a missing flag."""
import ctypes
import os

import numpy as np
import pytest

from tests import tile_packing as TP
from tests.emu.lockstep import build_world, lockstep
from tests.test_gpu_tile_edges import _Scene

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
STEPS = 90
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
f32 = np.float32
# Counters (edyn_b200/csrc/b2d_world.cuh) as b2d_debug_counters copies it: 28 words, coff / hoff / cchunk / hchunk of
# MAX_COLORS + 2 = 66 words each, npoff / npcount / npcursor of 16, then graph_changed.  The layout is private to the
# library, so test_graph_changed_follows_the_transitions first checks the word against what sets and clears it.
W_NNEW, W_GRAPH_CHANGED = 2, 28 + 4 * 66 + 48


def transitions_scene(E):
    from edyn_b200.rigidbody import KINEMATIC, SHAPE_BOX
    s = _Scene()
    h = 0.2
    tip = []
    for k, (ang, ax) in enumerate(((0.5, 0), (0.35, 2), (0.62, 0), (0.45, 2))):
        tip.append(s.body((3.0 * k, h * (np.cos(ang) + np.sin(ang)) + 0.005, 0.0), SHAPE_BOX, (h, h, h, 0)))
    # a box rising at 3 cm/s off a kinematic platform: points gone at 2 cm, the manifold at 2.6 cm (broadphase.hpp:18)
    s.body((0.0, 0.1, 6.0), SHAPE_BOX, (1.0, 0.1, 1.0, 0), KINEMATIC)
    riser = s.body((0.0, 0.2 + h, 6.0), SHAPE_BOX, (h, h, h, 0), linvel=(0, 0.03, 0))
    # a box hopping on a box that rests on a kinematic platform: 2.3 cm high, back after about 0.6 s
    s.body((6.0, 0.1, 6.0), SHAPE_BOX, (1.0, 0.1, 1.0, 0), KINEMATIC)
    base = s.body((6.0, 0.2 + 0.3, 6.0), SHAPE_BOX, (0.3, 0.3, 0.3, 0))
    hopper = s.body((6.0, 0.8 + h, 6.0), SHAPE_BOX, (h, h, h, 0), linvel=(0, 0.152, 0))
    scene = s.build(E, "point_transitions")
    b = scene["bodies"]
    for k, i in enumerate(tip):
        ang, ax = ((0.5, 0), (0.35, 2), (0.62, 0), (0.45, 2))[k]
        q = np.zeros(4, f32); q[ax] = np.sin(ang / 2); q[3] = np.cos(ang / 2)
        b["orn"][i] = q
    b["gravity"][riser] = 0.0
    b["gravity"][hopper] = (0.0, -0.5, 0.0)
    scene["roots"] = dict(tip=tip, riser=riser, hopper=hopper, base=base)
    return scene


class Transitions:
    """Per-step hook: the manifolds' point counts before and after each step, by ordered pair, and which transitions
    happened where (the tile of the manifold's island in the step before)."""

    def __init__(self, scene):
        self.pc = TP.PackingCheck(scene)
        self.prev, self.prev_tile, self.prev_n2, self.prev_dyn = {}, None, 0, None
        self.seen = {"0->n": 0, "n->0": 0, "2->3+ in a two-point tile": 0, "tile-less change": 0}

    def classify(self, now, n2):
        """The transitions from the last step's counts to `now` (dict pair -> points)."""
        out = []
        for p, n in now.items():
            if p not in self.prev or self.prev[p] == n:
                continue
            was = self.prev[p]
            key = p[0] if self.prev_dyn[p[0]] else p[1]
            tile = self.prev_tile[key]
            if was == 0:
                out.append("0->n")
            if n == 0:
                out.append("n->0")
            if tile == TP.TILE_NONE:
                out.append("tile-less change")
            if n > 2 and was <= 2 and tile != TP.TILE_NONE and tile < n2:
                out.append("2->3+ in a two-point tile")
        return out

    def counts(self, w):
        """After a narrowphase: the transitions since the last call."""
        c = w.contacts()
        now = {tuple(p): int(n) for p, n in zip(c["pairs"].tolist(), c["num"].tolist())}
        got = self.classify(now, self.prev_n2) if self.prev_tile is not None else []
        for t in got:
            self.seen[t] += 1
        self.prev = now
        return got

    def tiles(self, w):
        """After an island rebuild (or a step that reused one): the tiles the next narrowphase sees."""
        m = w.debug_tile_map()
        self.prev_tile, self.prev_n2 = m["btile"].astype(np.int64), m["ntiles2"]
        self.prev_dyn = w.islands() != TP.NO_ISLAND

    def __call__(self, step, w):
        self.pc(step, w)
        self.counts(w)
        self.tiles(w)


def test_point_transitions_lockstep(gpu, E, O):
    scene = transitions_scene(E)
    digests = {}
    for mode in MODES:
        tr = Transitions(scene)
        res = lockstep(E, O, scene, STEPS, mode=mode, hook=tr)
        assert res["ok"], (mode, res)
        assert tr.pc.rebuilt + tr.pc.reused == STEPS
        if mode == "plain":
            assert tr.pc.tiled_steps == STEPS
            for k in ("0->n", "n->0", "2->3+ in a two-point tile"):
                assert tr.seen[k] > 0, (k, tr.seen)
        if mode == "graph":
            assert res["reused"] > 0 and tr.pc.reused > 0, (res["reused"], tr.pc.reused)
        if mode == "dataflow":
            assert tr.pc.tiled_steps == 0 and tr.seen["tile-less change"] > 0, tr.seen
        digests[mode] = res["digests"]
    for mode in MODES[1:]:
        diff = [s for s, (a, b) in enumerate(zip(digests[MODES[0]], digests[mode])) if a != b]
        assert not diff, f"{mode} differs from {MODES[0]} from step {diff[0]} on"


def _counters(w):
    buf = np.zeros(W_GRAPH_CHANGED + 1, np.uint32)
    w._check(w.l.b2d_debug_counters(w.h, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes))
    return buf


@pytest.mark.parametrize("mode", ["plain", "dataflow"])
def test_graph_changed_follows_the_transitions(gpu, E, mode):
    """A step split after the narrowphase (b2d_run_phases: the same kernels as b2d_step without CUDA graphs): every step
    on which one of the merge's transitions happened leaves graph_changed set after the narrowphase, or the rebuild a
    graph step skips would run on stale inputs.  (The broadphase sets it too, for new and destroyed manifolds and for
    tile-less bodies that change cells, so a clear flag is not required elsewhere.)"""
    scene = transitions_scene(E)
    w = build_world(E, scene, mode, **scene["settings"])
    PH = E.world
    tr = Transitions(scene)
    w.run_phases(PH.PH_ALL)
    assert _counters(w)[W_GRAPH_CHANGED] == 0                     # cleared by the rebuild (solver phase)
    c = w.contacts()
    w.upload_contacts(c["pairs"], c["num"], c["pts"], c["att"], c["lifetime"])
    assert _counters(w)[W_GRAPH_CHANGED] != 0                     # set by an upload
    tr.counts(w)
    tr.tiles(w)
    flagged = 0
    for s in range(STEPS):
        w.run_phases(PH.PH_BROAD | PH.PH_NARROW)
        got = tr.counts(w)
        if got:
            assert _counters(w)[W_GRAPH_CHANGED] != 0, f"step {s}: {got} without graph_changed"
            flagged += 1
        w.run_phases(PH.PH_ISLANDS | PH.PH_SOLVE)
        tr.tiles(w)
    assert flagged > 0
    if mode == "plain":
        assert all(tr.seen[k] > 0 for k in ("0->n", "n->0", "2->3+ in a two-point tile")), tr.seen
    else:
        assert tr.seen["tile-less change"] > 0, tr.seen
    w.close()
