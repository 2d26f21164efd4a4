"""Island tiles come in two classes: two-point tiles (no manifold with more than 2 points) run k_island_tiles_2p, the
others k_island_tiles.  A manifold of a two-point tile that gains a third point must move its island to a generic tile
through a rebuild in the same step.  Both classes, and the crossing, must give the bits of the dataflow path.
Also runs against the CPU emulation (B2D_EMU=1 B2D_LIB=tests/emu/_build/libb2d_emu.so), which launches plainly."""
import os

import numpy as np
import pytest

from tests.parity import build_world, same_state

pytestmark = pytest.mark.gpu

TIP_DEG = 40.0          # the tipping box stands on one edge, off balance: 2 contact points until it lands on a face


def _scene(E):
    """A slice of the chains workload (two-point islands), nine boxes resting flat (4-point islands) and one box on an
    edge that tips onto a face, all on one plane."""
    from edyn_b200.rigidbody import DYNAMIC, SHAPE_BOX
    scene = E.scenes.hinge_chains(8, 8, 4)
    a = np.radians(TIP_DEG)
    gx, gz = np.meshgrid(np.arange(3), np.arange(3), indexing="ij")
    flat = np.stack([2.0 + 1.5 * gx.ravel(), np.full(9, 0.501), 12.0 + 1.5 * gz.ravel()], axis=1)
    tip = np.array([[12.0, 0.5 * (np.sin(a) + np.cos(a)) + 0.002, 14.0]])
    orn = np.tile(np.array([0, 0, 0, 1], np.float32), (10, 1))
    orn[9] = (0, 0, np.sin(a / 2), np.cos(a / 2))
    boxes = E.scenes._assemble(np.concatenate([flat, tip]), orn, np.full(10, SHAPE_BOX, np.uint32),
                               np.tile(np.array([0.5, 0.5, 0.5, 0], np.float32), (10, 1)), np.full(10, DYNAMIC, np.uint32))
    b = scene["bodies"]
    scene["bodies"] = {k: np.concatenate([b[k], boxes[k]]) for k in b}
    return scene, len(b["kind"]) + 9


def _points(w, body):
    c = w.contacts()
    hit = np.nonzero((c["pairs"] == body).any(axis=1))[0]
    return int(c["num"][hit].max()) if len(hit) else 0


def test_two_point_tile_crossing(gpu, E):
    scene, box = _scene(E)
    reuse = build_world(E, scene, "graph")
    plain = build_world(E, scene, "plain")
    dataflow = build_world(E, scene, "graph", env=dict(B2D_TILES="0"))
    worlds = (reuse, plain, dataflow)
    crossing, history = None, []
    for step in range(150):
        r0 = reuse.stats()["steps_rebuilt"]
        for w in worlds:
            w.step(1)
        same_state(reuse, plain, dataflow)
        n = _points(reuse, box)
        rebuilt = reuse.stats()["steps_rebuilt"] - r0
        if crossing is None and history and 0 < history[-1][0] <= 2 < n:
            crossing = step
            assert rebuilt == 1, f"step {step}: the box's manifold went from {history[-1][0]} to {n} points without a rebuild"
        history.append((n, rebuilt))
    assert history[0][0] == 2, history[:5]                 # on its edge
    assert crossing is not None, [h[0] for h in history]
    assert history[-1][0] == 4                             # on a face
    st = reuse.stats()
    if os.environ.get("B2D_EMU") != "1":
        assert st["steps_reused"] > 100, st                 # otherwise settled: the rebuild is skipped
    for w in worlds:
        assert w.stats()["error_flags"] == 0
    tiles = reuse.debug_tiles()
    assert tiles["tiles"] >= 2, tiles                       # a two-point tile and a generic one
