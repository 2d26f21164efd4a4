"""The random scenes of tests/test_ref_stepper.py (random_scene, random_scene_wide: kinematic platforms, tilted ground,
collision filters, hinges with arbitrary axes and pivots, 1-20 velocity and 0-6 position iterations) on the device, in
lock step with the oracle, in three modes: plain launches, CUDA graphs with rebuild reuse, dataflow only.  Every step:
the island-tile packing against its restatement (tests/tile_packing.py), ordered pair lists and island labels identical
to the oracle's, the state, contacts and hinge impulses bit-identical to the oracle replaying the device's order outside
the trig set of tests/parity.py, the three modes bit-identical to each other, no error flags.  One batched world puts 32 scenes side by
side, so dozens of tiles and the dataflow path run at once.  Also runs against the CPU emulation (B2D_EMU=1), with fewer
seeds and no graphs."""
import os

import numpy as np
import pytest

from tests import tile_packing as TP
from tests.parity import lockstep, report, same_digests
from tests.test_ref_stepper import random_scene, random_scene_wide

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
SEEDS = 3 if EMU else 32
STEPS = 60 if EMU else 150
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
NARROW_ITERS = [(10, 3), (1, 0), (20, 6)]


def _all_modes(E, O, scene, steps, **kw):
    """The lock step in every mode; returns the packing check of the plain launches."""
    digests, checks = {}, {}
    for mode in MODES:
        pc = checks[mode] = TP.PackingCheck(scene)
        res = lockstep(E, O, scene, steps, mode=mode, hook=pc, **kw)
        assert res["ok"], (scene["name"], mode, res)
        # nearly every body of these scenes spins at every step, so nearly every pose is in the trig set: what they hold
        # to bits is the velocities, contacts, hinge impulses, AABBs and inertias (the report line gives the split)
        report(f"{scene['name']} {mode}", res)
        assert pc.rebuilt + pc.reused == steps
        if mode == "dataflow":
            assert pc.tiled_steps == 0
        digests[f"{scene['name']} {mode}"] = res["digests"]
    same_digests(digests)
    return checks["plain"]


@pytest.mark.parametrize("seed", range(SEEDS))
def test_random_scene_lockstep(gpu, E, O, seed):
    vi, pi = NARROW_ITERS[seed % len(NARROW_ITERS)]
    _all_modes(E, O, random_scene(E, O, seed), STEPS, vel_iters=vi, pos_iters=pi)


@pytest.mark.parametrize("seed", range(SEEDS))
def test_random_scene_wide_lockstep(gpu, E, O, seed):
    _all_modes(E, O, random_scene_wide(E, O, seed), STEPS)


def batched_random_scenes(E, O, count=32, pitch=10.0):
    """`count` random_scene seeds on an 8-wide grid `pitch` metres apart, on one shared level plane; each scene's own
    plane is dropped, its hinges and exclusions are renumbered.  The first scene is crowded (200 bodies): its pile is
    an island too large for a tile, so the dataflow path runs next to the tiles."""
    parts, hinges, excl, base = [], [], [], 0
    for k in range(count):
        s = random_scene(E, O, 1000 + k, n=200 if k == 0 else 40)
        b = s["bodies"]
        keep = np.arange(len(b["kind"]) - 1)                 # the last body is the scene's ground plane
        part = {key: np.asarray(v)[keep].copy() for key, v in b.items() if v is not None}
        part["pos"][:, 0] += pitch * (k % 8)
        part["pos"][:, 2] += pitch * (k // 8)
        parts.append(part)
        h = s["hinges"]
        hinges.append({key: (v + base if key in ("a", "b") else v) for key, v in h.items()})
        excl.append((s["exclusions"][0] + base, s["exclusions"][1] + base))
        base += len(keep)
    plane = {key: np.asarray(v)[-1:] for key, v in s["bodies"].items() if v is not None}
    parts.append(plane)
    bodies = {key: np.concatenate([p[key] for p in parts]) for key in parts[0]}
    return dict(name=f"random_batch_{count}", bodies=bodies, hinges={key: np.concatenate([h[key] for h in hinges]) for key in hinges[0]},
                exclusions=(np.concatenate([e[0] for e in excl]).astype(np.uint32), np.concatenate([e[1] for e in excl]).astype(np.uint32)),
                dynamic=int((bodies["kind"] == 0).sum()), settings=dict(velocity_iterations=10, position_iterations=3))


def test_batched_random_scenes_lockstep(gpu, E, O):
    scene = batched_random_scenes(E, O, count=8 if EMU else 32)
    pc = _all_modes(E, O, scene, 40 if EMU else 100)
    # many tiles at once, and manifolds on the dataflow path in the same steps
    assert max(len(h["fill"]) for h in pc.history) >= (2 if EMU else 8), [len(h["fill"]) for h in pc.history]
    assert sum(h["dataflow"] > 0 and len(h["fill"]) > 1 for h in pc.history) >= len(pc.history) // 2, [h["dataflow"] for h in pc.history]
