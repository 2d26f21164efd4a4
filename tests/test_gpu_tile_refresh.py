"""The AABB and world-space inverse inertia of every body after each step, identical in every solver mode.  The island
tiles refresh their own bodies' (from the final pose and the body-space inverse inertia they hold on chip) and
k_finalize / k_integrate skip them; on the dataflow path k_finalize, or k_integrate without position iterations,
refreshes every body.  So tiles on and off must agree bit for bit on both, at every iteration setting, including the
one without position iterations.  Scenes: the island-tile capacity edges of tests/test_gpu_tile_edges.py (two-point
and generic tiles, joints, static and kinematic partners) and random scenes of tests/test_ref_stepper.py.  Also runs
against the CPU emulation (B2D_EMU=1), which has no graphs and runs fewer steps."""
import os

import numpy as np
import pytest

from tests import tile_packing as TP
from tests.parity import build_world
from tests.test_gpu_tile_edges import SCENES
from tests.test_ref_stepper import random_scene

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
STEPS = 20 if EMU else 60
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
ITERS = [(10, 3), (1, 0)] if EMU else [(10, 3), (1, 0), (20, 6)]
SEEDS = 2 if EMU else 6
KEYS = ("pos", "orn", "linvel", "angvel", "aabb", "inv_IW")


def _states(E, scene, mode, vi, pi):
    """Every step's full state (inverse world inertia included) of `scene` in `mode`, and how many steps ran tiles."""
    st = dict(scene["settings"], velocity_iterations=vi, position_iterations=pi)
    w = build_world(E, scene, mode, **st)
    pc = TP.PackingCheck(scene)
    out = []
    try:
        for s in range(STEPS):
            w.step(1)
            pc(s, w)
            g = w.download_state(aabb=True, inv_IW=True)
            out.append({k: g[k].copy() for k in KEYS})
        assert w.stats()["error_flags"] == 0
    finally:
        w.close()
    return out, pc.tiled_steps


def _same_in_every_mode(E, scene, vi, pi):
    ref, tiled = _states(E, scene, MODES[0], vi, pi)
    assert tiled > 0, f"{scene['name']}: no step ran the island tiles"
    assert np.abs(ref[-1]["inv_IW"]).max() > 0
    for mode in MODES[1:]:
        got, tiled = _states(E, scene, mode, vi, pi)
        if mode == "dataflow":
            assert tiled == 0
        for s, (a, b) in enumerate(zip(ref, got)):
            diff = [k for k in KEYS if a[k].tobytes() != b[k].tobytes()]
            assert not diff, f"{scene['name']} v{vi}p{pi}: {mode} differs from {MODES[0]} at step {s} in {diff}"


@pytest.mark.parametrize("iters", ITERS, ids=lambda it: f"v{it[0]}p{it[1]}")
@pytest.mark.parametrize("name", list(SCENES))
def test_tile_refresh_matches_dataflow_at_the_edges(gpu, E, name, iters):
    _same_in_every_mode(E, SCENES[name](E), *iters)


@pytest.mark.parametrize("seed", range(SEEDS))
def test_tile_refresh_matches_dataflow_random(gpu, E, O, seed):
    vi, pi = ITERS[seed % len(ITERS)]
    _same_in_every_mode(E, random_scene(E, O, seed), vi, pi)
