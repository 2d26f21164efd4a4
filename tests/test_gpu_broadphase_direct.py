"""The broadphase's direct cell table, against the cell hash and a brute-force pair search.

Each step, k_bp_cell_mode picks the cell lookup from the box of occupied key fields: the direct table (Dev::cstart, one
word per cell of the box, DENSE_CELLS_PER_BODY cells per body) when the box fits it, the cell hash otherwise.  The table
is never cleared: a reader accepts an entry only if it indexes a body of this step with the looked-up key, so entries
left by bodies that moved, by an earlier box or by removed bodies must all be turned away.

Every scene runs twice, with the table and without it (B2D_BP_CELL_TABLE=0: the cell hash on every step, the search as
it was before the table), and each run is held to:
  * every step's manifold pairs against `brute_force_broadphase` (tests/test_gpu_broadphase_edges.py), over the AABBs
    and the manifolds the step started from;
  * the mode the device chose (Counters::bp_direct) against the scene's design or a restatement of the occupied box;
and the two runs to each other: manifold pairs in slot order, contact points, and the body state with AABBs and inv_IW,
bit for bit after every step.  Scenes: bodies crossing cells, a world whose box outgrows the table and shrinks back,
removed bodies, and the clamped-key placements of the edge tests.  Each runs under plain launches and the step's CUDA
graph, with both search mappings.  test_under_emulation runs this file's gpu tests against the CPU emulation (tests/emu)."""
import ctypes
import hashlib
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

from tests import test_gpu_broadphase_edges as EDGES
from tests.parity import build_world

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.environ.get("B2D_EMU") == "1"
LAUNCHES = ["plain"] if EMU else ["plain", "graph"]
SEARCH = EDGES.SEARCH
HASH = {"B2D_BP_CELL_TABLE": "0"}
F32 = np.float32
R_SPHERE = 0.25
# Counters (edyn_b200/csrc/b2d_world.cuh) as b2d_debug_counters copies it: graph_changed at word 340 (see
# tests/test_gpu_point_transitions.py), steps_rebuilt and steps_reused from word 342, dbg[16] from word 346, then bp_direct
W_BP_DIRECT = 378


@pytest.fixture
def counters():
    def bp_direct(w):
        buf = np.zeros(W_BP_DIRECT + 1, np.uint32)
        w._check(w.l.b2d_debug_counters(w.h, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes))
        return int(buf[W_BP_DIRECT])
    return bp_direct


def _scene(bodies):
    return dict(bodies=bodies, hinges=None, exclusions=None, settings=dict(velocity_iterations=4, position_iterations=2))


def _digest(w):
    st = w.download_state(aabb=True, inv_IW=True)
    c = w.contacts()
    h = hashlib.sha256()
    for a in (w.pairs(), st["pos"], st["orn"], st["linvel"], st["angvel"], st["aabb"], st["inv_IW"], c["pairs"], c["num"], c["pts"]):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def run_steps(E, scene, launch, env, steps, counters, before_step=None):
    """Steps `scene` one step at a time.  before_step(w, s) may move or remove bodies and returns the removed mask.
    Per step: the mode the device chose, the pairs in slot order, the state digest; every step's pairs are checked
    against the brute force."""
    b = scene["bodies"]
    w = build_world(E, scene, launch, env)
    removed = np.zeros(len(b["kind"]), bool)
    modes, pairs, digests, aabbs = [], [], [], []
    try:
        before = []
        for s in range(steps):
            if before_step is not None:
                removed = before_step(w, s)
            bb = w.download_state()["aabb"]
            w.step(1)
            got = w.pairs().tolist()
            want = EDGES.brute_force_broadphase(bb, b["kind"], b["shape_kind"], removed=removed, manifolds=before)
            assert Counter(map(tuple, got)) == want, f"step {s}: extra {dict(Counter(map(tuple, got)) - want)}, missing {dict(want - Counter(map(tuple, got)))}"
            modes.append(counters(w)); pairs.append(got); digests.append(_digest(w)); aabbs.append(bb)
            before = got
        assert w.stats()["error_flags"] == 0
    finally:
        w.close()
    return modes, pairs, digests, aabbs


def same_as_hash(E, scene, launch, search, steps, counters, before_step=None, table=None):
    """The scene with the direct table (default size, or `table` cells per body) and with the cell hash only: the
    modes, pairs and AABBs of the first run, after both matched each other step by step."""
    env = {**SEARCH[search], **({"B2D_BP_CELL_TABLE": str(table)} if table else {})}
    m1, p1, d1, bb = run_steps(E, scene, launch, env, steps, counters, before_step)
    m0, p0, d0, _ = run_steps(E, scene, launch, {**SEARCH[search], **HASH}, steps, counters, before_step)
    assert not any(m0), "B2D_BP_CELL_TABLE=0 still used the direct table"
    for s in range(steps):
        assert p1[s] == p0[s], f"step {s}: manifold pairs or slots differ from the cell hash"
        assert d1[s] == d0[s], f"step {s}: state or contacts differ from the cell hash"
    return m1, p1, bb


def restated_modes(aabbs, table):
    """The mode each step should take: the occupied box of key fields (measured from the first step's AABBs, cells
    clamped to them; every body here is a grid body) against `table` cells per body."""
    cell = EDGES._cell_pitch(2 * R_SPHERE)
    n = len(aabbs[0])
    lo, hi = EDGES.key_box(aabbs[0], cell, np.arange(n))
    out = []
    for bb in aabbs:
        c = np.clip(np.floor((bb[:, :3] + bb[:, 3:]) * F32(0.5) / F32(cell)).astype(np.int64), lo, hi)
        out.append(int(np.prod(c.max(0) - c.min(0) + 1) <= table * n))
    return out


def _lattice(R, shape, spacing, origin, rng, speed):
    defs = []
    for i in np.ndindex(*shape):
        p = np.asarray(origin, np.float64) + np.array(i) * spacing
        defs.append(R.RigidBodyDef(position=tuple(p.tolist()), gravity=(0, 0, 0), shape=R.sphere_shape(R_SPHERE),
                                   linvel=tuple(rng.uniform(-speed, speed, 3).tolist())))
    return defs


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("search", list(SEARCH))
def test_bodies_crossing_cells(gpu, E, counters, launch, search):
    """A lattice of spheres flying apart through each other at up to 6 m/s: bodies leave cells every few steps, so the
    table keeps entries of cells that emptied, and the box (hence the linearisation) changes as the lattice spreads.
    A table of 256 cells per body keeps the direct mode all the way."""
    R = E.rigidbody
    rng = np.random.default_rng(5)
    defs = _lattice(R, (6, 3, 6), 0.6, (0.0, 0.0, 0.0), rng, 6.0)
    scene = _scene(R.bodies_soa(defs))
    steps = 24 if EMU else 48
    modes, pairs, aabbs = same_as_hash(E, scene, launch, search, steps, counters, table=256)
    assert modes == restated_modes(aabbs, 256) and all(modes)
    assert sum(len(p) for p in pairs) > 50


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("search", list(SEARCH))
def test_box_outgrows_the_table_and_shrinks_back(gpu, E, counters, launch, search):
    """Touching clusters and one sphere that is moved 16 m away and back between steps: while it is away the occupied
    box has far more cells than 4 per body and the step uses the cell hash; when it is back, the direct table, whose
    entries were written under the earlier, smaller box."""
    R = E.rigidbody
    defs = []
    for c in ((0.0, 0.0, 0.0), (2.0, 0.0, 0.0), (0.0, 0.0, 2.0)):
        for i in np.ndindex(2, 2, 2):
            p = np.asarray(c) + np.array(i) * EDGES.GAP
            defs.append(R.RigidBodyDef(position=tuple(p.tolist()), gravity=(0, 0, 0), shape=R.sphere_shape(R_SPHERE)))
    home = (1.2, 0.0, 1.2)
    wanderer = len(defs)
    defs.append(R.RigidBodyDef(position=home, gravity=(0, 0, 0), shape=R.sphere_shape(R_SPHERE)))
    scene = _scene(R.bodies_soa(defs))
    away = {3: (17.2, 16.0, 17.2), 6: home, 9: (-14.8, -16.0, 1.2), 12: home}

    def move(w, s):
        if s in away:
            w.upload_bodies([wanderer], pos=np.array([away[s]], F32), linvel=np.zeros((1, 3), F32))
        return np.zeros(len(defs), bool)

    modes, pairs, aabbs = same_as_hash(E, scene, launch, search, 16, counters, move)
    assert modes == restated_modes(aabbs, 4)
    assert [modes[s] for s in sorted(away)] == [0, 1, 0, 1]
    assert all(len(p) >= 3 * 28 for p in pairs)


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("search", list(SEARCH))
def test_removed_bodies(gpu, E, counters, launch, search):
    """A settling lattice of touching spheres loses a third of its bodies, the lowest sorted ones among them, then
    more: removed bodies leave the grid (their keys sort to the end), so table entries of the cells they held now name
    sorted indices of other cells or of the shapeless tail."""
    R = E.rigidbody
    rng = np.random.default_rng(7)
    defs = _lattice(R, (5, 3, 5), EDGES.GAP, (0.0, 0.0, 0.0), rng, 0.3)
    n = len(defs)
    scene = _scene(R.bodies_soa(defs))
    first = np.arange(0, n, 3)
    plan = {4: first, 8: np.setdiff1d(np.arange(1, 20), first)}

    def remove(w, s):
        if s in plan:
            w.remove_bodies(plan[s])
        removed = np.zeros(n, bool)
        for k, ids in plan.items():
            removed[ids] |= k <= s
        return removed

    modes, pairs, _ = same_as_hash(E, scene, launch, search, 12, counters, remove)
    assert all(modes)
    assert len(pairs[-1]) > 0 and len(pairs[-1]) < len(pairs[3])


def broadphase_after_move(E, S, launch, env, counters):
    """EDGES.run_case with the mode and the pairs in slot order: add_bodies, one PH_BROAD (measures the key fields),
    upload_state to the targets, one step, checked against the brute force."""
    b = S.R.bodies_soa(S.defs)
    nb = len(S.defs)
    w = build_world(E, _scene(b), launch, env, max_manifolds=max(4096, 40 * nb))
    try:
        w.run_phases(E.world.PH_BROAD)
        first = w.pairs().tolist()
        st = w.download_state()
        pos = st["pos"].copy()
        for i, t in enumerate(S.target):
            if t is not None:
                pos[i] = t
        w.upload_state(pos, st["orn"], st["linvel"], st["angvel"])
        st = w.download_state()
        w.step(1)
        got = w.pairs().tolist()
        want = EDGES.brute_force_broadphase(st["aabb"], b["kind"], b["shape_kind"], manifolds=first)
        EDGES._check(Counter(map(tuple, got)), want, 28 * sum(t is not None for t in S.target) // 8)
        assert w.stats()["error_flags"] == 0
        return counters(w), got, _digest(w)
    finally:
        w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("search", list(SEARCH))
@pytest.mark.parametrize("kind", ["faces", "edges", "corners", "boundary"])
def test_clamped_placements(gpu, E, counters, launch, search, kind):
    """Clusters past the faces, edges and corners of the measured key box and on its first and last fields, as in
    test_gpu_broadphase_edges.py: the occupied box is then the whole key box (62 x 63 x 63 cells at most), so a table
    of 8192 cells per body holds it (the scenes have 50 to 98 bodies) and the direct lookup meets every clamped cell; against the cell hash."""
    cell = EDGES._cell_pitch(2 * R_SPHERE)

    def scene():
        S = EDGES.Scene(E)
        centres = EDGES.placements(kind, cell)
        park = EDGES.frame(S, EDGES.LO, EDGES.HI, cell, 8 * len(centres))
        for c in centres:
            EDGES.cluster(S, c, cell)
        for d, p in zip(S.defs[2:], park):
            d.position = p
        return S

    m1, p1, d1 = broadphase_after_move(E, scene(), launch, {**SEARCH[search], "B2D_BP_CELL_TABLE": "8192"}, counters)
    m0, p0, d0 = broadphase_after_move(E, scene(), launch, {**SEARCH[search], **HASH}, counters)
    assert (m1, m0) == (1, 0)
    assert p1 == p0 and d1 == d0


def test_under_emulation():
    """This file's gpu tests against the CPU emulation of tests/emu (plain launches only)."""
    from tests.emu import build as B
    env = dict(os.environ, B2D_EMU="1", B2D_LIB=B.build(), B2D_GRAPH="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout, r.stdout[-1000:]
