"""The broadphase's count pass over half the neighbourhood, against the count pass over the whole of it.

The thread-per-body count pass (k_bp_pairs<count>) lets the grid body at sorted index t meet only the records after it,
so each pair of grid bodies is evaluated once, from the side the whole walk would evaluate it (the higher-id dynamic
body, or the dynamic one); a pair whose query body is the other record is counted there with an atomicAdd.  Static and
kinematic grid bodies walk too.  The large list is screened by lmask: a bit set by k_bp_separate for a manifold alive
with large_list[k] (k < 32) skips the candidate without a probe of the manifold hash.

Every scene is stepped by two worlds side by side, one with the half walk (the default) and one with the whole walk
(B2D_BP_HALF=0), both with a thread per query body (B2D_BP_WARP_MAX=0).  After every step each must report the count
pass it ran (Counters::bp_count_walk), and they must agree on the
per-body new-pair counts (newcount), the manifold pairs in slot order (newpairs and the slots they went to), the body
state with AABBs and inv_IW, and the contacts, bit for bit.  Scenes: the four bench.py workloads at small scale; random
scenes with exclusions, collision filters, static and kinematic bodies in the grid, a large dynamic body, thrown bodies,
and fewer or more than 32 large bodies; and the clamped-key placements of tests/test_gpu_broadphase_edges.py.
test_under_emulation runs this file's gpu tests against the CPU emulation (tests/emu)."""
import ctypes
import hashlib
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

import bench
from tests import test_gpu_broadphase_edges as EDGES
from tests.parity import build_world

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.environ.get("B2D_EMU") == "1"
LAUNCHES = ["plain"] if EMU else ["plain", "graph"]
THREAD = {"B2D_BP_WARP_MAX": "0"}
HALF, WHOLE = {**THREAD, "B2D_BP_HALF": "1"}, {**THREAD, "B2D_BP_HALF": "0"}
F32 = np.float32
# Counters::bp_count_walk (edyn_b200/csrc/b2d_world.cuh) as b2d_debug_counters copies it: the word after bp_direct
# (tests/test_gpu_broadphase_direct.py); 2 when the last count pass walked half the neighbourhood, 1 the whole
W_BP_COUNT_WALK = 379


def count_walk(w):
    buf = np.zeros(W_BP_COUNT_WALK + 1, np.uint32)
    w._check(w.l.b2d_debug_counters(w.h, buf.ctypes.data_as(ctypes.c_void_p), buf.nbytes))
    return int(buf[W_BP_COUNT_WALK])


def same_step(s, wh, ww):
    """The half-walk world wh and the whole-walk world ww after step s: each ran the count pass it was built with, and
    both have the same newcount, manifold pairs in slot order, state and contacts.  Returns wh's pairs and newcount."""
    assert (count_walk(wh), count_walk(ww)) == (2, 1), f"step {s}: the count passes were not the half and the whole walk"
    nh, nw = wh.debug_newcount(), ww.debug_newcount()
    assert np.array_equal(nh, nw), f"step {s}: newcount differs at bodies {np.nonzero(nh != nw)[0][:10].tolist()}"
    ph = wh.pairs().tolist()
    assert ph == ww.pairs().tolist(), f"step {s}: manifold pairs or slots differ"
    assert _digest(wh) == _digest(ww), f"step {s}: state or contacts differ"
    return ph, nh


def _digest(w):
    st = w.download_state(aabb=True, inv_IW=True)
    c = w.contacts()
    h = hashlib.sha256()
    for a in (st["pos"], st["orn"], st["linvel"], st["angvel"], st["aabb"], st["inv_IW"], c["pairs"], c["num"], c["pts"]):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def lockstep(E, scene, launch, steps, max_manifolds=None, check=None):
    """Steps `scene` in a half-walk and a whole-walk world side by side; after every step both must have the same newcount,
    manifold pairs in slot order, state and contacts.  check(step, aabb_before, pairs_before, pairs) may hold the step to
    more.  Returns the new pairs counted per step."""
    kw = {} if max_manifolds is None else dict(max_manifolds=max_manifolds)
    wh = build_world(E, scene, launch, HALF, **kw)
    ww = build_world(E, scene, launch, WHOLE, **kw)
    found, before = [], []
    try:
        for s in range(steps):
            bb = wh.download_state()["aabb"]
            wh.step(1); ww.step(1)
            ph, nh = same_step(s, wh, ww)
            if check is not None:
                check(s, bb, before, ph)
            found.append(int(nh.sum()))
            before = ph
        assert wh.stats()["error_flags"] == 0 and ww.stats()["error_flags"] == 0
    finally:
        wh.close(); ww.close()
    return found


# ----------------------------------------------------------------------------- the bench.py workloads

SCALES = {"boxes_4096": 1 / 64, "spheres_65536": 1 / 1024, "mixed_262144": 1 / 4096, "chains_1048576": 1 / 16384} if EMU else \
         {"boxes_4096": 1 / 8, "spheres_65536": 1 / 64, "mixed_262144": 1 / 512, "chains_1048576": 1 / 256}


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("workload", list(SCALES))
def test_bench_workloads(gpu, E, launch, workload):
    """Each bench.py workload at small scale, from its first step (bodies dropped onto the ground: new pairs for several
    steps) into contact."""
    scene = bench.make_scene(workload, SCALES[workload])
    n = len(scene["bodies"]["kind"])
    found = lockstep(E, scene, launch, 16 if EMU else 40, max_manifolds=bench.capacity(workload, n))
    assert sum(found[1:]) > 0, found


# ----------------------------------------------------------------------------- random scenes

def random_scene(E, seed, n_large):
    """Dynamic spheres, boxes and capsules thrown into a pile, a third with collision filters; static and kinematic
    bodies of grid size among them; a large dynamic box (over 4 x the mean dynamic diameter) dropped onto the pile; a
    ground plane and n_large - 2 more large static boxes around it (more than 32 large bodies: the lmask bits run out
    and the rest of the large list is probed); exclusions between neighbours in creation order."""
    R = E.rigidbody
    rng = np.random.default_rng(seed)
    n = 40 if EMU else 160
    defs = []
    for _ in range(n):
        shape = [R.sphere_shape(float(rng.uniform(0.1, 0.3))), R.box_shape(tuple(rng.uniform(0.08, 0.25, 3))),
                 R.capsule_shape(float(rng.uniform(0.08, 0.15)), float(rng.uniform(0.1, 0.2)), int(rng.integers(3)))][rng.integers(3)]
        q = rng.normal(size=4)
        d = R.RigidBodyDef(position=tuple(rng.uniform([-1.5, 0.2, -1.5], [1.5, 3.0, 1.5]).tolist()),
                           orientation=tuple((q / np.linalg.norm(q)).tolist()), linvel=tuple(rng.uniform(-3, 3, 3).tolist()),
                           angvel=tuple(rng.uniform(-3, 3, 3).tolist()), shape=shape)
        if rng.random() < 0.3:
            d.collision_group, d.collision_mask = int(rng.choice([1, 2, 4])), int(rng.choice([1, 3, 6, 7]))
        defs.append(d)
    for k in range(6):
        defs.append(R.RigidBodyDef(kind=R.STATIC if k % 2 else R.KINEMATIC, position=tuple(rng.uniform([-1.2, 0.2, -1.2], [1.2, 1.5, 1.2]).tolist()),
                                   linvel=tuple(rng.uniform(-0.5, 0.5, 3).tolist()) if k % 2 == 0 else (0, 0, 0),
                                   shape=R.sphere_shape(0.25) if k % 3 else R.box_shape((0.2, 0.15, 0.2))))
    defs.append(R.RigidBodyDef(position=(0.0, 4.5, 0.0), linvel=(0.0, -4.0, 0.0), shape=R.box_shape((0.9, 0.3, 0.9)), mass=20.0))
    defs.append(R.RigidBodyDef(kind=R.STATIC, shape=R.plane_shape((0, 1, 0), 0.0)))
    for k in range(n_large - 2):
        a = 2 * np.pi * k / max(1, n_large - 2)
        defs.append(R.RigidBodyDef(kind=R.STATIC, position=(float(2.6 * np.cos(a)), 0.5, float(2.6 * np.sin(a))),
                                   shape=R.box_shape((0.9, 0.5, 0.9))))
    ids = np.arange(n - 1, dtype=np.uint32)
    pick = ids[rng.random(n - 1) < 0.25]
    scene = dict(bodies=R.bodies_soa(defs), hinges=None, exclusions=(pick.copy(), pick + np.uint32(1)),
                 settings=dict(velocity_iterations=6, position_iterations=2))
    return scene


@pytest.mark.gpu
@pytest.mark.parametrize("launch", LAUNCHES)
@pytest.mark.parametrize("n_large", [4, 40])
@pytest.mark.parametrize("seed", range(1 if EMU else 3))
def test_random_scenes(gpu, E, launch, n_large, seed):
    """Random scenes (random_scene) for 24 steps: besides agreeing with the whole walk, every step's pairs are the brute
    force's (tests/test_gpu_broadphase_edges.py) over the AABBs and manifolds the step started from."""
    scene = random_scene(E, 300 + seed, n_large)
    b = scene["bodies"]
    excl = list(zip(*[x.tolist() for x in scene["exclusions"]]))

    def brute(s, bb, before, got):
        want = EDGES.brute_force_broadphase(bb, b["kind"], b["shape_kind"], group=b["group"], mask=b["mask"], exclusions=excl,
                                            manifolds=before)
        assert Counter(map(tuple, got)) == want, f"step {s}: the pairs are not the brute force's"

    found = lockstep(E, scene, launch, 12 if EMU else 24, check=brute)
    assert sum(found[1:]) > 0, found


# ----------------------------------------------------------------------------- clamped keys

@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["faces", "edges", "corners", "boundary"])
def test_clamped_placements(gpu, E, kind):
    """Clusters past the faces, edges and corners of the measured key box and on its first and last fields (the scenes
    of test_gpu_broadphase_edges.py): one PH_BROAD measures the key fields, upload_state moves the clusters there, and
    the next steps, where up to 27 neighbour offsets share one key, must count and place the same pairs."""
    cell = EDGES._cell_pitch(2 * EDGES.R_SPHERE)
    S = EDGES.Scene(E)
    centres = EDGES.placements(kind, cell)
    park = EDGES.frame(S, EDGES.LO, EDGES.HI, cell, 8 * len(centres))
    for c in centres:
        EDGES.cluster(S, c, cell)
    for d, p in zip(S.defs[2:], park):
        d.position = p
    scene = dict(bodies=S.R.bodies_soa(S.defs), hinges=None, exclusions=None, settings=dict(velocity_iterations=4, position_iterations=2))
    nb = len(S.defs)
    worlds = [build_world(E, scene, "plain", env, max_manifolds=max(4096, 40 * nb)) for env in (HALF, WHOLE)]
    try:
        for w in worlds:
            w.run_phases(E.world.PH_BROAD)
            st = w.download_state()
            pos = st["pos"].copy()
            for i, t in enumerate(S.target):
                if t is not None:
                    pos[i] = t
            w.upload_state(pos, st["orn"], st["linvel"], st["angvel"])
        found = 0
        for s in range(3):
            for w in worlds:
                w.step(1)
            _, nh = same_step(s, *worlds)
            found += int(nh.sum())
        assert found >= 28 * len(centres)
        assert all(w.stats()["error_flags"] == 0 for w in worlds)
    finally:
        for w in worlds:
            w.close()


def test_under_emulation():
    """This file's gpu tests against the CPU emulation of tests/emu (plain launches only)."""
    from tests.emu import build as B
    env = dict(os.environ, B2D_EMU="1", B2D_LIB=B.build(), B2D_GRAPH="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout, r.stdout[-1000:]
