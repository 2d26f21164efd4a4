"""The device's contact-point merge (np_merge / np_rearrange in edyn_b200/csrc/b2d_kernels.cuh) on manifolds with persisted
points, one PH_NARROW each: against the reference's own process_collision (tests/golden/merge.npz) and against the oracle
on fresh cases from the same generator (tests/golden/make_merge.py), bit for bit: point counts, all 18 columns (impulses,
material and local normal included), attachments and lifetimes.  The step keeps a lifetime modulo 2^30 (include/b2d.h),
so lifetimes are compared modulo 2^30; everything else exactly.  Also: a sleeping manifold is left untouched, and
b2d_upload_contacts rejects what the point layout cannot hold."""

import numpy as np
import pytest

from tests.golden import make_merge as M
from tests.test_oracle_merge import GOLD, assert_coverage, coverage, golden_world

pytestmark = pytest.mark.gpu
f32 = np.float32
LIFE = (1 << 30) - 1


def run_device(E, b, man, seed=0):
    """Upload the manifolds in a shuffled order (the counting sort by pair type then spreads each type over several
    256-slot windows, and the three narrowphase kernels run in the same launch), run PH_NARROW once, and return the
    result in the original order."""
    pairs, num, pts, att, life = man
    m = len(pairs)
    perm = np.random.default_rng(seed).permutation(m)
    w = E.World(len(b["kind"]), max_manifolds=m)
    w.add_bodies(b)
    w.upload_contacts(pairs[perm], num[perm], pts[perm], att[perm], life[perm])
    w.run_phases(E.world.PH_NARROW)
    c = w.contacts()
    assert w.stats()["error_flags"] == 0
    at = {tuple(p): k for k, p in enumerate(c["pairs"].tolist())}
    idx = np.array([at[tuple(p)] for p in pairs.tolist()])
    return {k: c[k][idx] for k in ("num", "pts", "att", "lifetime")}


def differing(got, want):
    bad = []
    for i in range(len(want["num"])):
        k = int(want["num"][i])
        if (int(got["num"][i]) != k or not np.array_equal(got["pts"][i, :k].view(np.uint32), want["pts"][i, :k].view(np.uint32))
                or not np.array_equal(got["att"][i, :k], want["att"][i, :k])
                or not np.array_equal(got["lifetime"][i, :k], want["lifetime"][i, :k] & np.uint32(LIFE))):
            bad.append(i)
    return bad


def test_device_merge_matches_reference_vectors(gpu, E, O):
    g = np.load(GOLD)
    b, man = golden_world(g)
    got = run_device(E, b, man)
    want = dict(num=g["out_num"], pts=g["out_pts"], att=g["out_att"], lifetime=g["out_lifetime"])
    bad = differing(got, want)
    assert not bad, f"{len(bad)} of {len(g['num'])} cases differ from the reference, first {bad[:8]}"
    # the branches those cases reach (the oracle's trace of the same inputs, equal to the reference above)
    o = O.OracleWorld(dt=float(M.DT))
    o.add_bodies(b)
    o.set_contacts(*man)
    o.set_merge_trace(True)
    o.run_phases(O.PH_NARROW)
    assert_coverage(coverage(O, o.merge_trace()))


@pytest.mark.parametrize("seed", [11, 12])
def test_device_merge_matches_oracle_on_fresh_cases(gpu, E, O, seed):
    rng = np.random.default_rng(seed)
    fns = O.ora_fns()
    cs = [c for c in (M.candidate(rng, fns) for _ in range(1200)) if c is not None]
    want, _ = M.run_oracle(O, cs)
    got = run_device(E, M.bodies(cs), M.manifolds(cs), seed)
    bad = differing(got, want)
    assert not bad, f"{len(bad)} of {len(cs)} fresh cases differ from the oracle, first {bad[:8]}"


def test_sleeping_manifold_is_left_untouched(gpu, E):
    """narrowphase.cpp:31 leaves manifolds whose bodies both sleep out of the view: their points, lifetimes and impulses
    stay as they are.  The ABI cannot put a body to sleep, so a box settles on a plane in a sleeping world first."""
    from edyn_b200.rigidbody import STATIC, RigidBodyDef, bodies_soa, box_shape, plane_shape
    soa = bodies_soa([RigidBodyDef(kind=STATIC, shape=plane_shape((0, 1, 0), 0.0)),
                      RigidBodyDef(position=(0, 0.499, 0), mass=1.0, shape=box_shape((0.5, 0.5, 0.5)))], (0.0, -9.8, 0.0))
    w = E.World(2, max_manifolds=8, flags=E.world.FLAG_SLEEPING)
    w.add_bodies(soa)
    for _ in range(600):
        w.step(1)
        if w.sleeping()[1]:
            break
    assert w.sleeping()[1], "the box did not fall asleep"
    c = w.contacts()
    assert len(c["num"]) == 1 and c["num"][0] > 0
    pts = c["pts"].copy()
    pts[0, :, 15:18] += f32(0.25)                                 # values no step would write
    life = np.full_like(c["lifetime"], LIFE)
    w.upload_contacts(c["pairs"], c["num"], pts, c["att"], life)
    w.run_phases(E.world.PH_NARROW)
    assert w.sleeping()[1]
    d = w.contacts()
    k = int(c["num"][0])
    assert int(d["num"][0]) == k
    assert np.array_equal(d["pts"][0, :k].view(np.uint32), pts[0, :k].view(np.uint32))
    assert np.array_equal(d["att"][0, :k], c["att"][0, :k]) and (d["lifetime"][0, :k] == LIFE).all()


def test_upload_rejects_what_a_point_cannot_hold(gpu, E):
    """A point stores attachment | lifetime << 2 in one word: lifetimes from 2^30 and attachments above 2 are refused
    rather than cut; 2^30 - 1 and attachment 2 round-trip."""
    from edyn_b200.rigidbody import RigidBodyDef, bodies_soa, sphere_shape
    soa = bodies_soa([RigidBodyDef(position=(0, 0, 0), mass=1.0, shape=sphere_shape(0.5)),
                      RigidBodyDef(position=(0, 0.99, 0), mass=1.0, shape=sphere_shape(0.5))], (0.0, 0.0, 0.0))
    w = E.World(2, max_manifolds=4)
    w.add_bodies(soa)
    pairs, num = np.array([[1, 0]], np.uint32), np.array([2], np.uint32)
    pts = np.random.default_rng(3).uniform(-1, 1, (1, 4, 18)).astype(f32)
    att = np.array([[2, 1, 0, 0]], np.uint32)
    w.upload_contacts(pairs, num, pts, att, np.array([[LIFE, LIFE - 1, 0, 0]], np.uint32))
    c = w.contacts()
    assert int(c["num"][0]) == 2 and list(c["lifetime"][0, :2]) == [LIFE, LIFE - 1] and list(c["att"][0, :2]) == [2, 1]
    assert np.array_equal(c["pts"][0, :2].view(np.uint32), pts[0, :2].view(np.uint32))
    for bad_att, bad_life in (([3, 0, 0, 0], [0, 0, 0, 0]), ([0, 0, 0, 0], [0, 1 << 30, 0, 0]), ([0, 0, 0, 0], [0xFFFFFFFF, 0, 0, 0])):
        with pytest.raises(E.world.B2DError):
            w.upload_contacts(pairs, num, pts, np.array([bad_att], np.uint32), np.array([bad_life], np.uint32))
    # slots past num are not points: whatever they hold is not checked
    w.upload_contacts(pairs, np.array([1], np.uint32), pts, np.array([[0, 7, 7, 7]], np.uint32), np.array([[5, 1 << 31, 0, 0]], np.uint32))
    assert list(w.contacts()["lifetime"][0, :1]) == [5]
