"""process_collision (include/edyn/util/collision_util.hpp:105-276) as a whole: the oracle's narrowphase on manifolds seeded
with 0-4 persisted points == the reference's own narrowphase::update (tests/golden/merge.npz, tests/golden/make_merge.py),
bit for bit: point counts, all 18 columns in slot order, attachments and lifetimes.  The oracle's merge trace says which
branches the committed cases reach; every branch of the catalogue (oracle/ora_world.hpp, merge_branch) has at least
MIN_CASES cases but those make_merge.py argues no input reaches or its sampling does not produce."""
import os

import numpy as np
import pytest

from tests.golden import make_merge as M

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "merge.npz")
MIN_CASES = 20


def golden_world(g):
    """Body SoA and manifolds of merge.npz, in the layout of World.add_bodies / upload_contacts."""
    n = len(g["kind"])
    b = dict(pos=g["pos"], orn=g["orn"], linvel=np.zeros((n, 3), np.float32), angvel=g["angvel"],
             inv_mass=np.where(g["kind"] == 0, 1.0, 0.0).astype(np.float32), inv_inertia=np.tile(np.eye(3, dtype=np.float32).reshape(9), (n, 1)),
             gravity=np.zeros((n, 3), np.float32), kind=g["kind"], shape_kind=g["shape_kind"], shape_params=g["shape_params"],
             friction=g["friction"], restitution=g["restitution"], group=None, mask=None)
    m = len(g["num"])
    pairs = np.stack([2 * np.arange(m), 2 * np.arange(m) + 1], axis=1).astype(np.uint32)
    return b, (pairs, g["num"], g["pts"], g["att"], g["lifetime"])


def coverage(O, trace):
    """Number of cases behind each branch name."""
    t = np.asarray(trace, np.uint64)
    return {name: int(((t >> np.uint64(k)) & np.uint64(1)).sum()) for k, name in enumerate(O.MERGE_BRANCHES)}


def assert_coverage(cov):
    short = {k: v for k, v in cov.items() if v < MIN_CASES and k not in M.UNREACHABLE + M.NOT_SAMPLED}
    assert not short, f"branches with fewer than {MIN_CASES} cases: {short}"
    assert all(cov[k] == 0 for k in M.UNREACHABLE), {k: cov[k] for k in M.UNREACHABLE}


def differing(got, want, n):
    """Cases whose count, 18 columns, attachments or lifetimes differ (slots past the count are not compared)."""
    bad = []
    for i in range(n):
        k = int(want["num"][i])
        if (int(got["num"][i]) != k or not np.array_equal(got["pts"][i, :k].view(np.uint32), want["pts"][i, :k].view(np.uint32))
                or not np.array_equal(got["att"][i, :k], want["att"][i, :k]) or not np.array_equal(got["lifetime"][i, :k], want["lifetime"][i, :k])):
            bad.append(i)
    return bad


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLD)


def test_oracle_merge_matches_reference_vectors(O, golden):
    g = golden
    b, man = golden_world(g)
    o = O.OracleWorld(dt=float(M.DT))
    o.add_bodies(b)
    o.set_contacts(*man)
    o.set_merge_trace(True)
    o.run_phases(O.PH_NARROW)
    got = o.contacts()
    want = dict(num=g["out_num"], pts=g["out_pts"], att=g["out_att"], lifetime=g["out_lifetime"])
    bad = differing(got, want, len(g["num"]))
    assert not bad, f"{len(bad)} of {len(g['num'])} cases differ from the reference, first {bad[:8]}"
    assert_coverage(coverage(O, o.merge_trace()))


def test_merge_vectors_hold_the_edge_values(golden):
    """The persisted lists carry the values that tell a kept point from a new one and the lifetime edge."""
    g = golden
    live = np.arange(4)[None, :] < g["num"][:, None]
    life = g["lifetime"][live]
    assert ((1 << 30) - 1) in life and ((1 << 30) - 2) in life
    assert (g["pts"][live][:, 15] != 0).all()
    fam = {tuple(x) for x in g["shape_kind"].reshape(-1, 2).tolist()}          # both body orders of every shape family
    assert all((a, b) in fam and (b, a) in fam for a, b in M.FAMILIES)


def test_oracle_merge_matches_reference_on_fresh_cases(O):
    """New cases from the same generator, the oracle against the reference's own narrowphase directly."""
    if O.ref_stepper() is None:
        pytest.skip("oracle/_ref/libedyn_stepper.so not available (needs /root/reference at build time)")
    rng = np.random.default_rng(7)
    fns = O.ora_fns()
    cs = [c for c in (M.candidate(rng, fns) for _ in range(1500)) if c is not None]
    got, _ = M.run_oracle(O, cs)
    ref = M.run_reference(O, cs)
    bad = differing(got, ref, len(cs))
    assert not bad, f"{len(bad)} of {len(cs)} fresh cases differ from the reference, first {bad[:8]}"
