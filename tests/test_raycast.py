"""Raycast (include/b2d.h b2d_raycast) without a GPU: the CPU restatement's shape_raycast (tests/raycast/ora_raycast.cpp)
against the reference's own (tests/raycast/ref_raycast.cpp, where the reference's objects were built), the reference's
test_raycast.cpp answers, the restatement's brute-force world query against edyn::raycast, and the device kernels under
the CPU emulation against that brute force, bit for bit."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests import raycast_support as S  # noqa: E402
SPHERE, CAPSULE, BOX, PLANE = 0, 2, 3, 6
MISS = 0xFFFFFFFF


@pytest.fixture(scope="module")
def refs():
    lib = S.ref()
    if lib is None:
        pytest.skip("the reference's object files (oracle/_ref/edyn_obj) are not available (needs /root/reference at build time)")
    return lib


class _Ora:
    @staticmethod
    def shape_raycast(kind, p, pos, orn, p0, p1):
        return S.shape_raycast(S.ora(), "ora_", kind, p, pos, orn, p0, p1)


def _ref_shape_raycast(lib, kind, p, pos, orn, p0, p1):
    return S.shape_raycast(lib, "rr_", kind, p, pos, orn, p0, p1)[1:]


def _cases(rng, n):
    """Random single-shape cases: sphere / box / capsule / plane with random orientations, segments through, past, from
    inside and short of the shape, axis-aligned ones (box faces, capsule axes) and grazing ones."""
    out = []
    for i in range(n):
        kind = [SPHERE, BOX, CAPSULE, PLANE][i % 4]
        p = np.zeros(4, np.float32)
        if kind == PLANE:
            nrm = rng.normal(size=3).astype(np.float32)
            if i % 8 == 3:
                nrm = np.eye(3, dtype=np.float32)[rng.integers(3)]
            p[:3] = nrm / np.linalg.norm(nrm); p[3] = rng.uniform(-1, 1)
        else:
            p[:3] = rng.uniform(0.1, 1.0, 3)
            if kind == CAPSULE:
                p[2] = rng.integers(0, 3)
        pos = rng.uniform(-2, 2, 3).astype(np.float32)
        q = rng.normal(size=4).astype(np.float32)
        orn = (q / np.linalg.norm(q)).astype(np.float32) if i % 3 else np.array([0, 0, 0, 1], np.float32)
        mode = rng.integers(6)
        p0 = (pos + rng.normal(size=3) * 3).astype(np.float32)
        if mode == 0:                                                # through the centre
            p1 = (pos + (pos - p0) * rng.uniform(0.2, 2.0)).astype(np.float32)
        elif mode == 1:                                              # from inside
            p0 = (pos + rng.normal(size=3) * 0.05).astype(np.float32)
            p1 = (p0 + rng.normal(size=3) * 3).astype(np.float32)
        elif mode == 2:                                              # axis-aligned
            p1 = p0.copy(); p1[rng.integers(3)] -= np.float32(rng.uniform(-6, 6))
        elif mode == 3:                                              # short of it
            p1 = (p0 + (pos - p0) * 0.3).astype(np.float32)
        else:
            p1 = (pos + rng.normal(size=3) * 3).astype(np.float32)
        if kind == BOX and np.array_equal(p0, p1):
            continue                                                 # the reference reads get_face_normal(SIZE_MAX)
        out.append((kind, p, pos, orn, p0, p1))
    return out


def test_shape_raycast_matches_reference(refs):
    """Fraction, feature and normal bits of the restatement == edyn::shape_raycast, except the capsule hemisphere normal,
    which the restatement takes at the hit point from the hemisphere centre (checked against that formula)."""
    ora = _Ora
    rng = np.random.default_rng(7)
    n_hits = 0
    for kind, p, pos, orn, p0, p1 in _cases(rng, 6000):
        hit, f, nrm, feat = ora.shape_raycast(kind, p, pos, orn, p0, p1)
        rf, rn, rfeat = _ref_shape_raycast(refs, kind, p, pos, orn, p0, p1)
        ctx = (kind, p, pos, orn, p0, p1)
        assert np.float32(f).view(np.uint32) == np.float32(rf).view(np.uint32), ctx
        assert feat == rfeat, ctx
        if not hit:
            continue
        n_hits += 1
        if kind == CAPSULE and feat in (0, 1):
            # hemisphere centre = capsule vertex: pos + dir * half_length (0) or pos - dir * half_length (1)
            x, y, z, w = orn.astype(np.float64)
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
            c = pos + R[:, int(p[2])] * p[1] * (1 if feat == 0 else -1)
            hp = p0.astype(np.float64) * (1 - f) + p1.astype(np.float64) * f
            want = (hp - c) / np.linalg.norm(hp - c)
            assert np.allclose(nrm, want, atol=1e-4), ctx
            continue
        assert np.array_equal(nrm.view(np.uint32), rn.view(np.uint32)), ctx
    assert n_hits > 2000


def test_capsule_hemisphere_normal_is_taken_at_the_hit_point():
    """A segment along a capsule's axis hits the hemisphere at its pole; the normal is the axis direction.  (The reference
    leaves u_in unwritten on this path and computes its normal from it.)"""
    ora = _Ora
    p = np.array([0.5, 1.0, 1, 0], np.float32)                        # radius 0.5, half length 1, axis y
    hit, f, n, feat = ora.shape_raycast(CAPSULE, p, [0, 0, 0], [0, 0, 0, 1], [0, 4, 0], [0, 0, 0])
    assert hit and feat == 0 and f == np.float32(0.625)
    assert np.array_equal(n, np.array([0, 1, 0], np.float32))
    hit, f, n, feat = ora.shape_raycast(CAPSULE, p, [0, 0, 0], [0, 0, 0, 1], [3, 1.5, 0], [-3, 1.5, 0])
    assert hit and feat == 0
    c = np.array([0, 1, 0], np.float32)
    x = np.array([3, 1.5, 0], np.float32) * (np.float32(1) - f) + np.array([-3, 1.5, 0], np.float32) * f
    assert abs(np.linalg.norm(x - c) - 0.5) < 1e-5
    assert np.allclose(n, (x - c) / np.linalg.norm(x - c), atol=1e-6)


def _box_world():
    o = S.BruteWorld()
    b = dict(pos=[[0.5, 0.5, 0.5]], orn=[[0, 0, 0, 1]], linvel=[[0, 0, 0]], angvel=[[0, 0, 0]], inv_mass=[0],
             inv_inertia=[np.zeros(9)], gravity=[[0, 0, 0]], kind=[2], shape_kind=[BOX], shape_params=[[0.5, 0.5, 0.5, 0]],
             friction=[0.5], restitution=[0])
    o.add_bodies(b)
    return o, b


def test_known_answers_of_the_reference_test():
    """test/edyn/collision/test_raycast.cpp: a unit box at (0.5, 0.5, 0.5); (2,2,2) -> (0,0,0) hits it at 0.5, and the
    vertical ray (0.5,2,0.5) -> (0.5,0,0.5) at 0.5 through face 2."""
    o, _ = _box_world()
    r = o.raycast([[2, 2, 2], [0.5, 2, 0.5]], [[0, 0, 0], [0.5, 0, 0.5]])
    assert r["body"].tolist() == [0, 0]
    assert r["fraction"].tolist() == [0.5, 0.5]
    assert int(r["feature"][1]) == 2
    assert r["normal"][1].tolist() == [0, 1, 0]


def test_known_answers_through_the_reference(refs):
    _, b = _box_world()
    w = S.RefWorld(b["pos"], b["orn"], b["shape_kind"], b["shape_params"])
    for p0, p1, face in (([2, 2, 2], [0, 0, 0], None), ([0.5, 2, 0.5], [0.5, 0, 0.5], 2)):
        body, f, _, feat = w.raycast(p0, p1)
        assert body == 0 and f == np.float32(0.5)
        if face is not None:
            assert feat == face
    w.close()


def test_world_raycast_matches_reference(refs):
    """The brute force == edyn::raycast on random static scenes, for segments whose reference answer lies in
    [0, 1].  The reference can answer with a fraction outside [0, 1] (quirk 1 of DESIGN.md section 6); those segments
    are counted, not compared."""
    sys.path.insert(0, ROOT)
    from tests.emu import raycast as R
    rng = np.random.default_rng(11)
    compared = outside = 0
    for seed in range(3):
        soa = R.scene(np.random.default_rng(seed), 150)
        w = S.RefWorld(soa["pos"], soa["orn"], soa["shape_kind"], soa["shape_params"])      # static bodies
        o = S.BruteWorld()
        o.add_bodies(soa)
        p0, p1 = R.segments(rng, np.asarray(soa["pos"], np.float32), 400)
        ok = np.isfinite(p0).all(1) & np.isfinite(p1).all(1) & ~(p0 == p1).all(1)
        p0, p1 = p0[ok], p1[ok]
        mine = o.raycast(p0, p1)
        for i in range(len(p0)):
            body, f, _, feat = w.raycast(p0[i], p1[i])
            if body != MISS and not (0 <= f <= 1):
                outside += 1
                continue
            compared += 1
            assert mine["body"][i] == body, (i, p0[i], p1[i], mine["body"][i], body)
            if body != MISS:
                assert mine["fraction"][i].view(np.uint32) == np.float32(f).view(np.uint32)
                assert mine["feature"][i] == feat
        w.close()
    assert compared > 400
    print(f"compared {compared}, reference answer outside [0, 1]: {outside}")


def test_emulated_raycast_kernels_match_brute_force():
    """k_ray_* under the CPU emulation == the brute force, bit for bit, on random worlds: tilted static boxes,
    a plane, large bodies, bodies far outside the measured cell range, removed bodies, both ignore forms, zero-length and
    non-finite segments, segments cast right after add_bodies."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emu", "raycast.py"), "1", "2", "3"], capture_output=True,
                       text=True, cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])["results"]
    assert len(res) == 3 * 16
    for x in res:
        assert x["mismatches"] == 0, x
    assert sum(x["hits"] for x in res) > 3000


GOLDEN = os.path.join(ROOT, "tests", "golden", "raycast.npz")


def golden_world_soa(g, sel):
    """The selected golden cases as static bodies of one world (each case sits in a 100 m cell of its own)."""
    m = int(sel.sum())
    return dict(pos=g["pos"][sel], orn=g["orn"][sel], linvel=np.zeros((m, 3), np.float32), angvel=np.zeros((m, 3), np.float32),
                inv_mass=np.zeros(m, np.float32), inv_inertia=np.zeros((m, 9), np.float32), gravity=np.zeros((m, 3), np.float32),
                kind=np.full(m, 2, np.uint32), shape_kind=g["kind"][sel], shape_params=g["params"][sel],
                friction=np.full(m, 0.5, np.float32), restitution=np.zeros(m, np.float32))


def golden_expected(g, sel):
    """The world answer of each selected case under the filter rule, from the reference's raw result: its own body if the
    fraction lies in [0, 1], a miss otherwise."""
    f = g["fraction"][sel]
    ok = (f >= 0) & (f <= 1)
    m = int(sel.sum())
    return dict(body=np.where(ok, np.arange(m), MISS).astype(np.uint32), fraction=np.where(ok, f, np.finfo(np.float32).max).astype(np.float32),
                normal=np.where(ok[:, None], g["normal"][sel], 0).astype(np.float32),
                feature=np.where(ok, g["feature"][sel], MISS).astype(np.uint32))


def test_golden_shape_raycast():
    """The restatement == the reference's recorded shape_raycast bits on tests/golden/raycast.npz (capsule hemisphere
    normals: the corrected formula, checked in test_shape_raycast_matches_reference)."""
    g = np.load(GOLDEN)
    ora = _Ora
    n = len(g["kind"])
    assert n >= 2000
    for i in range(n):
        hit, f, nrm, feat = ora.shape_raycast(int(g["kind"][i]), g["params"][i], g["pos"][i], g["orn"][i], g["p0"][i], g["p1"][i])
        assert np.float32(f).view(np.uint32) == g["fraction"][i].view(np.uint32), i
        assert feat == g["feature"][i], i
        if hit and not (g["kind"][i] == CAPSULE and feat in (0, 1)):
            assert np.array_equal(nrm.view(np.uint32), g["normal"][i].view(np.uint32)), i


def test_golden_filter_rule():
    """One brute-force world holding every non-plane golden case, one batch of their segments: each answer is the reference's
    raw result passed through the filter rule (hit iff 0 <= f <= 1).  Capsule hemisphere normals are left out."""
    sys.path.insert(0, ROOT)
    from tests.emu import raycast as R
    g = np.load(GOLDEN)
    sel = g["kind"] != PLANE
    o = S.BruteWorld()
    o.add_bodies(golden_world_soa(g, sel))
    got = o.raycast(g["p0"][sel], g["p1"][sel])
    want = golden_expected(g, sel)
    hemi = (g["kind"][sel] == CAPSULE) & (want["feature"] <= 1)
    got["normal"][hemi] = want["normal"][hemi]
    total, bad, first = R.compare(got, want)
    assert bad == 0, first
    assert int((want["body"] != MISS).sum()) > 300
    assert int(((g["fraction"][sel] < 0) | ((g["fraction"][sel] > 1) & (g["fraction"][sel] < 1e30))).sum()) > 50   # filtered
