"""The broadphase pair search where the cell key clamps, against a brute-force reference of the same operation.

`cell_key_of` packs a body's cell coordinates into key fields sized when the body population last changed (`measure_cells`:
the occupied extent plus max(16, span / 2) cells of room on each side, at most 16 bits per axis; x stops at 2^bits - 2).
A cell outside that box shares the boundary key, so up to three neighbour offsets per axis (27 at a corner) name the same
cell.  The search must walk such a cell once per query body: a pair found there twice would get two manifolds, and the
contact would be solved twice per iteration for as long as it lasts.

`brute_force_broadphase` restates what the device's broadphase computes, O(n^2) in float32 and with no grid: the
manifolds that survive `k_bp_separate`, plus one new manifold per pair `bp_candidate` accepts.  It is anchored on the CPU
against the pair lists of the reference's own dynamic trees (tests/golden/broadphase.npz) and against the oracle.  The
`gpu` tests then drive the device's broadphase alone: bodies are added spread out inside the box, one PH_BROAD measures the
key fields, and upload_state (which does not measure again) moves groups of touching bodies past the faces, edges and
corners of the key box, across its boundaries, past the 16-bit cap, next to large bodies, filters, exclusions and sleeping
bodies.  Every case runs with both search mappings (a thread per query body, and a warp per query body with one lane per
cell) and compares the manifold pairs as a multiset.  Also runs against the CPU emulation (B2D_EMU=1)."""
import os
from collections import Counter

import numpy as np
import pytest

from tests.parity import build_world

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EMU = os.environ.get("B2D_EMU") == "1"
SEARCH = {"thread": {"B2D_BP_WARP_MAX": "0"}, "warp": {"B2D_BP_WARP_MAX": str(1 << 30)}}
F32 = np.float32
BP_OFFSET = -F32(0.02)                      # m_aabb_offset
BP_SEPARATION = -(F32(0.02) * F32(1.3))     # -m_separation_threshold, rounded in float32 as the device does
SHAPE_NONE = 255
ALL = np.uint64(0xFFFFFFFFFFFFFFFF)


# ----------------------------------------------------------------------------- the brute-force reference

def _inset(bb, v):
    return np.concatenate([bb[..., :3] + v, bb[..., 3:] - v], axis=-1)


def _hits(a, b):
    """Closed-interval AABB intersection, broadcast over leading axes (geom.cpp intersect)."""
    return np.all((a[..., :3] <= b[..., 3:]) & (a[..., 3:] >= b[..., :3]), axis=-1)


def _should_collide(a, b, group, mask, has_filter, exclusions):
    """should_collide_default (collision/should_collide.cpp) and the exclusion list."""
    if has_filter[a] and has_filter[b]:
        if (group[a] & mask[b]) == 0 or (group[b] & mask[a]) == 0:
            return False
    elif has_filter[a] or has_filter[b]:
        f = a if has_filter[a] else b
        if group[f] == 0 or mask[f] == 0:
            return False
    return (min(a, b), max(a, b)) not in exclusions


def brute_force_broadphase(aabb, kind, shape, asleep=None, removed=None, group=None, mask=None, exclusions=(), manifolds=()):
    """The ordered manifold pairs after one broadphase, as a Counter (a multiset), with no grid.

    aabb (n, 6) float32 min | max: what the broadphase reads (the AABBs refreshed at the end of the previous step); kind
    0 dynamic, 1 kinematic, 2 static; shape 255 for none; asleep / removed per body; group / mask the collision filter
    (a body has one unless both are all ones); exclusions unordered (lo, hi) pairs; manifolds the ordered pairs alive before the broadphase.
    A manifold survives unless a body was removed or, with either body awake, inset(bb0, -0.02 * 1.3) misses bb1.  Only
    an awake dynamic body with a shape queries, with inset(bb, -0.02); of two awake dynamic bodies only the higher id
    tests the pair, and where its query misses but the other body's query hits, the other body becomes body[0].  A pair
    that already has a manifold is not searched again."""
    aabb = np.asarray(aabb, F32)
    n = len(aabb)
    kind, shape = np.asarray(kind), np.asarray(shape)
    asleep = np.zeros(n, bool) if asleep is None else np.asarray(asleep, bool)
    removed = np.zeros(n, bool) if removed is None else np.asarray(removed, bool)
    group = np.full(n, ALL) if group is None else np.asarray(group, np.uint64)
    mask = np.full(n, ALL) if mask is None else np.asarray(mask, np.uint64)
    has_filter = (group != ALL) | (mask != ALL)
    exclusions = {(min(a, b), max(a, b)) for a, b in exclusions}
    shaped = (shape != SHAPE_NONE) & ~removed
    dynamic = (kind == 0) & ~asleep & ~removed
    out, alive = Counter(), set()
    for a, b in manifolds:
        a, b = int(a), int(b)
        if removed[a] or removed[b]:
            continue
        if (dynamic[a] or dynamic[b]) and not _hits(_inset(aabb[a], BP_SEPARATION), aabb[b]):
            continue
        out[(a, b)] += 1
        alive.add((min(a, b), max(a, b)))
    query = _inset(aabb, BP_OFFSET)
    for A in np.nonzero(dynamic & shaped)[0].tolist():
        ids = np.arange(n)
        cand = shaped & (ids != A) & ~(dynamic & (ids > A))
        fwd = _hits(query[A], aabb)                         # A's query hits j
        back = _hits(query, aabb[A]) & dynamic              # j's query hits A (tested only between two dynamic bodies)
        for j in np.nonzero(cand & (fwd | back))[0].tolist():
            if not _should_collide(A, j, group, mask, has_filter, exclusions) or (min(A, j), max(A, j)) in alive:
                continue
            out[(A, j) if fwd[j] else (j, A)] += 1
    return out


# ----------------------------------------------------------------------------- anchors (CPU)

def test_brute_force_reproduces_reference_tree_pairs(E):
    """The 12 crowded scenes of tests/golden/broadphase.npz, whose ordered pair lists come from the reference's dynamic
    AABB trees: the brute force gives the same ordered pairs, each once."""
    g = np.load(os.path.join(GOLD, "broadphase.npz"))
    off = po = 0
    total = 0
    for n, c in zip(g["sizes"].tolist(), g["counts"].tolist()):
        want = Counter(map(tuple, g["pairs"][po:po + c].tolist()))
        got = brute_force_broadphase(g["aabb1"][off:off + n], g["soa_kind"][off:off + n], g["soa_shape_kind"][off:off + n],
                                     group=g["soa_group"][off:off + n], mask=g["soa_mask"][off:off + n])
        assert got == want, f"scene at body {off}: {len(got - want)} extra, {len(want - got)} missing"
        total += c
        off += n; po += c
    assert total > 5000


@pytest.mark.parametrize("seed", range(4))
def test_brute_force_agrees_with_oracle(E, O, seed):
    """Random scenes with collision filters and exclusions (tests/test_ref_stepper.py random_scene), stepped a few times
    by the oracle: after every broadphase its ordered manifold pairs are what the brute force makes of the AABBs and the
    manifolds it started from."""
    from tests.test_ref_stepper import random_scene
    scene = random_scene(E, O, seed)
    b = scene["bodies"]
    o = O.OracleWorld(vel_iters=scene["settings"]["velocity_iterations"], pos_iters=scene["settings"]["position_iterations"])
    o.add_bodies(b)
    excl = ()
    if scene["exclusions"] is not None:
        o.add_exclusions(*scene["exclusions"])
        excl = list(zip(*[np.asarray(x).tolist() for x in scene["exclusions"]]))
    before = []
    checked = 0
    for _ in range(12):
        bb = o.state()["aabb"]
        o.run_phases(O.PH_BROAD)
        want = brute_force_broadphase(bb, b["kind"], b["shape_kind"], group=b["group"], mask=b["mask"], exclusions=excl, manifolds=before)
        got = Counter(map(tuple, o.pairs().tolist()))
        assert got == want
        checked += len(got)
        o.run_phases(O.PH_NARROW | O.PH_ISLANDS | O.PH_SOLVE)
        before = o.pairs().tolist()
    assert checked > 0


def test_brute_force_agrees_with_oracle_at_the_margin(E, O):
    """Sphere pairs whose AABBs lie 0.02 apart to within a few float32 ulps, including pairs where only the lower id's
    query reaches the other AABB (then the lower id is body[0]): the oracle and the brute force agree pair by pair, so
    the float32 inset and the orientation rule are pinned, not only the pair set."""
    R = E.rigidbody
    rng = np.random.default_rng(77)
    defs = []
    for g in range(64):
        r1, r2 = F32(rng.uniform(0.1, 0.25)), F32(rng.uniform(0.1, 0.25))
        asym = g % 2 == 0
        x = (2.0 ** int(rng.integers(0, 4)) - rng.uniform(0.0005, 0.019) - float(r1)) if asym else rng.uniform(-40, 40)
        pl, pr = _gap_pair(F32(x), r1, r2, asym, int(rng.integers(-3, 4)))
        y, z = 3.0 * (g % 8), 3.0 * (g // 8)
        defs += [R.RigidBodyDef(position=(float(pl), y, z), shape=R.sphere_shape(float(r1))),
                 R.RigidBodyDef(position=(float(pr), y, z), shape=R.sphere_shape(float(r2)))]
    b = R.bodies_soa(defs)
    o = O.OracleWorld()
    o.add_bodies(b)
    bb = o.state()["aabb"]
    o.run_phases(O.PH_BROAD)
    got = Counter(map(tuple, o.pairs().tolist()))
    assert got == brute_force_broadphase(bb, b["kind"], b["shape_kind"])
    assert sum(1 for p0, p1 in got if p0 < p1) > 0 and 10 < len(got) < 64


# ----------------------------------------------------------------------------- the device at the edges of the key box

R_SPHERE = 0.25
GAP = 0.49                                  # sphere spacing in a cluster: AABBs overlap by 0.01


def _cell_pitch(max_diameter):
    """d.cell: the largest grid body's bounding diameter + 2 x 0.02 + 1e-3, in float32 (reclassify)."""
    return float(F32(F32(max_diameter) + F32(2) * F32(0.02)) + F32(1e-3))


def key_box(aabb, cell, grid):
    """measure_cells restated: per axis, the first cell coordinate of the key field and its last (x: 2^bits - 2)."""
    inv = F32(1) / F32(cell)
    c = np.floor((aabb[grid, :3] + aabb[grid, 3:]) * F32(0.5) * inv).astype(np.int64)
    lo, hi = [], []
    for k in range(3):
        span = int(c[:, k].max() - c[:, k].min() + 1)
        room = max(16, span // 2)
        bits = 1
        while (1 << bits) < span + 2 * room + 2 and bits < 16:
            bits += 1
        org = max(int(c[:, k].min()) - room, -(1 << 30))
        lo.append(org)
        hi.append(org + (1 << bits) - (2 if k == 0 else 1))
    return np.array(lo), np.array(hi)


class Scene:
    """Bodies for one broadphase case: `defs` as RigidBodyDef, the exclusions, and the position each body is moved to
    after the key fields are measured (None: stays)."""

    def __init__(self, E):
        self.R = E.rigidbody
        self.defs, self.target, self.excl = [], [], []

    def add(self, d, target=None):
        self.defs.append(d); self.target.append(target)
        return len(self.defs) - 1

    def sphere(self, target, r=R_SPHERE):
        """A dynamic sphere without gravity, parked inside the box until the fields are measured, then moved to `target`."""
        return self.add(self.R.RigidBodyDef(position=(0, 0, 0), gravity=(0, 0, 0), shape=self.R.sphere_shape(r)), target)


def cluster(S, center, cell, shape=(2, 2, 2)):
    """Touching spheres on a GAP lattice around `center` (in cells); every AABB pair of the lattice intersects."""
    c = (np.asarray(center, np.float64) + 0.5) * cell
    ids = []
    for i in np.ndindex(*shape):
        ids.append(S.sphere(tuple((c + (np.array(i) - (np.array(shape) - 1) / 2) * GAP).tolist())))
    return ids


def frame(S, lo_cell, hi_cell, cell, n_park):
    """Two static spheres at opposite corners fix the measured extent; the dynamic bodies are parked 1.2 m apart inside it
    (no pair among them) until they move."""
    R = S.R
    for c in (lo_cell, hi_cell):
        S.add(R.RigidBodyDef(kind=R.STATIC, position=tuple(((np.asarray(c, np.float64) + 0.5) * cell).tolist()), shape=R.sphere_shape(R_SPHERE)))
    side = int(np.ceil(n_park ** (1 / 3)))
    assert side * 1.2 < (np.min(np.asarray(hi_cell) - np.asarray(lo_cell)) - 1) * cell, "frame too small for the parked bodies"
    base = (np.asarray(lo_cell, np.float64) + 1.5) * cell
    return [tuple((base + 1.2 * np.array(np.unravel_index(k, (side,) * 3))).tolist()) for k in range(n_park)]


def run_case(E, S, env, flags=0, after_measure=None):
    """add_bodies, one PH_BROAD (measures the key fields), upload_state to the targets, one more PH_BROAD: the device's
    manifold pairs against the brute force, and the key box the fields were measured to.  Returns (got, want, box, state):
    got counts the device's error flags under the key "error_flags"."""
    nb = len(S.defs)
    b = S.R.bodies_soa(S.defs)
    scene = dict(bodies=b, hinges=None, exclusions=None, settings=dict(velocity_iterations=4, position_iterations=2))
    w = build_world(E, scene, env=env, flags=flags, max_manifolds=max(4096, 40 * nb))
    try:
        if S.excl:
            w.add_exclusions([a for a, _ in S.excl], [c for _, c in S.excl])
        w.run_phases(E.world.PH_BROAD)
        first = w.pairs().tolist()
        st = w.download_state()
        grid = (b["shape_kind"] != SHAPE_NONE)
        diam = np.where(b["shape_kind"] == 0, 2 * b["shape_params"][:, 0], 0)
        cell = _cell_pitch(diam.max())
        large = np.zeros(nb, bool)
        dyn_d = diam[(b["kind"] == 0) & (diam > 0)]
        large |= (b["shape_kind"] != 0) | (diam > 4 * dyn_d.mean())        # planes and boxes here are the large bodies
        box = key_box(st["aabb"], cell, grid & ~large)
        if after_measure is not None:
            after_measure(w, box)
        pos = st["pos"].copy()
        for i, t in enumerate(S.target):
            if t is not None:
                pos[i] = t
        w.upload_state(pos, st["orn"], st["linvel"], st["angvel"])
        st = w.download_state()
        asleep = w.sleeping().astype(bool)
        w.run_phases(E.world.PH_BROAD)
        got = Counter(map(tuple, w.pairs().tolist()))
        got["error_flags"] = w.stats()["error_flags"]
        want = brute_force_broadphase(st["aabb"], b["kind"], b["shape_kind"], asleep=asleep, group=b["group"], mask=b["mask"],
                                      exclusions=S.excl, manifolds=first)
        return got, want, box, st
    finally:
        w.close()


def _check(got, want, min_pairs):
    got = Counter(got)
    flags = got.pop("error_flags", 0)
    extra, missing = got - want, want - got
    assert not extra and not missing, f"device has {sum(extra.values())} extra manifolds {dict(list(extra.items())[:6])}, " \
                                      f"misses {sum(missing.values())} {dict(list(missing.items())[:6])}"
    assert flags == 0 and sum(want.values()) >= min_pairs


LO, HI = np.array([0, 0, 0]), np.array([20, 20, 20])          # extent of the frame, in cells (key box: 64 cells per axis)


def _box_of_frame(cell):
    """The key box the frame's extent measures to (16 cells of room, 6 bits: x 0..62, y and z 0..63 from -16)."""
    return LO - 16, LO - 16 + np.array([62, 63, 63])


def placements(kind, cell):
    """Cluster centres (in cells) relative to the frame's key box for one family of placements."""
    lo, hi = _box_of_frame(cell)
    mid = (LO + HI) // 2
    out = []
    if kind == "faces":
        for k in range(3):
            for side, at in ((-1, lo[k] - 6), (1, hi[k] + 6)):
                c = mid.copy(); c[k] = at; out.append(c)
    elif kind == "edges":
        for k1, k2 in ((0, 1), (0, 2), (1, 2)):
            for s1 in (-1, 1):
                for s2 in (-1, 1):
                    c = mid.copy()
                    c[k1] = lo[k1] - 5 if s1 < 0 else hi[k1] + 5
                    c[k2] = lo[k2] - 5 if s2 < 0 else hi[k2] + 5
                    out.append(c)
    elif kind == "corners":
        for s in np.ndindex(2, 2, 2):
            out.append(np.where(np.array(s) == 0, lo - 4, hi + 4))
    elif kind == "boundary":
        # on the first and last field of every axis, and one cell outside: the offsets there clamp on one side only
        for k in range(3):
            for at in (lo[k], lo[k] - 1, hi[k], hi[k] + 1):
                c = mid.copy(); c[k] = at; out.append(c)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("search", list(SEARCH))
@pytest.mark.parametrize("kind", ["faces", "edges", "corners", "boundary", "straddle"])
def test_clamped_clusters(gpu, E, search, kind):
    """Clusters of touching spheres past each face, each edge and each corner of the measured key box (where 3, 9 or 27
    neighbour offsets share one key), on its first and last fields (x: 2^bits - 2) and one cell outside them, and rows
    that straddle each boundary, half in range and half out."""
    S = Scene(E)
    cell = _cell_pitch(2 * R_SPHERE)
    lo, hi = _box_of_frame(cell)
    if kind == "straddle":
        rows = []
        for k in range(3):
            for at in (lo[k], hi[k]):
                c = ((LO + HI) // 2).astype(np.float64); c[k] = at
                rows.append((c, k))
        n_park = 8 * len(rows)
    else:
        centres = placements(kind, cell)
        n_park = 8 * len(centres)
    park = frame(S, LO, HI, cell, n_park)
    if kind == "straddle":
        for c, k in rows:
            start = (c + 0.5) * cell
            for i in range(8):
                p = start.copy(); p[k] += (i - 3.5) * GAP
                S.sphere(tuple(p.tolist()))
    else:
        for c in centres:
            cluster(S, c, cell)
    for d, p in zip(S.defs[2:], park):
        d.position = p
    got, want, box, st = run_case(E, S, SEARCH[search])
    assert np.array_equal(box[0], lo) and np.array_equal(box[1], hi)
    moved = [i for i, t in enumerate(S.target) if t is not None]
    cells = np.floor((st["aabb"][moved, :3] + st["aabb"][moved, 3:]) * F32(0.5) / F32(cell)).astype(np.int64)
    outside = np.any((cells < lo) | (cells > hi), axis=1)
    assert outside.any() and (kind != "straddle" or (~outside).any())
    _check(got, want, (7 if kind == "straddle" else 28) * len(moved) // 8)


@pytest.mark.gpu
@pytest.mark.parametrize("search", list(SEARCH))
def test_sixteen_bit_cap(gpu, E, search):
    """A world 70 000 cells wide in x: the field has 16 bits, so bodies inside the measured extent clamp at x = 65534, a
    static sphere among them included; clusters at the far end and between the cap and the far end."""
    S = Scene(E)
    cell = _cell_pitch(2 * R_SPHERE)
    far = 70000
    park = frame(S, LO, np.array([far, 10, 10]), cell, 8 * 3)
    cluster(S, (far, 10, 9), cell)                 # against the static sphere at the far corner (body 1)
    cluster(S, (far - 3, 2, 2), cell)
    cluster(S, (40000, 5, 5), cell)                # past the cap, inside the extent
    for d, p in zip(S.defs[2:], park):
        d.position = p
    got, want, box, _ = run_case(E, S, SEARCH[search])
    assert box[1][0] - box[0][0] == 65534 and box[1][0] < 40000
    assert any(1 in p for p in want)
    _check(got, want, 3 * 10)


@pytest.mark.gpu
@pytest.mark.parametrize("search", list(SEARCH))
def test_clamped_near_large_bodies_filters_and_sleepers(gpu, E, search):
    """Clamped clusters resting on a plane and against a static box large enough for the brute-force list (F_LARGE), with
    collision filters, exclusions and sleeping bodies inside the clamped cells."""
    S = Scene(E)
    R = S.R
    cell = _cell_pitch(2 * R_SPHERE)
    lo, hi = _box_of_frame(cell)
    S.add(R.RigidBodyDef(kind=R.STATIC, shape=R.plane_shape((0, 1, 0), float((lo[1] - 3) * cell))))
    bx = (np.array([hi[0] + 8, (LO[1] + HI[1]) // 2, (LO[2] + HI[2]) // 2]) + 0.5) * cell
    S.add(R.RigidBodyDef(kind=R.STATIC, position=tuple(bx.tolist()), shape=R.box_shape((0.3, 3.0, 3.0))))
    centres = [np.array([(LO[0] + HI[0]) // 2, lo[1] - 3, hi[2] + 5]),        # on the plane, past +z and below -y
               np.array([hi[0] + 8, 0, 0]),                                     # against the box, past +x
               np.array([hi[0] + 9, 12, 14]),
               np.array([lo[0] - 4, lo[1] - 3, lo[2] - 4])]                     # on the plane at a corner
    n_park = 8 * len(centres)
    park_at = frame(S, LO, HI, cell, n_park)
    groups = [1, 2, 6]
    ids = []
    for k, c in enumerate(centres):
        c = c.astype(np.float64)
        if k in (0, 3):
            c[1] = lo[1] - 3 + (R_SPHERE + 0.005) / cell - 0.5            # lowest layer just above the plane
        if k == 1:
            c[0] = hi[0] + 8 - (0.3 + 0.49) / cell                          # touching the box's -x face
        for j, i in enumerate(cluster(S, c, cell)):
            ids.append(i)
            if k == 2:                                                      # filters: group g collides with mask g only
                S.defs[i].collision_group = S.defs[i].collision_mask = groups[j % 3]
    S.excl = [(ids[0], ids[1]), (ids[8], ids[10]), (ids[26], ids[27])]
    for d, p in zip(S.defs[4:], park_at):
        d.position = p
    sleepers = ids[24:28] + ids[8:10]

    def put_to_sleep(w, box):
        for _ in range(130):                         # at rest and unconnected: every island falls asleep after 2 s
            w.run_phases(E.world.PH_ISLANDS)
        awake = [i for i in range(len(S.defs)) if i not in sleepers]
        w.wake_bodies(awake)
        assert w.sleeping()[sleepers].all() and not w.sleeping()[ids[:8]].any()

    got, want, box, _ = run_case(E, S, SEARCH[search], flags=E.world.FLAG_SLEEPING, after_measure=put_to_sleep)
    plane, big = 0, 1
    assert any(plane in p for p in want) and any(big in p for p in want)
    _check(got, want, 40)


def _diameter(b):
    """shape_diameter (b2d_api.cu) in float32; planes infinite."""
    p = b["shape_params"].astype(F32)
    sk = b["shape_kind"]
    d = np.full(len(sk), np.inf, F32)
    d[sk == 0] = F32(2) * p[sk == 0, 0]
    d[sk == 2] = F32(2) * (p[sk == 2, 0] + p[sk == 2, 1])
    d[sk == 3] = F32(2) * np.sqrt(np.sum(p[sk == 3, :3] * p[sk == 3, :3], axis=1, dtype=F32))
    d[sk == SHAPE_NONE] = 0
    return d


def _gap_pair(pl, r1, r2, asymmetric, ulps):
    """x of two spheres (radii r1 left, r2 right) whose AABBs lie 0.02 apart to within float32 rounding, with the sphere
    AABBs the device computes (pos -+ r).  asymmetric: the right AABB starts where the left body's query (max + 0.02)
    still reaches it but the right body's query (min - 0.02) misses the left AABB -- possible where max + 0.02 crosses a
    power of two and rounds on the coarser grid above it (the opposite case does not occur in float32); else `ulps` steps
    from max + 0.02, whatever the two queries then say."""
    c = F32(0.02)
    a = F32(pl + r1)                                       # left AABB max
    b0 = F32(a + c)
    for k in range(-8, 9):
        b = b0
        for _ in range(abs(k)):
            b = np.nextafter(b, F32(np.inf) if k > 0 else F32(-np.inf), dtype=F32)
        left_hits, right_hits = F32(a + c) >= b, F32(b - c) <= a
        if (asymmetric and left_hits and not right_hits) or (not asymmetric and k == ulps):
            break
    pr = F32(b + r2)
    for _ in range(8):                                     # a centre whose AABB min rounds to b
        if F32(pr - r2) == b:
            break
        pr = np.nextafter(pr, F32(np.inf) if F32(pr - r2) < b else F32(-np.inf), dtype=F32)
    return pl, pr


@pytest.mark.gpu
@pytest.mark.parametrize("search", list(SEARCH))
@pytest.mark.parametrize("seed", range(2 if EMU else 6))
def test_random_clamped_placements(gpu, E, search, seed):
    """Seeded fuzz: spheres, boxes and capsules of random size and orientation in clusters at random offsets relative to
    the measured key box (inside, on its first and last fields, a few cells past it, past edges and corners), and pairs of
    spheres whose AABBs are 0.02 +- a few ulps apart, where only one of the two queries may hit: then body[0] is the
    lower id."""
    rng = np.random.default_rng(1000 + seed)
    S = Scene(E)
    R = S.R
    shapes, centres = [], []
    for _ in range(10):
        centres.append([rng.choice(["in", "lo", "hi", "below", "above"]) for _ in range(3)])
        for _ in range(int(rng.integers(3, 7))):
            shapes.append([R.sphere_shape(float(rng.uniform(0.1, 0.3))), R.box_shape(tuple(rng.uniform(0.08, 0.2, 3))),
                           R.capsule_shape(float(rng.uniform(0.08, 0.15)), float(rng.uniform(0.1, 0.2)), int(rng.integers(3)))][rng.integers(3)])
    n_gap = 12
    n_park = len(shapes) + 2 * n_gap
    # the cell pitch follows the largest shape: place the frame in cells of that pitch
    cell = _cell_pitch(max(float(_diameter(R.bodies_soa([R.RigidBodyDef(shape=s)]))[0]) for s in shapes + [R.sphere_shape(R_SPHERE)]))
    park = frame(S, LO, HI, cell, n_park)
    lo, hi = _box_of_frame(cell)
    mid = (LO + HI) // 2

    def axis_cell(where, k):
        off = int(rng.integers(0, 6))
        return {"in": mid[k] + int(rng.integers(-3, 4)), "lo": lo[k] - off // 3, "hi": hi[k] + off // 3,
                "below": lo[k] - 1 - off, "above": hi[k] + 1 + off}[where]

    k = 0
    for where in centres:
        c = (np.array([axis_cell(wh, a) for a, wh in enumerate(where)], np.float64) + 0.5) * cell
        n = int(rng.integers(3, 7)) if k < len(shapes) else 0
        for s in shapes[k:k + n]:
            S.add(R.RigidBodyDef(position=(0, 0, 0), gravity=(0, 0, 0), shape=s,
                                 orientation=tuple((lambda q: q / np.linalg.norm(q))(rng.normal(size=4)).tolist())),
                  tuple((c + rng.uniform(-0.35, 0.35, 3)).tolist()))
        k += n
    for s in shapes[k:]:
        S.add(R.RigidBodyDef(position=(0, 0, 0), gravity=(0, 0, 0), shape=s), tuple(((mid + 0.5) * cell + rng.uniform(-0.4, 0.4, 3)).tolist()))
    for g in range(n_gap):
        r1, r2 = F32(rng.uniform(0.1, 0.25)), F32(rng.uniform(0.1, 0.25))
        where = [rng.choice(["in", "hi", "above", "lo", "below"]) for _ in range(3)]
        p = (np.array([axis_cell(wh, a) for a, wh in enumerate(where)], np.float64) + 0.5) * cell
        asym = g % 2 == 0
        if asym:                                           # the left AABB ends just below 4 or 8 m (y and z may lie outside)
            p[0] = (4.0 if g % 4 else 8.0) - rng.uniform(0.0005, 0.019) - float(r1)
        else:
            p[0] += 20.0                                   # larger coordinates: coarser ulps
        pl, pr = _gap_pair(F32(p[0]), r1, r2, asym, int(rng.integers(-3, 4)))
        pa, pb = p.copy(), p.copy()
        pa[0], pb[0] = float(pl), float(pr)
        for r, q in ((r1, pa), (r2, pb)):                  # the right sphere, whose query misses, takes the higher id
            S.sphere(tuple(q.tolist()), r=float(r))
    for d, q in zip(S.defs[2:], park):
        d.position = q
    got, want, box, st = run_case(E, S, SEARCH[search])
    _check(got, want, 20)
    dyn = np.asarray(R.bodies_soa(S.defs)["kind"]) == 0
    swapped = sum(v for (p0, p1), v in want.items() if p0 < p1 and dyn[p0] and dyn[p1])
    assert swapped > 0, "no pair took the branch where only the lower id's query hits"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain"] if EMU else ["plain", "graph"])
@pytest.mark.parametrize("search", list(SEARCH))
def test_falling_past_the_key_box(gpu, E, mode, search):
    """Whole steps: a cluster slides off a finite static box floor and columns of spheres beside it fall, the upper ones a
    little faster, so they meet only after they have left the key box measured at the first step (about 9 m down).  Every step's manifold
    pairs against the brute force over the AABBs and the manifolds the previous step left."""
    R = E.rigidbody
    steps = 36 if EMU else 90
    defs = [R.RigidBodyDef(kind=R.STATIC, position=(0, -0.1, 0), shape=R.box_shape((2.0, 0.1, 2.0)))]
    for i in np.ndindex(2, 2, 2):
        defs.append(R.RigidBodyDef(position=tuple((np.array([1.0, 0.25, 0.0]) + np.array(i) * GAP).tolist()), linvel=(4.0, 0, 0), shape=R.sphere_shape(R_SPHERE)))
    for c, closing in enumerate((0.055, 0.065, 0.08)):     # the 0.03 m above the 0.02 margin close at 0.55 .. 0.375 s
        for k in range(5):
            defs.append(R.RigidBodyDef(position=(3.0 + 0.8 * c, 0.25 + 0.55 * k, 1.0 - 0.8 * c), linvel=(0, -25.0 - closing * k, 0),
                                       shape=R.sphere_shape(R_SPHERE)))
    scene = dict(bodies=R.bodies_soa(defs), hinges=None, exclusions=None, settings=dict(velocity_iterations=6, position_iterations=2))
    b = scene["bodies"]
    w = build_world(E, scene, mode, SEARCH[search])
    try:
        cell = _cell_pitch(2 * R_SPHERE)
        bb0 = w.download_state()["aabb"]
        lo, _ = key_box(bb0, cell, np.arange(1, len(defs)))
        before, met_outside = [], 0
        for s in range(steps):
            bb = w.download_state()["aabb"]
            w.step(1)
            got = Counter(map(tuple, w.pairs().tolist()))
            want = brute_force_broadphase(bb, b["kind"], b["shape_kind"], manifolds=before)
            assert got == want, f"step {s}: extra {dict(got - want)}, missing {dict(want - got)}"
            below = np.floor((bb[:, 1] + bb[:, 4]) * F32(0.5) / F32(cell)) < lo[1]
            met_outside += sum(v for p, v in (want - Counter(map(tuple, before))).items() if below[p[0]] and below[p[1]])
            before = w.pairs().tolist()
        assert w.stats()["error_flags"] == 0
        assert met_outside > 0, "no pair was found below the key box"
    finally:
        w.close()
