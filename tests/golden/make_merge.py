"""Regenerates tests/golden/merge.npz: the reference's own narrowphase (narrowphase::update: update_contact_distances,
detect_collision, process_collision with its sequential create / destroy functors) on manifolds seeded with 0-4 points,
through oracle/ref_stepper.cpp (refs_seed_manifolds, refs_narrowphase, refs_get_seeded).

    python tests/golden/make_merge.py          # needs oracle/_ref (build() where /root/reference exists)

A case is two bodies and one manifold.  Shape families: every pair the three narrowphase kernels run (the seven light
types, box-box, capsule-box), each in both body orders; partners are static planes, static and kinematic boxes and
dynamic bodies, so dynamic spheres and capsules roll on either side.  The persisted points are built around this step's
collision result in the bodies' local frames, with offsets spread across the thresholds that decide the branches
(MERGING 0.01, BREAKING 0.02 along the normal and tangentially, CACHING 0.04), collinear triples and near-duplicates,
random lifetimes (2^30 - 1 and 2^30 - 2 among them), non-zero impulses, and a friction and restitution that differ from
the material mix.  Only the narrowphase runs, on the seeded manifolds alone, so every case sits
near the origin (where float32 positions are finest) and bodies of different cases may overlap.  Cases are drawn in
batches and kept while they reach a branch of process_collision that has fewer
than QUOTA cases (the oracle's merge trace, OracleWorld.merge_trace), plus a few at random.

Rolling cases keep every distance find_nearest_contact_rolling compares with CACHING_THRESHOLD^2 at least 1e-3 relative
away from it: that is the one decision that goes through sinf / cosf (integrate(orn, angvel, -dt)), so with that margin
every output column is a copied or correctly rounded value and the device, the oracle and the reference agree bit for bit.
Consumers: tests/test_oracle_merge.py (oracle == these vectors, oracle == reference on fresh cases),
tests/test_gpu_merge.py (device == these vectors, device == oracle on fresh cases)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "merge.npz")
SEED = 20261017
SPHERE, CAPSULE, BOX, PLANE = 0, 2, 3, 6
DYNAMIC, KINEMATIC, STATIC = 0, 1, 2
FAMILIES = [(SPHERE, SPHERE), (SPHERE, PLANE), (BOX, PLANE), (CAPSULE, PLANE), (SPHERE, BOX), (CAPSULE, CAPSULE),
            (CAPSULE, SPHERE), (BOX, BOX), (CAPSULE, BOX)]
MERGING, BREAKING, CACHING = 0.01, 0.02, 0.04
DT = np.float32(1.0 / 60)
QUOTA = 25
# ins3_col2: no input reaches it.  insertion_point_index's collinear branch computes d2 = dot(p2 - p0, p1 - p0), the same
# products summed in the same order as d0 = dot(p1 - p0, p2 - p0), so d2 == d0 bit for bit, and d0 in (0, 1) has
# already returned REPLACE at index 1.
# similar_then_replace: a result point SIMILAR to a persisted point P that P did not take (it merged, through pivot B,
# into a third result point), then a fourth result point REPLACE-ing the same index: four-point results in that
# arrangement; the sampling here has not produced one in 48 000 candidates.
UNREACHABLE = ("ins3_col2",)
NOT_SAMPLED = ("similar_then_replace",)
f32 = np.float32


def rot(q):
    x, y, z, w = (float(v) for v in q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def unit(v):
    return v / np.linalg.norm(v)


def rand_quat(rng):
    return unit(rng.normal(size=4)).astype(f32)


def shape_params(rng, kind):
    p = np.zeros(4, f32)
    tiny = rng.random() < 0.25                   # result points closer than MERGING: SIMILAR onto a point created this pass
    if kind == SPHERE:
        p[0] = rng.uniform(0.2, 0.6)
    elif kind == CAPSULE:
        p[:3] = rng.uniform(0.15, 0.4), (rng.uniform(0.002, 0.0045) if tiny else rng.uniform(0.2, 0.6)), rng.integers(3)
    elif kind == BOX:
        p[:3] = rng.uniform(0.2, 0.7, 3)
        if tiny:
            p[rng.integers(3)] = rng.uniform(0.002, 0.0045)
            p[rng.integers(3)] = rng.uniform(0.002, 0.0045)
    else:
        p[:4] = 0, 1, 0, 0
    return p


def bound(kind, p):
    return {SPHERE: p[0], CAPSULE: p[0] + p[1], BOX: float(np.linalg.norm(p[:3]))}.get(kind, 0.0)


def place(rng, fns, kA, pA, kB, pB, origin):
    """Poses that touch: B moved along a random direction (or A above the plane B) to the largest separation at which
    collide() still reports points, minus a random penetration.  Returns posA, ornA, posB, ornB."""
    ornA, ornB = rand_quat(rng), rand_quat(rng)
    if rng.random() < 0.3:                      # axis-aligned: face contacts, parallel capsules
        ornA = np.array([0, 0, 0, 1], f32)
        ornB = np.array([0, 0, 0, 1], f32) if rng.random() < 0.5 else ornB
    posA = (origin + rng.uniform(-1, 1, 3)).astype(f32)
    if kB == PLANE or kA == PLANE:
        d = np.array([0.0, 1.0, 0.0])
    else:
        d = unit(rng.normal(size=3)) if rng.random() < 0.7 else np.eye(3)[rng.integers(3)] * rng.choice([-1, 1])
    plane_first = kA == PLANE

    def poses(t):
        if kB == PLANE:
            return (origin + d * t).astype(f32), ornA, origin.astype(f32), np.array([0, 0, 0, 1], f32)
        if plane_first:
            return origin.astype(f32), np.array([0, 0, 0, 1], f32), (origin + d * t).astype(f32), ornB
        return posA, ornA, (posA + d * t).astype(f32), ornB

    lo, hi = 0.0, bound(kA, pA) + bound(kB, pB) + 0.1
    for _ in range(18):
        mid = 0.5 * (lo + hi)
        pa, oa, pb, ob = poses(mid)
        if len(fns.collide(kA, pA, kB, pB, pa, oa, pb, ob)[0]):
            lo = mid
        else:
            hi = mid
    return poses(max(0.0, lo - rng.choice([rng.uniform(-0.01, 0.0), rng.uniform(0.0, 0.02), rng.uniform(0.02, 0.06)])))


def to_world(p, pos, orn):
    return rot(orn) @ np.asarray(p, np.float64) + pos


def to_local(p, pos, orn):
    return rot(orn).T @ (np.asarray(p, np.float64) - pos)


def persisted(rng, res, posA, ornA, posB, ornB, prev):
    """0-4 points around the result res (n, 10: pivotA pivotB normal distance), in slot order.  prev: per body its
    orientation one step back (integrate(orn, angvel, -dt)) if it rolls, else None."""
    n_res = len(res)
    num = int(rng.choice([0, 1, 2, 3, 4], p=[0.08, 0.17, 0.25, 0.25, 0.25]))
    pts = np.zeros((4, 18), f32)
    att = np.zeros(4, np.uint32)
    life = np.zeros(4, np.uint32)
    if n_res:
        n0 = res[0, 6:9].astype(np.float64)
        centre = to_world(res[:, 0:3].mean(0), posA, ornA)
    else:
        n0 = unit(rng.normal(size=3))
        centre = 0.5 * (posA.astype(np.float64) + posB.astype(np.float64))
    t1 = unit(np.cross(n0, rng.normal(size=3)))
    t2 = np.cross(n0, t1)
    rolls = [k for k in (0, 1) if prev[k] is not None]
    layout = rng.choice(["free", "collinear", "duplicates", "quad", "roll"], p=[0.4, 0.2, 0.1, 0.15, 0.15])
    if layout == "roll" and not rolls:
        layout = "free"
    cross_slot = int(rng.integers(4)) if rng.random() < 0.5 else -1
    line_dir = unit(t1 * rng.normal() + t2 * rng.normal())
    spacing = rng.choice([rng.uniform(0.02, 0.3), rng.uniform(0.4, 0.6), rng.uniform(1.05, 1.6)])
    order = rng.permutation(3)
    # half the lines run through a result point, so that the point is collinear with the persisted ones: the two-point
    # replace / none branches and every collinear three-point branch
    line_base = rng.choice([0.0, rng.uniform(0.05, 0.3)]) * rng.choice([-1, 1])
    if n_res and rng.random() < 0.5:
        centre_line = to_world(res[int(rng.integers(n_res)), 0:3], posA, ornA)
        line_base = rng.uniform(0.05, 0.3) * rng.choice([-1, 1]) if rng.random() < 0.6 else 0.0
    else:
        centre_line = centre
    quad = [(1, 1), (1, -1), (-1, -1), (-1, 1)]
    qs = rng.uniform(0.03, 0.4)
    for s in range(num):
        mode = rng.choice(["match", "cross", "free"], p=[0.45, 0.15, 0.4])
        if layout in ("collinear", "quad") and s < (3 if layout == "collinear" else 4):
            mode = "cross" if layout == "quad" and s == cross_slot else "free"
        elif layout == "roll":
            mode = "roll"
        if not n_res:
            mode = "free"
        i = int(rng.integers(n_res)) if n_res else 0
        normal = res[i, 6:9].astype(np.float64) if n_res and rng.random() < 0.8 else unit(rng.normal(size=3))
        if mode == "roll":
            # the rolling search finds res[i]: the point's pivot, placed with the body's previous orientation, lands
            # near the result's pivotA placed with the same body's pose (for body B too, as the reference does)
            k = rolls[int(rng.integers(len(rolls)))]
            pos, orn = (posA, ornA) if k == 0 else (posB, ornB)
            target = to_world(res[i, 0:3], pos, orn) + unit(rng.normal(size=3)) * CACHING * rng.choice([rng.uniform(0.0, 0.8), rng.uniform(1.2, 2.0)])
            piv = to_local(target, pos, prev[k])
            other = res[i, 3:6] if k == 0 else res[i, 0:3]
            far = other + unit(rng.normal(size=3)) * CACHING * rng.uniform(1.1, 3.0)
            pa, pb = (piv, far) if k == 0 else (far, piv)
        elif mode in ("match", "cross"):
            scale = CACHING * rng.choice([rng.uniform(0.0, 0.25), rng.uniform(0.2, 0.9), rng.uniform(0.9, 1.1), rng.uniform(1.1, 2.0)])
            pa = res[i, 0:3] + unit(rng.normal(size=3)) * scale
            if mode == "cross" and n_res > 1:
                j = (i + 1 + int(rng.integers(n_res - 1))) % n_res
                pa = res[i, 0:3] + unit(rng.normal(size=3)) * MERGING * rng.uniform(0.1, 0.9)
                pb = res[j, 3:6] + unit(rng.normal(size=3)) * MERGING * rng.uniform(0.0, 0.3)
            else:
                pb = res[i, 3:6] + unit(rng.normal(size=3)) * CACHING * rng.choice([rng.uniform(0.0, 0.5), rng.uniform(0.9, 2.0)])
        else:
            if layout == "collinear" and s < 3:
                w = centre_line + line_dir * (line_base + spacing * (order[s] - (0 if line_base else 1)))
            elif layout == "duplicates" and s > 0:
                w = to_world(pts[s - 1, 0:3], posA, ornA) + rng.normal(size=3) * rng.choice([0.0, 1e-4, 0.004, 0.012])
            elif layout == "quad":
                w = centre + (t1 * quad[s][0] + t2 * quad[s][1]) * qs * rng.uniform(0.9, 1.1)
            else:
                w = centre + (t1 * rng.normal() + t2 * rng.normal()) * rng.choice([0.05, 0.2, 0.5])
            # separation of pB from pA: along the normal and tangentially, across BREAKING
            stay = layout in ("collinear", "quad") and rng.random() < 0.8
            dn = rng.choice([rng.uniform(-0.05, 0.0), rng.uniform(0.0, 0.019)] + ([] if stay else [rng.uniform(0.021, 0.05)]))
            dt = rng.choice([0.0, rng.uniform(0.0, 0.019)] + ([] if stay else [rng.uniform(0.021, 0.05)]))
            tang = unit(np.cross(normal, rng.normal(size=3)))
            pa = to_local(w, posA, ornA)
            pb = to_local(w - normal * dn - tang * dt, posB, ornB)
        pts[s, 0:3], pts[s, 3:6], pts[s, 6:9] = pa, pb, normal
        pts[s, 9:12] = unit(rng.normal(size=3))
        pts[s, 12] = rng.uniform(-0.05, 0.05)
        pts[s, 13], pts[s, 14] = rng.uniform(0.05, 1.5), rng.uniform(0.0, 0.9)
        pts[s, 15:18] = rng.uniform(0.01, 2.0), rng.uniform(-1, 1), rng.uniform(-1, 1)
        att[s] = rng.integers(3)
        life[s] = rng.choice([rng.integers(0, 50), rng.integers(0, 1 << 30), (1 << 30) - 1, (1 << 30) - 2])
    return num, pts, att, life


def rolling_margin_ok(fns, c):
    """Every distance find_nearest_contact_rolling compares with CACHING^2 is at least 1e-3 relative away from it."""
    thr = CACHING * CACHING
    res = c["res"]
    for side in (0, 1):
        if not c["rolling"][side] or not len(res):
            continue
        pos, orn, av = c["pos"][side], c["orn"][side], c["angvel"][side]
        prev = fns.integrate(orn, av, -DT)
        for s in range(c["num"]):
            piv = c["pts"][s, 3 * side:3 * side + 3]
            pp = to_world(piv, pos.astype(np.float64), prev)
            for r in res:
                d = float(np.sum((to_world(r[0:3], pos.astype(np.float64), orn) - pp) ** 2))
                if abs(d / thr - 1.0) < 1e-3:
                    return False
    return True


def candidate(rng, fns):
    kA, kB = FAMILIES[rng.integers(len(FAMILIES))]
    if rng.random() < 0.5:
        kA, kB = kB, kA
    pA, pB = shape_params(rng, kA), shape_params(rng, kB)
    origin = np.zeros(3)
    posA, ornA, posB, ornB = place(rng, fns, kA, pA, kB, pB, origin)
    kinds = []
    for k, other in ((kA, kB), (kB, kA)):
        if k == PLANE:
            kinds.append(STATIC)
        elif other == PLANE or len(kinds) and kinds[0] != DYNAMIC:
            kinds.append(DYNAMIC)
        else:
            kinds.append(int(rng.choice([DYNAMIC, DYNAMIC, STATIC, KINEMATIC])) if k == BOX or len(kinds) else DYNAMIC)
    if DYNAMIC not in kinds:
        kinds[int(rng.integers(2))] = DYNAMIC
    if kinds[0] != DYNAMIC and kinds[1] != DYNAMIC:
        kinds[0] = DYNAMIC
    angvel = np.zeros((2, 3), f32)
    for s in (0, 1):
        if kinds[s] == DYNAMIC and rng.random() < 0.8:
            angvel[s] = rng.normal(size=3) * rng.choice([0.5, 3.0, 12.0])
    res, _ = fns.collide(kA, pA, kB, pB, posA, ornA, posB, ornB)
    rolling = [kinds[s] == DYNAMIC and (kA, kB)[s] in (SPHERE, CAPSULE) for s in (0, 1)]
    prev = [fns.integrate(o, w, -DT) if r else None for o, w, r in zip((ornA, ornB), angvel, rolling)]
    num, pts, att, life = persisted(rng, res, posA, ornA, posB, ornB, prev)
    c = dict(kinds=np.array([kA, kB], np.uint32), params=np.stack([pA, pB]), pos=np.stack([posA, posB]), orn=np.stack([ornA, ornB]),
             body_kind=np.array(kinds, np.uint32), angvel=angvel, friction=rng.uniform(0.1, 1.0, 2).astype(f32),
             restitution=rng.uniform(0.0, 0.5, 2).astype(f32), num=num, pts=pts, att=att, lifetime=life, res=res,
             rolling=rolling)
    return c if rolling_margin_ok(fns, c) else None


def bodies(cs):
    """Body SoA of the cases, two bodies per case (case i: bodies 2i = A, 2i + 1 = B)."""
    n = 2 * len(cs)
    cat = lambda k: np.concatenate([c[k] for c in cs])
    return dict(pos=cat("pos"), orn=cat("orn"), linvel=np.zeros((n, 3), f32), angvel=cat("angvel"),
                inv_mass=np.where(cat("body_kind") == DYNAMIC, 1.0, 0.0).astype(f32),
                inv_inertia=np.tile(np.eye(3, dtype=f32).reshape(9), (n, 1)), gravity=np.zeros((n, 3), f32),
                kind=cat("body_kind"), shape_kind=cat("kinds"), shape_params=cat("params"), friction=cat("friction"),
                restitution=cat("restitution"), group=None, mask=None)


def manifolds(cs):
    """pairs, num, pts (m, 4, 18), att, lifetime of the cases' seeded manifolds."""
    m = len(cs)
    pairs = np.stack([2 * np.arange(m), 2 * np.arange(m) + 1], axis=1).astype(np.uint32)
    return (pairs, np.array([c["num"] for c in cs], np.uint32), np.stack([c["pts"] for c in cs]),
            np.stack([c["att"] for c in cs]), np.stack([c["lifetime"] for c in cs]))


def run_oracle(O, cs):
    """The oracle's narrowphase on the cases: (contacts dict, merge trace per case)."""
    o = O.OracleWorld(dt=float(DT))
    o.add_bodies(bodies(cs))
    o.set_contacts(*manifolds(cs))
    o.set_merge_trace(True)
    o.run_phases(O.PH_NARROW)
    return o.contacts(), o.merge_trace()


def run_reference(O, cs):
    r = O.RefWorld(dt=float(DT))
    r.add_bodies(bodies(cs), sleeping_disabled=True)
    r.seed_manifolds(*manifolds(cs))
    r.narrowphase()
    return r.seeded()


def draw(O, rng, total, quota=QUOTA, batch=400, random_share=0.02, max_batches=150):
    """Cases chosen by branch: a batch of candidates through the oracle, keep those that reach a branch still short of
    `quota` cases (and `random_share` of the others), until every reachable branch has its quota and `total` cases."""
    fns = O.ora_fns()
    counts = np.zeros(len(O.MERGE_BRANCHES), np.int64)
    reach = np.array([b not in UNREACHABLE + NOT_SAMPLED for b in O.MERGE_BRANCHES])
    keep = []
    for _ in range(max_batches):
        cs = [c for c in (candidate(rng, fns) for _ in range(batch)) if c is not None]
        _, tr = run_oracle(O, cs)
        for c, t in zip(cs, tr.tolist()):
            bits = np.array([(t >> b) & 1 for b in range(len(O.MERGE_BRANCHES))], bool)
            if (bits & (counts < quota)).any() or rng.random() < random_share:
                keep.append(c)
                counts += bits
        if len(keep) >= total and (counts[reach] >= quota).all():
            break
    return keep, counts


def main():
    from oracle import oracle as O
    if O.ref_stepper() is None:
        raise SystemExit("the reference's stepper library is needed (oracle/_ref/libedyn_stepper.so: build() where /root/reference exists)")
    rng = np.random.default_rng(SEED)
    cs, _ = draw(O, rng, total=1500)
    got = run_reference(O, cs)
    pairs, num, pts, att, life = manifolds(cs)
    b = bodies(cs)
    np.savez_compressed(OUT, pos=b["pos"], orn=b["orn"], angvel=b["angvel"], kind=b["kind"], shape_kind=b["shape_kind"],
                        shape_params=b["shape_params"], friction=b["friction"], restitution=b["restitution"],
                        num=num, pts=pts, att=att, lifetime=life,
                        out_num=got["num"], out_pts=got["pts"], out_att=got["att"], out_lifetime=got["lifetime"])
    print(f"{OUT}: {len(cs)} cases, {int(num.sum())} persisted points, {int(got['num'].sum())} points after the merge")


if __name__ == "__main__":
    main()
