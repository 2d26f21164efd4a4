"""TEST INFRASTRUCTURE.  The raycast kernels (k_ray_* in b2d_kernels.cuh) against the CPU brute force
(tests/raycast/ora_raycast.cpp), bit for bit: body, fraction, normal and feature of every segment.  Also the scene and segment
generators the GPU raycast tests use.

    python tests/emu/raycast.py SEED [SEED ...]      -> one JSON line (runs the kernels under the CPU emulation)
Runs in its own process because B2D_LIB has to be set before edyn_b200 is imported."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests import raycast_support as S  # noqa: E402

SPHERE, CAPSULE, BOX, PLANE = 0, 2, 3, 6


def random_quat(rng, n):
    q = rng.normal(size=(n, 4)).astype(np.float32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)


def scene(rng, n=300, extent=12.0, far=0):
    """Random bodies: dynamic / kinematic / static spheres, capsules and boxes (static ones tilted), a few large boxes, a
    tilted ground plane and `far` bodies hundreds of metres away from the rest."""
    kind = rng.choice([0, 0, 0, 1, 2], size=n).astype(np.uint32)
    shape = rng.choice([SPHERE, CAPSULE, BOX], size=n).astype(np.uint32)
    params = np.zeros((n, 4), np.float32)
    params[:, 0] = rng.uniform(0.1, 0.6, n)
    params[:, 1] = rng.uniform(0.1, 0.6, n)
    params[:, 2] = rng.uniform(0.1, 0.6, n)
    cap = shape == CAPSULE
    params[cap, 2] = rng.integers(0, 3, cap.sum())
    pos = rng.uniform(-extent, extent, (n, 3)).astype(np.float32)
    pos[:, 1] = rng.uniform(0.0, extent, n)
    big = rng.choice(n, size=max(1, n // 60), replace=False)          # larger than 4 x the mean: the brute-force list
    shape[big] = BOX; kind[big] = 2; params[big, :3] = rng.uniform(2.0, 4.0, (len(big), 3))
    if far:
        fi = rng.choice(n, size=far, replace=False)
        pos[fi] += rng.choice([-1.0, 1.0], size=(far, 3)).astype(np.float32) * rng.uniform(300, 900, (far, 3)).astype(np.float32)
    orn = random_quat(rng, n)
    # one tilted ground plane
    nrm = np.array([0.1, 1.0, -0.05], np.float32); nrm /= np.linalg.norm(nrm)
    kind = np.append(kind, np.uint32(2)); shape = np.append(shape, np.uint32(PLANE))
    params = np.vstack([params, np.append(nrm, np.float32(-0.5))[None]]).astype(np.float32)
    pos = np.vstack([pos, np.zeros((1, 3), np.float32)]); orn = np.vstack([orn, np.array([[0, 0, 0, 1]], np.float32)])
    m = len(kind)
    dyn = kind == 0
    return dict(pos=pos, orn=orn, linvel=np.zeros((m, 3), np.float32), angvel=np.zeros((m, 3), np.float32),
                inv_mass=np.where(dyn, 1.0, 0.0).astype(np.float32),
                inv_inertia=np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (m, 1)) * dyn[:, None].astype(np.float32),
                gravity=np.tile(np.array([0, -9.8, 0], np.float32), (m, 1)) * dyn[:, None].astype(np.float32),
                kind=kind, shape_kind=shape, shape_params=params, friction=np.full(m, 0.5, np.float32),
                restitution=np.zeros(m, np.float32))


def segments(rng, pos, n, extent=12.0):
    """Mixed segments: random ones through the scene, short ones starting at body centres (inside the body), long ones,
    axis-aligned ones, zero-length ones, ones with a NaN or infinite coordinate and ones ending at a body centre."""
    p0 = rng.uniform(-extent * 1.2, extent * 1.2, (n, 3)).astype(np.float32)
    p1 = rng.uniform(-extent * 1.2, extent * 1.2, (n, 3)).astype(np.float32)
    k = n // 8
    src = rng.integers(0, len(pos), k)
    p0[:k] = pos[src]
    p1[:k] = pos[src] + rng.normal(size=(k, 3)).astype(np.float32) * 2
    p1[k:2 * k] = p0[k:2 * k] * 80                                         # long: out to the far bodies
    axis = rng.integers(0, 3, k)
    p1[2 * k:3 * k] = p0[2 * k:3 * k]
    p1[2 * k + np.arange(k), axis] -= np.float32(extent)                   # axis-aligned
    p1[3 * k:3 * k + 4] = p0[3 * k:3 * k + 4]                              # zero length
    p0[3 * k + 4, 1] = np.nan
    p1[3 * k + 5, 0] = np.inf
    tgt = pos[rng.integers(0, len(pos), k)]                                # aimed at body centres, far ones included, from
    p1[4 * k:5 * k] = tgt                                                  # a few tens of metres away
    p0[4 * k:5 * k] = tgt + rng.uniform(-30, 30, (k, 3)).astype(np.float32)
    return p0, p1


def _bits_differ(x, y):
    """Bitwise inequality, except that any two NaNs are equal: the reference's normal is NaN for a segment through a
    sphere's centre or a capsule's axis (0 / 0), and the GPU and the CPU spell that NaN differently."""
    return (x.view(np.uint32) != y.view(np.uint32)) & ~(np.isnan(x) & np.isnan(y))


def compare(a, b):
    """Bitwise equality of two raycast result dicts; returns (#rays, #mismatches, first mismatch index or -1)."""
    bad = (a["body"] != b["body"]) | (a["feature"] != b["feature"]) | _bits_differ(a["fraction"], b["fraction"]) | \
          _bits_differ(a["normal"], b["normal"]).any(axis=1)
    idx = np.nonzero(bad)[0]
    return len(bad), int(len(idx)), int(idx[0]) if len(idx) else -1


def check_world(E, seed, n=300, rays=1500, steps=3):
    """One random world through its life: right after add_bodies, after steps, after removals and after more bodies
    arrived far outside the grid's measured extent; both ignore forms.  Returns a list of per-stage results."""
    rng = np.random.default_rng(seed)
    soa = scene(rng, n, far=8)
    nb = len(soa["kind"])
    w = E.World(max_bodies=nb + 64)
    o = S.BruteWorld()
    w.add_bodies(soa); o.add_bodies(soa)
    out = []

    def stage(name):
        st = w.download_state()
        p0, p1 = segments(rng, st["pos"], rays)
        ign = rng.choice(w.num_bodies, size=5, replace=False)
        ib = rng.integers(0, w.num_bodies, rays).astype(np.uint32)
        ib[::3] = E.RAY_MISS
        for kw in (dict(), dict(ignore=ign), dict(ignore_body=ib), dict(ignore=ign, ignore_body=ib)):
            g = w.raycast(p0, p1, **kw)
            c = o.raycast(p0, p1, **kw)
            total, bad, first = compare(g, c)
            hits = int((c["body"] != E.RAY_MISS).sum())
            out.append(dict(stage=name, ignore=sorted(kw), rays=total, hits=hits, mismatches=bad, first=first))

    stage("after add_bodies")
    w.step(steps)
    g = w.download_state()
    o.set_state(g["pos"], g["orn"], g["linvel"], g["angvel"])
    stage("after steps")
    dead = rng.choice(n, size=10, replace=False)
    w.remove_bodies(dead); o.remove_bodies(dead)
    stage("after remove_bodies")
    more = {k: v[:-1] for k, v in scene(rng, 24, extent=4.0).items()}      # no second plane
    more["pos"] = more["pos"] + np.float32(5000.0)                          # beyond the cell key range measured at the last step
    w.add_bodies(more); o.add_bodies(more)
    g = w.download_state()
    o.set_state(g["pos"], g["orn"], g["linvel"], g["angvel"])
    stage("after add_bodies outside the extent")
    w.close()
    return out


def main():
    from tests.emu import build
    lib = build.build()
    os.environ.update(B2D_EMU="1", B2D_LIB=lib, B2D_GRAPH="0")
    import edyn_b200 as E
    res = []
    for s in sys.argv[1:]:
        res.extend(check_world(E, int(s), n=120, rays=400, steps=2))
    print(json.dumps(dict(results=res)))


if __name__ == "__main__":
    main()
