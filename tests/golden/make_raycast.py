"""Regenerates tests/golden/raycast.npz: the reference's own edyn::shape_raycast (src/edyn/collision/raycast.cpp, through
tests/raycast/ref_raycast.cpp) on sphere / box / capsule / plane cases, raw (unfiltered) fraction, normal and feature.

    python tests/golden/make_raycast.py          # needs /root/reference at build time; the .npz travels, the reference does not

Every case sits in a cell of its own, 100 m from the next, with its segment inside that cell, so the non-plane cases can
run as one world and one batch on the device without moving anything (planes are infinite: they are checked one by one).
Cases: segments through, past, from inside and short of the shape, ending short and reaching beyond it, axis-aligned ones
(box faces, parallel to a box face within EDYN_EPSILON, along capsule axes) and grazing ones (tangent to a sphere, the
distance off by a few ulps either way).  The capsule hemisphere normals of segments along the capsule axis are the
reference's undefined behaviour (it reads an unwritten u_in, raycast.cpp:217, geom.cpp:1248-1250) and differ between
builds; no test compares them.  Consumers: tests/test_raycast.py (oracle == reference bits, the filter rule),
tests/test_gpu_raycast.py (device, one batch)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "raycast.npz")
SPHERE, CAPSULE, BOX, PLANE = 0, 2, 3, 6
PER_KIND = 600
EPS = np.float32(np.finfo(np.float32).eps)


def cell_origin(i):
    return np.array([(i % 16) * 100.0, ((i // 16) % 16) * 100.0, (i // 256) * 100.0], np.float32)


def cases(rng):
    out = []
    for i in range(4 * PER_KIND):
        kind = [SPHERE, BOX, CAPSULE, PLANE][i % 4]
        o = cell_origin(i)
        p = np.zeros(4, np.float32)
        q = rng.normal(size=4)
        orn = (q / np.linalg.norm(q)).astype(np.float32) if i % 3 else np.array([0, 0, 0, 1], np.float32)
        pos = (o + rng.uniform(-1, 1, 3)).astype(np.float32)
        if kind == PLANE:
            n = rng.normal(size=3) if i % 8 != 3 else np.eye(3)[rng.integers(3)]
            p[:3] = (n / np.linalg.norm(n)).astype(np.float32)
            p[3] = np.float32(np.dot(p[:3].astype(np.float64), o.astype(np.float64)) + rng.uniform(-1, 1))
            pos = o.copy()
        else:
            p[:3] = rng.uniform(0.1, 1.0, 3)
            if kind == CAPSULE:
                p[2] = rng.integers(0, 3)
        mode = (i // 4) % 8
        p0 = (pos + rng.normal(size=3) * 3).astype(np.float32)
        if mode == 0:                                              # through the centre
            p1 = (pos + (pos - p0) * rng.uniform(0.2, 2.0)).astype(np.float32)
        elif mode == 1:                                            # from inside
            p0 = (pos + rng.normal(size=3) * 0.05).astype(np.float32)
            p1 = (p0 + rng.normal(size=3) * 3).astype(np.float32)
        elif mode == 2:                                            # axis-aligned (world axes; parallel to box faces at identity)
            p1 = p0.copy(); p1[rng.integers(3)] -= np.float32(rng.uniform(-6, 6))
        elif mode == 3:                                            # ends short of it
            p1 = (p0 + (pos - p0) * 0.3).astype(np.float32)
        elif mode == 4 and kind == SPHERE:                         # grazing: tangent, distance off by a few ulps
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            u = np.cross(d, rng.normal(size=3)); u /= np.linalg.norm(u)
            r = p[0] * (1 + rng.integers(-4, 5) * EPS)
            p0 = (pos + u * r - d * 3).astype(np.float32); p1 = (pos + u * r + d * 3).astype(np.float32)
        elif mode == 4 and kind == BOX:                            # parallel to a face within EPSILON, on its plane +- ulps
            orn = np.array([0, 0, 0, 1], np.float32)
            a = rng.integers(3)
            p0 = (pos + rng.uniform(-0.5, 0.5, 3) * p[:3]).astype(np.float32)
            p0[a] = pos[a] + p[a] * (1 + rng.integers(-3, 4) * EPS)
            p1 = p0.copy(); b = (a + 1) % 3
            p1[b] += np.float32(6); p0[b] -= np.float32(3); p1[a] += np.float32(EPS * 0.25)
        elif mode == 4 and kind == CAPSULE:                        # along the capsule axis (parallel branch)
            ax = np.zeros(3); ax[int(p[2])] = 1
            x, y, z, w = orn.astype(np.float64)
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
            d = R @ ax
            off = np.cross(d, rng.normal(size=3)); off = off / np.linalg.norm(off) * rng.uniform(0, 0.8) * p[0]
            p0 = (pos + off + d * 4).astype(np.float32); p1 = (pos + off - d * rng.uniform(0.5, 8)).astype(np.float32)
        elif mode == 5:                                            # reaching beyond it: the hit lies past p1
            p1 = (p0 + (pos - p0) * 0.1).astype(np.float32)
            p0, p1 = p1, p0
        else:
            p1 = (pos + rng.normal(size=3) * 3).astype(np.float32)
        if kind == BOX and np.array_equal(p0, p1):
            p1 = p1 + np.float32(1)                                # the reference reads get_face_normal(SIZE_MAX) otherwise
        out.append((kind, p, pos, orn, p0, p1))
    return out


def main():
    from tests import raycast_support as S
    lib = S.ref()
    if lib is None:
        raise SystemExit("the reference's object files are needed (oracle/_ref/edyn_obj: build() where /root/reference exists)")
    rng = np.random.default_rng(20261015)
    cs = cases(rng)
    n = len(cs)
    kind = np.array([c[0] for c in cs], np.uint32)
    params, pos, orn, p0, p1 = (np.stack([c[k] for c in cs]).astype(np.float32) for k in range(1, 6))
    frac, nrm, feat = np.zeros(n, np.float32), np.zeros((n, 3), np.float32), np.zeros(n, np.uint32)
    for i in range(n):
        _, frac[i], nrm[i], feat[i] = S.shape_raycast(lib, "rr_", kind[i], params[i], pos[i], orn[i], p0[i], p1[i])
    np.savez_compressed(OUT, kind=kind, params=params, pos=pos, orn=orn, p0=p0, p1=p1, fraction=frac, normal=nrm, feature=feat)
    hit = frac != np.float32(np.finfo(np.float32).max)
    print(f"{OUT}: {n} cases, {int(hit.sum())} with a reference result, {int((hit & (frac >= 0) & (frac <= 1)).sum())} of them in [0, 1]")


if __name__ == "__main__":
    main()
