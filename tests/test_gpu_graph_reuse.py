"""Island rebuild reuse: a CUDA-graph step skips the connected components, colouring, tile packing and solver-order sorts
while the constraint graph is unchanged.  The results must be the bits of plain launches, which rebuild every step."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINKS = 4


def _world(E, scene, monkeypatch, graph, reuse=True):
    with monkeypatch.context() as m:
        m.setenv("B2D_GRAPH", "1" if graph else "0")
        m.setenv("B2D_GRAPH_REUSE", "1" if reuse else "0")
        return E.scenes.build_world(scene)


def _same(a, b):
    sa, sb = a.download_state(), b.download_state()
    for k in ("pos", "orn", "linvel", "angvel", "aabb"):
        assert np.array_equal(sa[k], sb[k]), k


@pytest.mark.parametrize("timing", [True, False])
def test_reused_rebuild_matches_plain_launches(gpu, E, monkeypatch, timing):
    """A settled slice of the chains workload, 200 steps as graphs with reuse, as graphs without and as plain launches.
    Mid-run one chain is thrown upwards (its plane contacts break and re-form) and one body is removed."""
    scene = E.scenes.hinge_chains(16, 16, LINKS)
    plain = _world(E, scene, monkeypatch, graph=False)
    reuse = _world(E, scene, monkeypatch, graph=True)
    full = _world(E, scene, monkeypatch, graph=True, reuse=False)
    worlds = (plain, reuse, full)
    for w in worlds:
        w.set_timing(timing)
        w.step(150)                                            # settle, as bench.py does
    _same(plain, reuse); _same(plain, full)

    def counts():
        st = reuse.stats()
        return st["steps_rebuilt"], st["steps_reused"]

    # settled: nothing is created or destroyed, the rebuild is skipped on (almost) every step
    r0, u0 = counts()
    for w in worlds:
        w.step(60)
    r1, u1 = counts()
    assert (r1 - r0) + (u1 - u0) == 60
    assert u1 - u0 >= 54, (r1 - r0, u1 - u0)
    _same(plain, reuse); _same(plain, full)

    # throw chain 37 upwards: its manifolds with the plane are destroyed, then created again (with points, in the same
    # step) when it lands: at least two rebuilds, the other steps reuse
    ids = np.arange(37 * LINKS, 38 * LINKS, dtype=np.uint32)
    up = np.tile(np.array([0.0, 3.0, 0.0], np.float32), (LINKS, 1))
    for w in worlds:
        w.upload_bodies(ids, linvel=up)
        w.step(70)
    _same(plain, reuse); _same(plain, full)
    r2, u2 = counts()
    assert r2 - r1 >= 2 and u2 - u1 >= 50, (r2 - r1, u2 - u1)

    # remove one link of chain 101: its contact and its two hinges go
    r3, _ = counts()
    for w in worlds:
        w.remove_bodies(np.array([101 * LINKS + 2], np.uint32))
        w.step(1)
    r4, _ = counts()
    assert r4 - r3 == 1
    for w in worlds:
        w.step(69)
    _same(plain, reuse); _same(plain, full)

    st_r, st_f, st_p = reuse.stats(), full.stats(), plain.stats()
    assert st_f["steps_reused"] == 0 and st_f["steps_rebuilt"] == st_f["steps"]
    assert st_p["steps_reused"] == 0 and st_p["steps_rebuilt"] == st_p["steps"]
    assert st_r["steps_rebuilt"] + st_r["steps_reused"] == st_r["steps"]
    for st in (st_r, st_f, st_p):
        assert st["error_flags"] == 0
    assert st_r["kernel_launches"] == st_f["kernel_launches"]          # a skipped rebuild counts its kernels all the same
