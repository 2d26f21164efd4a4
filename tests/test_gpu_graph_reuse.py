"""Island rebuild reuse: a CUDA-graph step skips the connected components, colouring, tile packing and solver-order sorts
while the constraint graph is unchanged.  The results must be the bits of plain launches, which rebuild every step."""
import numpy as np
import pytest

from tests.parity import build_world, same_state

pytestmark = pytest.mark.gpu

LINKS = 4


@pytest.mark.parametrize("timing", [True, False])
def test_reused_rebuild_matches_plain_launches(gpu, E, timing):
    """A settled slice of the chains workload, 200 steps as graphs with reuse, as graphs without and as plain launches.
    Mid-run one chain is thrown upwards (its plane contacts break and re-form) and one body is removed."""
    scene = E.scenes.hinge_chains(16, 16, LINKS)
    plain = build_world(E, scene, env=dict(B2D_GRAPH="0", B2D_GRAPH_REUSE="1"))
    reuse = build_world(E, scene, env=dict(B2D_GRAPH="1", B2D_GRAPH_REUSE="1"))
    full = build_world(E, scene, env=dict(B2D_GRAPH="1", B2D_GRAPH_REUSE="0"))
    worlds = (plain, reuse, full)
    for w in worlds:
        w.set_timing(timing)
        w.step(150)                                            # settle, as bench.py does
    same_state(plain, reuse, full)

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
    same_state(plain, reuse, full)

    # throw chain 37 upwards: its manifolds with the plane are destroyed, then created again (with points, in the same
    # step) when it lands: at least two rebuilds, the other steps reuse
    ids = np.arange(37 * LINKS, 38 * LINKS, dtype=np.uint32)
    up = np.tile(np.array([0.0, 3.0, 0.0], np.float32), (LINKS, 1))
    for w in worlds:
        w.upload_bodies(ids, linvel=up)
        w.step(70)
    same_state(plain, reuse, full)
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
    same_state(plain, reuse, full)

    st_r, st_f, st_p = reuse.stats(), full.stats(), plain.stats()
    assert st_f["steps_reused"] == 0 and st_f["steps_rebuilt"] == st_f["steps"]
    assert st_p["steps_reused"] == 0 and st_p["steps_rebuilt"] == st_p["steps"]
    assert st_r["steps_rebuilt"] + st_r["steps_reused"] == st_r["steps"]
    for st in (st_r, st_f, st_p):
        assert st["error_flags"] == 0
    assert st_r["kernel_launches"] == st_f["kernel_launches"]          # a skipped rebuild counts its kernels all the same
