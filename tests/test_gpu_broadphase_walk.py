"""The broadphase's neighbourhood search reads cell-ordered candidate records, with a thread per query body walking
columns of three cells (B2D_BP_WARP_MAX=0, what a million bodies run) and with a warp per query body, one lane per cell
(what small worlds run).  Both mappings
must find the same pairs in the same order, and so give the same manifold slots and the same state: every step the
ordered pair set is checked against the oracle (tests/emu/lockstep.py), and the two runs are compared bit for bit:
World.contacts() pairs in slot order, the island tiles' pairs (debug_tile_map) and the state.

Scenes: the four benchmark scenes at reduced size, large dynamic and static bodies, collision filters and exclusions,
and a row of spheres across the edge of the cell-key range, where cell_key_of clamps z.  There two or three of a body's
z offsets share one key; the search walks that cell once, so no pair gets a second manifold, in any scene
(tests/test_gpu_broadphase_edges.py covers the other clamped placements).
Also runs against the CPU emulation (B2D_EMU=1: smaller scenes, fewer steps)."""
import os

import numpy as np
import pytest

from tests import large_scenes as L
from tests.emu.lockstep import lockstep

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
STEPS = 20 if EMU else 60
SEARCH = {"warp": {"B2D_BP_WARP_MAX": str(1 << 30)}, "thread": {"B2D_BP_WARP_MAX": "0"}}


def clamped_row(E):
    """Spheres in a row along z across cell z = 32767, the last cell of the default 16-bit key field (the static sphere
    80 000 cells away keeps the measured extent from covering them), resting on a plane."""
    R = E.rigidbody
    cell = 0.5 + 2 * 0.02 + 1e-3                          # largest diameter + 2 x breaking threshold + 1e-3
    z0 = 32767 * cell
    defs = [R.RigidBodyDef(kind=R.STATIC, shape=R.plane_shape((0, 1, 0), 0.0)),
            R.RigidBodyDef(kind=R.STATIC, position=(0, 0.25, 0), shape=R.sphere_shape(0.25)),
            R.RigidBodyDef(kind=R.STATIC, position=(0, 0.25, 80000 * cell), shape=R.sphere_shape(0.25))]
    for i in range(24):
        defs.append(R.RigidBodyDef(position=(0.1 * (i % 2), 0.26, z0 + 0.49 * (i - 12)), shape=R.sphere_shape(0.25)))
    return dict(name="clamped_row", bodies=R.bodies_soa(defs), hinges=None, exclusions=None, dynamic=24,
                settings=dict(velocity_iterations=10, position_iterations=3))


def make(E, O, name):
    S = E.scenes
    if name == "boxes":
        return S.boxes_on_plane(3 if EMU else 8)
    if name == "spheres":
        return S.spheres_in_box(3, 4, 3) if EMU else S.spheres_in_box(16, 8, 16)
    if name == "mixed":
        return S.mixed_pile(4 if EMU else 12)
    if name == "chains":
        return S.hinge_chains(2, 2) if EMU else S.hinge_chains(16, 16)
    if name == "large":
        return L.SCENES["plank_boxes"](E)
    if name == "filters":
        from tests.test_ref_stepper import random_scene
        return random_scene(E, O, 7)
    return clamped_row(E)


class Recorder:
    def __init__(self):
        self.contacts, self.tiles, self.dups = [], [], 0

    def __call__(self, step, w):
        c = w.contacts()
        self.contacts.append(np.ascontiguousarray(c["pairs"]).tobytes())
        self.tiles.append(np.ascontiguousarray(w.debug_tile_map()["pairs"]).tobytes())
        p = [tuple(sorted(q)) for q in c["pairs"].tolist()]
        self.dups = max(self.dups, len(p) - len(set(p)))


@pytest.mark.parametrize("name", ["boxes", "spheres", "mixed", "chains", "large", "filters", "clamped_row"])
def test_column_walk_thread_and_warp(E, O, name):
    scene = make(E, O, name)
    if name == "filters":
        assert scene["exclusions"] is not None and np.any(np.asarray(scene["bodies"]["mask"]) != np.uint64(0xFFFFFFFFFFFFFFFF))
    out = {}
    for s, env in SEARCH.items():
        rec = Recorder()
        res = lockstep(E, O, scene, STEPS, mode="plain", hook=rec, env=env)
        assert res["ok"], (s, res)
        out[s] = (res, rec)
    (rw, cw), (rt, ct) = out["warp"], out["thread"]
    assert rw["digests"] == rt["digests"]
    assert cw.contacts == ct.contacts
    assert cw.tiles == ct.tiles
    assert sum(len(x) for x in cw.contacts) > 0
    assert cw.dups == 0 and ct.dups == 0
