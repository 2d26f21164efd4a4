"""The EnTT binding (edyn_b200/csrc/host/stepper_b2d.hpp) with sensors and the material mixing table on the device: its
harness (tests/materials/binding_materials.cpp) linked with edyn_b200/libb2d.so.  A real Edyn registry whose bodies carry
material ids or no material, with material_mix_table entries inserted, overwritten and removed between steps, steps bit
for bit as edyn_b200.World fed the same arrays and table through the C ABI directly; mirrored sensor points carry no
contact_point_material and no contact_point_impulse."""
import numpy as np
import pytest

from tests import material_oracle as M
from tests.test_gpu_materials import FLOOR, NONE, RUBBER, STONE, TABLE, _scene
from tests.test_stepper_b2d_materials import binding_world, check_mirrored_points

pytestmark = pytest.mark.gpu
EDITS = {10: [(RUBBER, FLOOR, 0.2, 0.9)], 20: [(FLOOR, RUBBER)], 30: [(STONE, STONE, 1.0, 0.5)]}


def _apply(targets, entries):
    ins = [e for e in entries if len(e) == 4]
    rem = [e for e in entries if len(e) == 2]
    for t in targets:
        if ins:
            a, b, f, r = (np.array(c) for c in zip(*ins))
            t.set_material_mixing(a, b, f, r)
        if rem:
            a, b = (np.array(c) for c in zip(*rem))
            t.remove_material_mixing(a, b)


@pytest.mark.parametrize("shape", ["box", "sphere"])
def test_binding_follows_the_abi_on_the_device(gpu, E, O, shape):
    lib = M.library(O, "binding_materials_dev")
    if lib is None:
        pytest.skip("tests/materials/_build/libbinding_materials_dev.so not available (needs /root/reference at build time)")
    scene, _ = _scene(E, shape, 3)
    sensor = np.asarray(scene["bodies"]["material"]) == NONE
    n = len(scene["bodies"]["kind"])
    w, wm = binding_world(O, lib, scene, max_manifolds=1 << 16)
    d = E.scenes.build_world(scene, max_manifolds=1 << 16, max_bodies=n + 8, max_hinges=1)      # the binding's capacities
    moving = np.asarray(scene["bodies"]["kind"]) != 2        # static bodies keep the AABB make_rigidbody gave them
    _apply([wm, d], TABLE)
    seen = 0
    for s in range(45):
        if s in EDITS:
            _apply([wm, d], EDITS[s])
        w.step(1)
        d.step(1)
        a, b = w.state(), d.download_state(aabb=True)
        for k in ("pos", "orn", "linvel", "angvel"):
            assert np.array_equal(a[k], b[k][:n]), f"step {s}: {k}"
        assert np.array_equal(a["aabb"][moving], b["aabb"][:n][moving]), f"step {s}: AABBs"
        if s % 5 == 4:
            w.mirror_contacts()
            seen += check_mirrored_points(wm.contacts(), sensor, True)
    assert seen > 0
    assert d.stats()["error_flags"] == 0
    w.close()
