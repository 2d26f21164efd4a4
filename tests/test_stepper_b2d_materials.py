"""The EnTT binding (edyn_b200/csrc/host/stepper_b2d.hpp) with sensors and the material mixing table, on the CPU: its
harness (tests/materials/binding_materials.cpp) linked with the C ABI mock (tests/integration/b2d_mock.cpp).

  * After mirror_contacts(), a sensor's points carry contact_point, contact_point_list and contact_point_geometry only, as
    the reference's own narrowphase leaves them (collision_util.cpp:358-384; compared with the real stepper's registry),
    the other points also contact_point_material and contact_point_impulse, and a user's contact_started_tag listener
    sees every new point, sensor or not.
  * Unsupported changes throw: a body gaining or losing its material, a table entry with a contact extra, any table entry
    when the linked library lacks the mixing entry points (the mock); destroying a body (which takes its material along)
    does not.
The mock answers the ABI with the oracle, which has no materials: that the binding stages sensors, ids and the table as
the arrays handed to the ABI directly is checked on the device (tests/test_gpu_binding_materials.py)."""
import ctypes as C

import numpy as np
import pytest

from tests import material_oracle as M
from tests.test_gpu_materials import FLOOR, NONE, RUBBER, TABLE, _scene
from tests.test_stepper_b2d import EdynB2dWorld

_u = C.c_uint32


def binding_world(O, lib, scene, max_manifolds=1 << 16):
    """A real Edyn registry holding `scene` with its materials (sensors have no material component), stepped by
    edyn::stepper_b2d: (EdynB2dWorld, RefMaterials)."""
    st = scene["settings"]
    w = EdynB2dWorld.__new__(EdynB2dWorld)
    w.lib, w.sleeping = lib, False
    w.r = O.RefWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"], library=lib)
    rm = M.RefMaterials(lib, w.r)
    rm.populate(scene)
    w._attach(len(scene["bodies"]["kind"]), max_manifolds, len(scene["hinges"]["a"]) if scene["hinges"] else 0)
    return w, rm


def set_table(rm, table):
    a, b, f, r = (np.array(c) for c in zip(*table))
    rm.set_material_mixing(a, b, f, r)


@pytest.fixture(scope="module")
def lib(O):
    if O.ref_stepper() is None:
        pytest.skip("needs the reference's objects (oracle/_ref)")
    M.build()
    lib = M.library(O, "binding_materials_mock")
    if lib is None:
        pytest.skip("tests/materials/_build/libbinding_materials_mock.so not available")
    for name in ("eb2d_world", "eb2d_body_id"):
        getattr(lib, name).restype = C.c_void_p if name == "eb2d_world" else C.c_uint32
    return lib


def check_mirrored_points(c, sensor, mirrored):
    """c: RefMaterials.contacts() of a registry.  Returns the sensor points seen."""
    seen = 0
    for k, (a, b) in enumerate(c["pairs"].tolist()):
        nm = int(c["num"][k])
        pts = c["mat"][k, :nm]
        if sensor[a] or sensor[b]:
            # no contact_point_material (friction, restitution read as 0), no contact_point_impulse, no contact_constraint
            assert not pts.any(), (mirrored, (a, b), pts)
            seen += nm
        else:
            assert np.all(pts[:, 3] == 1), (mirrored, (a, b))
            assert np.all(pts[:, 2] == (0 if mirrored else 1))              # the binding does not mirror constraints
    return seen


def test_mirrored_sensor_points_match_the_reference(O, lib, E):
    refm = M.library(O, "ref_materials")
    scene, n = _scene(E, "box", 3)
    sensor = np.asarray(scene["bodies"]["material"]) == NONE
    w, wm = binding_world(O, lib, scene)               # no table here: the mock has no mixing entry points (the binding refuses)
    r = O.RefWorld(vel_iters=scene["settings"]["velocity_iterations"], pos_iters=scene["settings"]["position_iterations"],
                   library=refm)
    rm = M.RefMaterials(refm, r)
    rm.populate(scene)
    set_table(rm, TABLE)
    seen = [0, 0]
    for step in range(40):
        w.step(1)
        r.step(1)
        (_, points, created, _), (started, _) = w.mirror_contacts()
        c = wm.contacts()
        seen[0] += check_mirrored_points(c, sensor, True)
        seen[1] += check_mirrored_points(rm.contacts(), sensor, False)
        assert points == int(c["num"].sum())
        assert started >= created
    assert seen[0] > 0 and seen[1] > 0
    w.close()


def test_unsupported_material_changes_throw(O, lib, E):
    scene, n = _scene(E, "box", 2)
    w, _ = binding_world(O, lib, scene)
    w.step(2)
    lib.refm_toggle_material(w.r.h, _u(0), C.c_int(0))          # a body with a material loses it
    assert lib.eb2d_step(w.r.h, _u(1)) != 0
    w.close()
    w, _ = binding_world(O, lib, scene)
    w.step(2)
    lib.refm_toggle_material(w.r.h, _u(n), C.c_int(1))          # a sensor gains one
    assert lib.eb2d_step(w.r.h, _u(1)) != 0
    w.close()
    w, _ = binding_world(O, lib, scene)
    lib.refm_insert_spin_mixing(w.r.h, _u(RUBBER), _u(FLOOR), C.c_float(0.1))
    assert lib.eb2d_step(w.r.h, _u(1)) != 0
    w.close()
    w, wm = binding_world(O, lib, scene)                        # a table entry, but a libb2d without the mixing entry points
    set_table(wm, TABLE)
    assert lib.eb2d_step(w.r.h, _u(1)) != 0
    w.close()
    w, _ = binding_world(O, lib, scene)                         # destroying a body takes its material along: no toggle
    w.step(2)
    w.destroy_body(0)
    w.destroy_body(n)
    w.step(2)
    w.close()
