"""TEST INFRASTRUCTURE.  k_presentation (b2d_kernels.cuh) under the CPU emulation against the restatement of
update_presentation / snap_presentation (tests/presentation/ora_presentation.hpp), bit for bit: both sides call glibc's
sinf / cosf here.

    python tests/emu/presentation.py          -> one JSON line
Runs in its own process because B2D_LIB has to be set before edyn_b200 is imported."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    from tests.emu import build as B
    os.environ["B2D_LIB"] = B.build()
    import edyn_b200 as E
    from tests.test_stepper_b2d_presentation import ora_presentation, restatement
    lib = restatement()
    scene = E.scenes.mixed_pile(4, jitter=0.01)
    b = dict(scene["bodies"])
    b["presentation"] = (b["kind"] == 0).astype(np.uint32)
    b["presentation"][::5] = 0
    kin = E.bodies_soa([E.RigidBodyDef(kind=E.KINEMATIC, position=(x, 7.0, 0.0), shape=E.sphere_shape(0.3),
                                       linvel=(0.5, 0.0, 0.0), angvel=(0.0, 1e-4, 0.0)) for x in (-2.0, 2.0)])
    kin["presentation"][:] = 1
    w = E.scenes.build_world(dict(scene, bodies=b), max_bodies=len(b["kind"]) + 2)
    w.add_bodies(kin)
    kind = np.concatenate([b["kind"], kin["kind"]]).astype(np.uint32)
    present = np.concatenate([b["presentation"], kin["presentation"]]).astype(np.uint32)
    asleep = np.zeros(len(kind), np.uint32)
    st = w.download_state(aabb=False)
    op, oq = st["pos"].copy(), st["orn"].copy()          # def.position / def.orientation
    calls = mismatched = 0
    for k, dt in enumerate([-1.0 / 60, -0.004, -1e-5, 0.0, 0.003, 1.0 / 60] * 8):
        if k % 3 == 0:
            w.step(3)
        st = w.download_state(aabb=False)
        snap = k % 11 == 4
        if snap:
            w.snap_presentation()
        else:
            w.update_presentation(dt)
        ora_presentation(lib, snap, dt, st, kind, asleep, present, op, oq)
        op[present == 0], oq[present == 0] = st["pos"][present == 0], st["orn"][present == 0]     # reported as pos / orn
        gp, gq = w.presentation()
        calls += 1
        mismatched += int(not (np.array_equal(gp.view(np.uint32), op.view(np.uint32)) and
                               np.array_equal(gq.view(np.uint32), oq.view(np.uint32))))
    w.close()
    print(json.dumps(dict(calls=calls, mismatched=mismatched, bodies=int(len(gp)))))


if __name__ == "__main__":
    main()
