"""Presentation transforms on the device (b2d_update_presentation / b2d_snap_presentation, k_presentation): held per call
to the device's own state, through both downloads, through the EnTT binding against the reference's stepper_sequential,
and across an island hand-over.

present_position = pos + linvel dt is float32 arithmetic (the library is built with -fmad=false), so it is checked bit for
bit against numpy; present_orientation = integrate(orn, angvel, dt) uses the device's sinf / cosf, so it is held to the
+-2-ulp candidate relation of tests/test_gpu_integrate.py."""
import threading

import numpy as np
import pytest

from tests import parity as P
from tests.golden import make_whole_step as G
from tests.test_gpu_integrate import check_candidates
from tests.test_stepper_b2d_presentation import FIXED_DT, build_harness, jittered, load_harness, run_sequence, sequences

pytestmark = pytest.mark.gpu
f32 = np.float32


def pile(E, sleeping=False):
    """A pile of boxes and spheres on a plane (sleeping: a box that falls asleep, woken by a second one landing on it) with
    presentation on the dynamic bodies, plus three kinematic bodies (one
    with presentation, as a caller of the C ABI may give it) and dynamic bodies without presentation."""
    scene = E.scenes.sleep_and_wake() if sleeping else E.scenes.mixed_pile(6, jitter=0.01)
    b = dict(scene["bodies"])
    n = len(b["kind"])
    b["presentation"] = (b["kind"] == 0).astype(np.uint32)
    b["presentation"][::7] = 0
    flags = E.world.FLAG_SLEEPING if sleeping else 0
    w = E.scenes.build_world(dict(scene, bodies=b), flags=flags, max_bodies=n + 3)
    kin = E.bodies_soa([E.RigidBodyDef(kind=E.KINEMATIC, position=(x, 9.0, 0.0), shape=E.sphere_shape(0.3),
                                       linvel=(0.5, 0.0, 0.0), angvel=(0.0, 1.0, 0.0)) for x in (-3.0, 0.0, 3.0)])
    kin["presentation"][:] = (1, 0, 1)
    w.add_bodies(kin)
    present = np.concatenate([b["presentation"], kin["presentation"]]).astype(bool)
    kind = np.concatenate([b["kind"], kin["kind"]])
    return w, present, kind


def expected(prev_p, prev_q, st, present, kind, asleep, dt):
    """(present_position wanted bit for bit, mask of bodies whose orientation is the candidate-checked integrate)."""
    upd = present & (kind == 0) & ~asleep
    want = prev_p.copy()
    want[upd] = st["pos"][upd] + st["linvel"][upd] * f32(dt)
    want[~present] = st["pos"][~present]
    return want, upd


@pytest.mark.parametrize("sleeping", [False, True])
def test_update_follows_the_state(gpu, E, sleeping):
    w, present, kind = pile(E, sleeping)
    p, q = w.presentation()
    st = w.download_state(aabb=False)
    assert np.array_equal(p, st["pos"]) and np.array_equal(q, st["orn"])     # def.position / def.orientation
    seen_asleep = 0
    for k, dt in enumerate([-FIXED_DT, -0.004, -1e-5, 0.0, 0.003, FIXED_DT] * 30):
        if k % 3 == 0:
            w.step(4)
        if k % 17 == 5:
            w.snap_presentation()
            p, q = w.presentation()
            st = w.download_state(aabb=False)
            assert np.array_equal(P._bits(p), P._bits(st["pos"])) and np.array_equal(P._bits(q), P._bits(st["orn"])), f"snap {k}"
        prev_p, prev_q = p, q
        w.update_presentation(dt)
        p, q = w.presentation()
        st = w.download_state(aabb=False)
        asleep = w.sleeping()
        seen_asleep += int(asleep.sum())
        want, upd = expected(prev_p, prev_q, st, present, kind, asleep, dt)
        assert np.array_equal(P._bits(p), P._bits(want)), f"call {k}: present_position"
        keep = present & ~upd
        assert np.array_equal(P._bits(q[keep]), P._bits(prev_q[keep])), f"call {k}: a sleeping / kinematic body's orientation moved"
        assert np.array_equal(P._bits(q[~present]), P._bits(st["orn"][~present])), f"call {k}: bodies without presentation"
        check_candidates(f"present_orientation, call {k}", q[upd], st["orn"][upd], st["angvel"][upd], dt)
    if sleeping:
        assert seen_asleep > 0, "nothing fell asleep"
    w.close()


def test_kind_patch_and_removal(gpu, E):
    """A body patched dynamic -> kinematic keeps its last present transform; a removed body reports its state."""
    w, present, kind = pile(E)
    w.step(10)
    w.update_presentation(-0.01)
    dyn = np.flatnonzero(present & (kind == 0))
    a, gone = int(dyn[0]), int(dyn[1])
    w.upload_bodies([a], kind=[E.KINEMATIC])
    p0, q0 = w.presentation()
    w.remove_bodies([gone])
    w.step(5)
    w.update_presentation(-0.01)
    p, q = w.presentation()
    st = w.download_state(aabb=False)
    assert np.array_equal(P._bits(p[a]), P._bits(p0[a])) and np.array_equal(P._bits(q[a]), P._bits(q0[a]))
    assert np.array_equal(P._bits(p[gone]), P._bits(st["pos"][gone])) and np.array_equal(P._bits(q[gone]), P._bits(st["orn"][gone]))
    w.close()


def test_device_download_equals_host_download(gpu, E):
    import torch
    w, _, _ = pile(E)
    n = w.num_bodies
    pos = torch.full((n, 3), float("nan"), dtype=torch.float32, device="cuda")
    orn = torch.full((n, 4), float("nan"), dtype=torch.float32, device="cuda")
    for k in range(6):
        w.step(3)
        w.update_presentation(-FIXED_DT * (k + 1) / 7)
        w.presentation_device(pos.data_ptr(), orn.data_ptr())
        w.sync()
        hp, hq = w.presentation()
        assert np.array_equal(P._bits(pos.cpu().numpy()), P._bits(hp)) and np.array_equal(P._bits(orn.cpu().numpy()), P._bits(hq))
    w.close()


def test_step_launches_unchanged_by_presentation(gpu, E):
    """No step kernel reads the presentation: the same scene with and without it launches the same kernels per step and
    computes the same state; each presentation call is one launch."""
    scene = E.scenes.mixed_pile(5, jitter=0.01)
    with_p = dict(scene["bodies"], presentation=(scene["bodies"]["kind"] == 0).astype(np.uint32))
    a = E.scenes.build_world(scene)
    b = E.scenes.build_world(dict(scene, bodies=with_p))
    for _ in range(3):
        l0, m0 = a.stats()["kernel_launches"], b.stats()["kernel_launches"]
        a.step(5); b.step(5)
        assert a.stats()["kernel_launches"] - l0 == b.stats()["kernel_launches"] - m0
        m1 = b.stats()["kernel_launches"]
        b.update_presentation(-0.01)
        assert b.stats()["kernel_launches"] - m1 == 1
    sa, sb = a.download_state(), b.download_state()
    for k in ("pos", "orn", "linvel", "angvel"):
        assert np.array_equal(P._bits(sa[k]), P._bits(sb[k])), k
    a.close(); b.close()


@pytest.fixture(scope="module")
def dev(gpu, O):
    build_harness()
    lib = load_harness(O, "dev")
    if lib is None:
        pytest.skip("tests/presentation/_build/libedyn_b2d_pres_dev.so not shipped (needs the reference at build time)")
    return lib


@pytest.mark.parametrize("seq", list(sequences()))
@pytest.mark.parametrize("name", ["boxes_27", "chains_16"])
def test_binding_on_device_presents_like_the_reference(dev, O, E, name, seq):
    """stepper_b2d over libb2d.so against stepper_sequential: the step counts exactly, present_position bit for bit against
    the reference's update_presentation on the device's state, present_orientation within tests/parity.py's trig
    tolerance (every orientation goes through the device's cosf)."""
    run_sequence(O, dev, G.build_scene(E, name), sequences()[seq], orn_tol=P.TRIG_TOL)


def test_binding_on_device_sleeping_and_mid_run_bodies(dev, O, E):
    scene = E.scenes.sleep_and_wake()
    ops = jittered(11, 120)
    ops = ops + [("update", ops[-1][1] + i / 60) for i in range(1, 420)]
    run_sequence(O, dev, scene, ops, sleeping=True, orn_tol=P.TRIG_TOL)
    extra = E.bodies_soa([E.RigidBodyDef(position=(float(x), 6.0, 0.5), shape=E.box_shape((0.2, 0.2, 0.2)),
                                         linvel=(0.0, 1.0, 0.0), angvel=(0.0, 0.5, 2.0)) for x in (-1, 0, 1)])
    t = [("update", i / 144) for i in range(1, 60)]
    ops = t + [("add", extra, True)] + [("update", 60 / 144 + i / 144) for i in range(40)] + [("add", extra, False)] + \
        [("update", 100 / 144 + i / 144) for i in range(60)]
    run_sequence(O, dev, G.build_scene(E, "boxes_27"), ops, orn_tol=P.TRIG_TOL)


def test_handover_keeps_present_transforms(gpu, E):
    """Two ranks as threads on one device: the stacks that meet move to rank 0, and every migrated body arrives with the
    flag and the exact present transform it had on rank 1."""
    import torch
    from edyn_b200 import dist
    scene = E.scenes.approaching_stacks(height=3, gap=0.6, speed=3.0)
    scene = dict(scene, bodies=dict(scene["bodies"], presentation=(scene["bodies"]["kind"] == 0).astype(np.uint32)))
    shared = dist.ThreadComm.Shared(2)
    sent, arrived, errs = {}, {}, []

    def body(rank):
        try:
            torch.cuda.set_device(0)
            sw = dist.DeviceShardedWorld(scene, rank, 2, dist.ThreadComm(shared, rank), device=0,
                                         labels=dist.initial_islands(scene), slack=1.0)
            w = sw.world
            pack, unpack = w.handover_pack, w.handover_unpack

            def pack_and_record(dst, ptr, cap):
                p, q = w.presentation()
                ent = w.entities()
                sent.update({int(e): (p[i].copy(), q[i].copy()) for i, e in enumerate(ent)})
                pack(dst, ptr, cap)

            def unpack_and_record(ptr, nbytes):
                n0 = w.num_bodies
                c = unpack(ptr, nbytes)
                p, q = w.presentation()
                ent = w.entities()
                arrived.update({int(ent[i]): (p[i].copy(), q[i].copy()) for i in range(n0, w.num_bodies)})
                return c

            w.handover_pack, w.handover_unpack = pack_and_record, unpack_and_record
            for k in range(60):
                sw.step(1)
                w.update_presentation(-FIXED_DT * (k % 5 + 1) / 6)
            sw.close()
        except BaseException as e:               # noqa: BLE001  (a dead rank must not leave its peer in the barrier)
            errs.append(e)
            shared.barrier.abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=300)
    assert not errs, errs
    assert len(arrived) == 3, sorted(arrived)
    for e, (p, q) in arrived.items():
        sp, sq = sent[e]
        assert np.array_equal(P._bits(p), P._bits(sp)) and np.array_equal(P._bits(q), P._bits(sq)), f"entity {e}"
    moved = [e for e, (p, _) in arrived.items() if not np.array_equal(p, scene["bodies"]["pos"][e])]
    assert moved, "the present transforms never left their initial values"


def test_python_update_and_pause(gpu, E):
    """edyn.update(world, elapsed): steps as before, then update_presentation with min(float32(acc - fixed_dt), fixed_dt);
    while paused only the snap; set_paused restarts the accumulator."""
    w = E.attach(64)
    ids = E.make_rigidbody(w, [E.RigidBodyDef(position=(float(i), 5.0, 0.0), shape=E.box_shape((0.2, 0.2, 0.2)),
                                              angvel=(0.0, 2.0, 0.5)) for i in range(4)])
    assert ids == 0
    fdt = f32(w.fixed_dt)
    acc, seen_zero = 0.0, 0
    for k, elapsed in enumerate([0.007] * 30 + [0.4] + [0.011] * 10):
        acc += elapsed
        n = int(acc / w.fixed_dt)
        acc -= n * w.fixed_dt
        assert E.update(w, elapsed) == min(n, w.max_steps_per_update)
        seen_zero += n == 0
        dt = min(f32(acc - float(fdt)), fdt)
        st = w.download_state(aabb=False)
        p, q = w.presentation()
        assert np.array_equal(P._bits(p), P._bits(st["pos"] + st["linvel"] * dt)), f"call {k}"
        check_candidates(f"python update {k}", q, st["orn"], st["angvel"], dt)
    assert seen_zero > 0
    E.set_paused(w, True)
    assert w._accum == 0.0 and E.update(w, 1.0) == 0
    st = w.download_state(aabb=False)
    p, q = w.presentation()
    assert np.array_equal(p, st["pos"]) and np.array_equal(q, st["orn"])
    E.set_paused(w, False)
    assert E.update(w, 0.02) == 1
    w.close()
