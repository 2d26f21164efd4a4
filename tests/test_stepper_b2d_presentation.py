"""Presentation transforms through the EnTT binding: edyn::update(registry, time) with present_position /
present_orientation on the dynamic bodies (rigidbody_def::presentation, the reference's default), run by the reference's
own stepper_sequential and by edyn::stepper_b2d on two registries built by the same code.

After every update() call:
  * both ran the same number of fixed steps (the accumulator, floor, max_steps_per_update and pause rules of
    stepper_sequential.cpp:28-69, :148-151);
  * on each side, every present transform is what the reference's own update_presentation / snap_presentation
    (sys/update_presentation.cpp:56-93, called on that side's state) gives for the interpolation_dt of
    stepper_sequential.cpp:104-105, computed here in double as the reference computes it -- bit for bit;
  * bodies whose state is bitwise equal on the two sides have bitwise equal present transforms.
Each side is held to its own state because the two steppers order contact rows differently once bodies touch.

CPU suite: the binding's C ABI is answered by tests/presentation/b2d_mock_presentation.cpp (the oracle's mock with the
restatement of the two presentation functions, tests/presentation/ora_presentation.hpp).  tests/test_gpu_presentation.py
runs the same sequences with the binding on the device."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from tests.golden import make_whole_step as G
from tests.test_stepper_b2d import EdynB2dWorld

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "presentation", "_build")
_f, _u = np.float32, C.c_uint32
FIXED_DT = float(np.float32(1.0 / 60))        # settings.fixed_dt is a float; the accumulator works in double
MAX_STEPS = 10                                 # settings.max_steps_per_update


def build_harness():
    """(Re)build tests/presentation where the reference is present; elsewhere the shipped libraries are used as they are."""
    if os.path.isdir("/root/reference/include/edyn") and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "edyn_obj")):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "presentation")], check=True)


def load_harness(O, variant):
    """tests/presentation/_build/libedyn_b2d_pres_{mock,dev}.so with its signatures, or None where it was not shipped."""
    path = os.path.join(BUILD, f"libedyn_b2d_pres_{variant}.so")
    if not os.path.exists(path):
        return None
    lib = O.load_refs_library(path)
    lib.eb2d_world.restype = C.c_void_p
    lib.eb2d_body_id.restype = C.c_uint32
    return declare(lib)


def restatement():
    """tests/presentation/_build/liborapres.so (built on demand: g++ only)."""
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "presentation"), "restatement"], check=True)
    lib = C.CDLL(os.path.join(BUILD, "liborapres.so"))
    lib.orap_presentation.argtypes = [C.c_uint32, C.c_int, C.c_float] + [C.c_void_p] * 9
    return lib


def ora_presentation(lib, snap, dt, st, kind, asleep, present, ppos, porn):
    """The restatement on packed arrays: ppos / porn are updated in place (bodies it does not write keep theirs)."""
    a = [np.ascontiguousarray(st[k], _f) for k in ("pos", "orn", "linvel", "angvel")]
    f = [np.ascontiguousarray(x, np.uint32) for x in (kind, asleep, present)]
    assert ppos.flags.c_contiguous and porn.flags.c_contiguous and ppos.dtype == _f and porn.dtype == _f
    lib.orap_presentation(_u(len(kind)), int(snap), C.c_float(dt), *[x.ctypes.data_as(C.c_void_p) for x in a + f + [ppos, porn]])


def declare(lib):
    for name in ("eb2d_ref_update", "eb2d_ref_step_simulation", "eb2d_step_simulation", "eb2d_update"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_double]
    lib.eb2d_count_steps.restype = C.c_uint64
    lib.eb2d_ref_presentation.argtypes = [C.c_uint32, C.c_int, C.c_float] + [C.c_void_p] * 9
    return lib


def ref_presentation(lib, snap, dt, st, kind, asleep, present):
    """The reference's update_presentation (snap=False, interpolation_dt = dt) or snap_presentation on the given state."""
    n = len(kind)
    a = [np.ascontiguousarray(st[k], _f) for k in ("pos", "orn", "linvel", "angvel")]
    f = [np.ascontiguousarray(x, np.uint32) for x in (kind, asleep, present)]
    pos, orn = np.zeros((n, 3), _f), np.zeros((n, 4), _f)
    lib.eb2d_ref_presentation(_u(n), int(snap), C.c_float(dt), *[x.ctypes.data_as(C.c_void_p) for x in a + f + [pos, orn]])
    return pos, orn


class Clock:
    """stepper_sequential's time keeping (stepper_sequential.cpp:28-69, :104-105, :148-151) in double precision."""

    def __init__(self):
        self.last, self.acc, self.paused = 0.0, 0.0, False

    def update(self, t):
        """-> (steps, interpolation_dt), or (0, None) while paused (snap)."""
        if self.paused:
            return 0, None
        elapsed = max(t - self.last, 0.0)
        self.acc += elapsed
        n = math.floor(self.acc / FIXED_DT)
        self.acc -= float(n) * FIXED_DT
        self.last = t
        sim_time = self.last - self.acc
        return min(n, MAX_STEPS), min(_f(t - FIXED_DT - sim_time), _f(FIXED_DT))

    def step_simulation(self, t):
        self.last = t

    def set_paused(self, p):
        self.paused, self.acc = p, 0.0


class Side:
    """One registry with presentation on its dynamic bodies, stepped by the reference (ref=True) or by stepper_b2d."""

    def __init__(self, O, lib, scene, ref, sleeping):
        self.lib, self.ref = lib, ref
        self.w = EdynB2dWorld(O, lib, scene, sleeping=sleeping) if not ref else None
        if ref:
            st = scene["settings"]
            self.r = O.RefWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"], library=lib)
            if sleeping:
                self.r.add_bodies(scene["bodies"], sleeping_disabled=False)
            else:
                G.populate(self.r, scene)
            lib.eb2d_ref_set_paused(self.r.h, 0)
        else:
            self.r = self.w.r
        self.kind = np.asarray(scene["bodies"]["kind"], np.uint32).copy()
        self.present = np.zeros(len(self.kind), np.uint32)
        self.give_presentation(np.flatnonzero(self.kind == 0))
        lib.eb2d_count_steps(self.r.h)
        self.pre = self.presentation()[:2]

    def give_presentation(self, ids):
        for i in ids:
            self.lib.eb2d_add_presentation(self.r.h, _u(int(i)))
            self.present[i] = 1

    def add_bodies(self, soa, present, sleeping):
        first = self.r.num_bodies
        self.r.add_bodies(soa, sleeping_disabled=not sleeping)
        self.kind = np.concatenate([self.kind, np.asarray(soa["kind"], np.uint32)])
        self.present = np.concatenate([self.present, np.zeros(len(soa["kind"]), np.uint32)])
        if present:
            self.give_presentation(first + np.flatnonzero(np.asarray(soa["kind"]) == 0))
        n = self.r.num_bodies
        p, q = self.pre
        self.pre = (np.concatenate([p, np.zeros((n - len(p), 3), _f)]), np.concatenate([q, np.zeros((n - len(q), 4), _f)]))

    def update(self, t):
        if self.ref:
            self.lib.eb2d_ref_update(self.r.h, t)
        else:
            assert self.lib.eb2d_update(self.r.h, t) == 0

    def step_simulation(self, t):
        if self.ref:
            self.lib.eb2d_ref_step_simulation(self.r.h, t)
        else:
            assert self.lib.eb2d_step_simulation(self.r.h, t) == 0

    def set_paused(self, p):
        if self.ref:
            self.lib.eb2d_ref_set_paused(self.r.h, int(p))
        else:
            self.lib.eb2d_set_paused(self.r.h, int(p))

    def steps(self):
        return int(self.lib.eb2d_count_steps(self.r.h))

    def presentation(self):
        n = self.r.num_bodies
        pos, orn, has = np.zeros((n, 3), _f), np.zeros((n, 4), _f), np.zeros(n, np.uint32)
        self.lib.eb2d_get_presentation(self.r.h, pos.ctypes.data_as(C.c_void_p), orn.ctypes.data_as(C.c_void_p),
                                       has.ctypes.data_as(C.c_void_p))
        return pos, orn, has

    def check(self, dt, what, orn_tol=0.0):
        """The present transforms against the reference's functions on this side's own state; returns the state.
        orn_tol: allowed difference of present_orientation (the device's sinf / cosf are not glibc's)."""
        st = self.r.state()
        pos, orn, has = self.presentation()
        assert np.array_equal(has, self.present), f"{what}: which bodies have presentation"
        asleep = self.r.sleeping().astype(np.uint32)
        if dt is None:
            want_p, want_q = ref_presentation(self.lib, True, 0.0, st, self.kind, asleep, self.present)
        else:
            want_p, want_q = ref_presentation(self.lib, False, dt, st, self.kind, asleep, self.present)
            kept = (self.present == 1) & ((self.kind != 0) | (asleep == 1))    # not in the linear / angular views
            want_p[kept], want_q[kept] = self.pre[0][kept], self.pre[1][kept]
        m = self.present == 1
        side = "reference" if self.ref else "stepper_b2d"
        for got, want, k, tol in ((pos, want_p, "present_position", 0.0), (orn, want_q, "present_orientation", orn_tol)):
            bad = np.flatnonzero(m & ~np.all(np.abs(got - want) <= tol, axis=1))
            assert not len(bad), f"{what}: {side} {k} of bodies {bad[:8].tolist()}: {got[bad[0]]} != {want[bad[0]]}"
        self.pre = (pos, orn)
        return st

    def close(self):
        if self.w is not None:
            self.w.close()


def run_sequence(O, lib, scene, ops, sleeping=False, orn_tol=0.0):
    """ops: ("update", t) | ("step", t) | ("pause", bool) | ("add", soa, present).  Both sides follow them; everything in
    the module docstring is checked after every update.  Returns (updates, updates that ran no step, total steps)."""
    ref, dev = Side(O, lib, scene, True, sleeping), Side(O, lib, scene, False, sleeping)
    clock = Clock()
    nupd = nzero = 0
    for k, op in enumerate(ops):
        if op[0] == "pause":
            clock.set_paused(op[1]); ref.set_paused(op[1]); dev.set_paused(op[1])
        elif op[0] == "step":
            clock.step_simulation(op[1]); ref.step_simulation(op[1]); dev.step_simulation(op[1])
        elif op[0] == "add":
            ref.add_bodies(op[1], op[2], sleeping); dev.add_bodies(op[1], op[2], sleeping)
        else:
            s0 = ref.steps()
            n, dt = clock.update(op[1])
            ref.update(op[1]); dev.update(op[1])
            what = f"op {k} update({op[1]!r})"
            assert ref.steps() - s0 == n, f"{what}: the reference ran {ref.steps() - s0} steps, the clock says {n}"
            assert dev.steps() == ref.steps(), f"{what}: stepper_b2d has run {dev.steps()} steps, the reference {ref.steps()}"
            a, b = ref.check(dt, what), dev.check(dt, what, orn_tol)
            same = np.ones(len(ref.kind), bool)
            for key in ("pos", "orn", "linvel", "angvel"):
                same &= np.all(a[key] == b[key], axis=1)
            same &= ref.r.sleeping() == dev.r.sleeping()
            assert np.array_equal(ref.pre[0][same], dev.pre[0][same]), f"{what}: equal states, different present_position"
            assert np.all(np.abs(ref.pre[1][same] - dev.pre[1][same]) <= orn_tol), f"{what}: equal states, different present_orientation"
            nupd += 1
            nzero += n == 0
    total = ref.steps()
    ref.close(); dev.close()
    return nupd, nzero, total


def frames(hz, seconds, t0=0.0):
    return [("update", t0 + i / hz) for i in range(1, int(seconds * hz) + 1)]


def jittered(seed, n, t0=0.0):
    rng = np.random.default_rng(seed)
    t, out = t0, []
    for _ in range(n):
        t += float(rng.choice([0.0, rng.uniform(0, 0.004), rng.uniform(0.004, 0.03), rng.uniform(0.03, 0.06)]))
        out.append(("update", t))
    return out


def sequences():
    """name -> ops (the scenes' bodies are created at time 0)."""
    return {
        "144hz": frames(144, 1.5),
        "30hz": frames(30, 2.0),
        "jitter": jittered(7, 240),
        "gap": frames(60, 0.3) + [("update", 0.3 + 12 * FIXED_DT + 0.005)] + frames(60, 0.3, 0.3 + 12 * FIXED_DT + 0.005),
        "pause": frames(90, 0.5) + [("pause", True), ("update", 0.52), ("step", 0.53), ("update", 0.55), ("step", 0.56),
                                    ("update", 0.9), ("pause", False)] + frames(90, 0.6, 0.9),
    }


@pytest.fixture(scope="module")
def mock(O):
    if O.ref_stepper() is None:
        pytest.skip("needs the reference's objects (oracle/_ref)")
    build_harness()
    lib = load_harness(O, "mock")
    if lib is None:
        pytest.skip("tests/presentation/_build/libedyn_b2d_pres_mock.so not available")
    return lib


@pytest.mark.parametrize("seq", list(sequences()))
@pytest.mark.parametrize("name", ["boxes_27", "chains_16"])
def test_update_presents_like_the_reference(mock, O, E, name, seq):
    ops = sequences()[seq]
    nupd, nzero, total = run_sequence(O, mock, G.build_scene(E, name), ops)
    assert nupd == sum(op[0] == "update" for op in ops) and total > 0
    if seq in ("144hz", "jitter"):
        assert nzero > 0                                # frames between two steps: presentation alone


@pytest.mark.parametrize("seq", ["144hz", "jitter"])
def test_update_presents_sleeping_bodies_like_the_reference(mock, O, E, seq):
    """Island sleeping on: the box falls asleep (its present transform stays), the second box lands on it and wakes it."""
    scene = E.scenes.sleep_and_wake()
    ops = sequences()[seq]
    ops = ops + [("update", ops[-1][1] + i / 60) for i in range(1, 420)]       # long enough to sleep, wake, sleep
    run_sequence(O, mock, scene, ops, sleeping=True)


def test_bodies_created_mid_run(mock, O, E):
    """Bodies made between two update() calls, with presentation (interpolated from the next call on, even before their
    first step) and without it (no components, never written)."""
    scene = G.build_scene(E, "boxes_27")
    extra = E.bodies_soa([E.RigidBodyDef(position=(float(x), 6.0, 0.5), shape=E.box_shape((0.2, 0.2, 0.2)),
                                         linvel=(0.0, 1.0, 0.0), angvel=(0.0, 0.5, 2.0)) for x in (-1, 0, 1)])
    ops = frames(144, 0.4) + [("add", extra, True)] + frames(144, 0.3, 0.4) + [("add", extra, False)] + frames(144, 0.5, 0.7)
    run_sequence(O, mock, scene, ops)


def test_restatement_equals_the_reference(mock, O, E):
    """tests/presentation/ora_presentation.hpp's update_presentation / snap_presentation == the reference's, bit for bit, on
    random states: |w| on both sides of the 0.001 branch of integrate, negative and positive dt, sleeping, kinematic and
    static bodies, bodies with and without presentation."""
    lib = restatement()
    rng = np.random.default_rng(3)
    n = 400
    kind = rng.choice([0, 0, 0, 1, 2], n).astype(np.uint32)
    q = rng.normal(size=(n, 4))
    axis = rng.normal(size=(n, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    speed = np.exp(rng.uniform(np.log(1e-5), np.log(50), n))            # 1e-5 .. 50 rad/s: both branches
    speed[:8] = [0.0, 0.000999, 0.001, 0.0010001, 1e-9, 3.0, 0.0005, 0.002]
    st = dict(pos=rng.uniform(-50, 50, (n, 3)).astype(_f), orn=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(_f),
              linvel=rng.normal(0, 5, (n, 3)).astype(_f), angvel=(axis * speed[:, None]).astype(_f))
    st["linvel"][kind == 2] = 0
    st["angvel"][kind == 2] = 0
    asleep = (rng.uniform(size=n) < 0.2).astype(np.uint32)
    present = rng.choice([0, 1, 1, 1], n).astype(np.uint32)
    m = present == 1
    upd = m & (kind == 0) & (asleep == 0)
    for dt in (-FIXED_DT, -0.0123, -1e-4, 0.0, 1e-4, 0.007, FIXED_DT):
        for snap in (False, True):
            m = (present == 1) if snap else upd        # update: the others keep what they had (both sides start differently)
            ppos, porn = np.zeros((n, 3), _f), np.zeros((n, 4), _f)
            ora_presentation(lib, snap, dt, st, kind, asleep, present, ppos, porn)
            if not snap:
                assert not ppos[~upd].any() and not porn[~upd].any(), f"dt {dt}: a body outside the views was written"
            want_p, want_q = ref_presentation(mock, snap, dt, st, kind, asleep, present)
            assert np.array_equal(ppos[m].view(np.uint32), want_p[m].view(np.uint32)), f"dt {dt} snap {snap}: position"
            assert np.array_equal(porn[m].view(np.uint32), want_q[m].view(np.uint32)), f"dt {dt} snap {snap}: orientation"
    assert upd.sum() > 100 and ((present == 1) & ~upd).sum() > 50
