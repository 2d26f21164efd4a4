"""integrate(q, w, dt) (edyn_b200/csrc/b2d_math.cuh; the reference's math/quaternion.cpp:7-22) on the device, held to
an exact statement.  It is the one function whose device result may differ from the oracle's and the reference's: its
sinf / cosf are the device's, which may differ from glibc's.  Everything else in it is float32 arithmetic restated here
in numpy operation for operation (the library is built with -fmad=false):

    every component of the device's quaternion equals, bit for bit, the restatement evaluated with SOME s and c within
    +-2 ulps of the correctly rounded sin and cos of the float32 argument 0.5f * ws * dt

-- two ulps being CUDA's documented bound for sinf / cosf.  The correctly rounded values are float64 sin / cos of that
argument rounded to float32; 25 candidate (s, c) pairs per body.  The device integrates in two places and both are run:
k_integrate (bodies outside the island tiles) and k_island_tiles (hinge pairs in two-body tiles, no position iterations,
so the tile writes back the integrated pose unchanged).  tests/parity.py bit-checks everything else in a step against
the oracle; this pins the one difference it lets through.  Also runs against the CPU emulation (glibc's sinf is one of
the candidates)."""
import os

import numpy as np
import pytest

from tests import parity as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32
ULPS = 2                                  # CUDA's bound for sinf / cosf (CUDA C++ Programming Guide, single-precision functions)
DTS = (1.0 / 30, 1.0 / 60, 1.0 / 240)


def _nudge(x, k):
    """x moved k floats along the float32 line (negative: down)."""
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf) if k > 0 else f32(-np.inf)).astype(f32)
    return x


def restate(q, w, dt, s, c):
    """integrate(q, w, dt) of b2d_math.cuh in numpy float32 with the sine s and cosine c given (arrays over the bodies;
    s is not used on the Taylor branch): the length, the branch at 0.001f, the quaternion product r * q and normalize
    as four true divisions by sqrtf."""
    dt = f32(dt)
    x, y, z = w[:, 0], w[:, 1], w[:, 2]
    ws = np.sqrt((x * x + y * y) + z * z)
    k = f32(1.0) / f32(48.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(ws < f32(0.001), f32(0.5) * dt - dt * dt * dt * k * ws * ws, s / ws).astype(f32)
    rx, ry, rz, rw = x * t, y * t, z * t, c
    qx, qy, qz, qw = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    ox = rw * qx + rx * qw + ry * qz - rz * qy
    oy = rw * qy + ry * qw + rz * qx - rx * qz
    oz = rw * qz + rz * qw + rx * qy - ry * qx
    ow = rw * qw - rx * qx - ry * qy - rz * qz
    n = np.sqrt(ox * ox + oy * oy + oz * oz + ow * ow)
    return np.stack([ox / n, oy / n, oz / n, ow / n], axis=1).astype(f32)


def argument(w, dt):
    """0.5f * ws * dt in float32, as integrate() computes it."""
    x, y, z = w[:, 0], w[:, 1], w[:, 2]
    return f32(0.5) * np.sqrt((x * x + y * y) + z * z) * f32(dt)


def check_candidates(what, got, q, w, dt):
    """Every body's quaternion `got` equals the restatement with one of the 25 candidate (s, c) pairs, all four
    components bit for bit.  Returns the share of bodies the correctly rounded pair itself reproduces."""
    a = argument(w, dt).astype(np.float64)
    s0, c0 = np.sin(a).astype(f32), np.cos(a).astype(f32)
    hit = np.zeros(len(q), bool)
    for i in range(-ULPS, ULPS + 1):
        for j in range(-ULPS, ULPS + 1):
            want = restate(q, w, dt, _nudge(s0, i), _nudge(c0, j))
            same = (P._bits(want) == P._bits(got)).all(axis=1)
            if i == 0 and j == 0:
                rounded = same.mean()
            hit |= same
    bad = np.nonzero(~hit)[0]
    assert not len(bad), (f"{what}: {len(bad)} of {len(q)} bodies match no candidate; first body {bad[0]}: q {q[bad[0]]!r} w {w[bad[0]]!r} "
                          f"dt {dt!r} -> {got[bad[0]]!r}, correctly rounded sin / cos give {restate(q, w, dt, s0, c0)[bad[0]]!r}")
    return rounded


def random_unit_quaternions(rng, n):
    q = rng.normal(size=(n, 4)).astype(f32)
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f32)


def angular_velocities(rng, dt):
    """(w, kinematic): |w| log-uniform over 1e-6 .. 1e4 rad/s and arguments 0.5 |w| dt log-uniform over pi/4 .. 1e4 rad
    (where the device's range reduction takes its slow path), on random axes; |w| one float below, at and above 0.001f
    (the Taylor branch's threshold), on a coordinate axis so that float32 |w| is exactly that; zero; and a few kinematic
    bodies, which are not integrated at all."""
    def on_axes(ws):
        d = rng.normal(size=(len(ws), 3))
        return (d / np.linalg.norm(d, axis=1, keepdims=True) * ws[:, None]).astype(f32)
    sweep = on_axes(10.0 ** rng.uniform(-6, 4, 512))
    far = on_axes(2 * 10.0 ** rng.uniform(np.log10(np.pi / 4), 4, 256) / dt)
    edge = [_nudge(f32(0.001), k) for k in (-2, -1, 0, 1, 2)]
    thr = np.zeros((3 * len(edge), 3), f32)
    for i, v in enumerate(edge):
        for ax in range(3):
            thr[3 * i + ax, ax] = v * (1 if (i + ax) % 2 else -1)
    # the same magnitudes on random axes: float32 |w| lands a float or two around them
    thr_axes = on_axes(np.repeat(np.array(edge, np.float64), 4))
    w = np.concatenate([sweep, far, thr, thr_axes, np.zeros((4, 3), f32), on_axes(np.array([0.5, 3.0, 40.0, 1e-4]))])
    kinematic = np.zeros(len(w), bool)
    kinematic[-4:] = True
    return w, kinematic


def free_bodies(q, w, kinematic):
    """Shapeless bodies without gravity: no pair, no contact, no solve -- k_integrate alone moves them."""
    m = len(q)
    return dict(pos=np.zeros((m, 3), f32), orn=q, linvel=np.zeros((m, 3), f32), angvel=w,
                inv_mass=np.where(kinematic, 0, 1).astype(f32),
                inv_inertia=np.where(kinematic[:, None], 0, np.tile(np.eye(3, dtype=f32).reshape(9), (m, 1))).astype(f32),
                gravity=np.zeros((m, 3), f32), kind=np.where(kinematic, 1, 0).astype(np.uint32), shape_kind=np.full(m, 255, np.uint32),
                shape_params=np.zeros((m, 4), f32), friction=np.zeros(m, f32), restitution=np.zeros(m, f32), group=None, mask=None)


# dt = 1000 s: at a real step the Taylor branch agrees with the sine to well under an ulp near 0.001 rad/s, so neither
# the branch taken at the threshold nor the Taylor coefficient would show; at 1000 s they differ by hundreds of ulps
@pytest.mark.parametrize("dt", DTS + (1000.0,), ids=["dt30", "dt60", "dt240", "dt1000"])
def test_integrate_untiled_matches_candidate_restatement(gpu, E, dt):
    rng = np.random.default_rng(int(1 / dt))
    w, kin = angular_velocities(rng, dt)
    q = random_unit_quaternions(rng, len(w))
    assert (argument(w[:-8], dt).max() > 5e3) and (argument(w[:-8], dt) > np.pi / 4).sum() >= 256
    world = E.World(len(q), fixed_dt=dt)
    world.add_bodies(free_bodies(q, w, kin))
    world.step(1)
    g = world.download_state(aabb=False)
    world.close()
    assert np.array_equal(P._bits(g["angvel"]), P._bits(w)), "a free body's angular velocity changed"
    assert np.array_equal(P._bits(g["orn"][kin]), P._bits(q[kin])), "a kinematic body was integrated"
    rounded = check_candidates(f"k_integrate, dt {dt}", g["orn"][~kin], q[~kin], w[~kin], dt)
    # the threshold bodies on a coordinate axis: float32 |w| is exactly the float intended, both sides of 0.001f
    thr = w[768:783]
    ws = np.sqrt((thr[:, 0] * thr[:, 0] + thr[:, 1] * thr[:, 1]) + thr[:, 2] * thr[:, 2])
    assert np.array_equal(ws, np.repeat([_nudge(f32(0.001), k) for k in (-2, -1, 0, 1, 2)], 3))
    assert rounded > 0.5, rounded                  # most bodies take the correctly rounded values themselves


def hinge_pairs(rng, n, dt):
    """n gravity-free two-body hinge pairs, far apart, with random orientations, pivots, axes and angular velocities:
    each pair is a two-body island and goes to an island tile."""
    m = 2 * n
    pos = np.zeros((m, 3), f32)
    pos[:, 0] = np.repeat(np.arange(n) * 10.0, 2)
    pos[1::2, 1] = 1.0
    ws = np.concatenate([10.0 ** rng.uniform(-6, 4, m - 8), np.full(4, 0.001), np.zeros(4)])
    d = rng.normal(size=(m, 3))
    w = (d / np.linalg.norm(d, axis=1, keepdims=True) * ws[:, None]).astype(f32)
    b = free_bodies(random_unit_quaternions(rng, m), w, np.zeros(m, bool))
    b["pos"] = pos
    b["linvel"][:] = f32(-0.0)           # a hinge's linear rows add -0 to a velocity component: -0 stays -0 only if Δv starts at +0
    b["shape_kind"] = np.zeros(m, np.uint32)                   # spheres, far from each other: no contact
    b["shape_params"][:, 0] = 0.2
    b["friction"][:] = 0.5
    axis = rng.normal(size=(n, 3)).astype(f32)
    h = dict(a=np.arange(0, m, 2, dtype=np.uint32), b=np.arange(1, m, 2, dtype=np.uint32), pivot_a=np.tile([0, 0.5, 0], (n, 1)).astype(f32),
             pivot_b=np.tile([0, -0.5, 0], (n, 1)).astype(f32), axis_a=axis, axis_b=axis)
    return b, h


@pytest.mark.parametrize("dt", DTS, ids=["dt30", "dt60", "dt240"])
def test_integrate_tiled_matches_candidate_restatement(gpu, E, O, dt):
    """The tile kernel's integrate: the restatement from the pre-step orientation and the device's post-step angular
    velocity, which is first checked bit for bit against the oracle (with the linear velocities and hinge impulses)."""
    rng = np.random.default_rng(7 + int(1 / dt))
    b, h = hinge_pairs(rng, 256, dt)
    env = {**P.MODES["plain"]}
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        world = E.World(len(b["kind"]), max_hinges=len(h["a"]), fixed_dt=dt, velocity_iterations=8, position_iterations=0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    world.add_bodies(b)
    world.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    o = O.OracleWorld(dt=dt, vel_iters=8, pos_iters=0)
    o.add_bodies(b)
    o.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    world.step(1)
    P.oracle_step(O, o, world)
    g = world.download_state(aabb=False)
    want = o.state()
    for k in ("linvel", "angvel"):
        P.check_bits(0, k, g[k], want[k])
    P.check_hinge_impulses(0, world.hinge_impulses(), o.hinge_impulses())
    tiled = world.debug_tile_map()["btile"] != 0xFFFFFFFF
    assert world.stats()["error_flags"] == 0
    world.close()
    assert tiled.all(), f"{(~tiled).sum()} hinge bodies are not in an island tile"
    assert not np.array_equal(P._bits(g["angvel"]), P._bits(b["angvel"])), "the hinges did nothing"
    check_candidates(f"k_island_tiles, dt {dt}", g["orn"], b["orn"], g["angvel"], dt)


def test_integrate_reference_vectors_match_candidate_restatement(gpu, E):
    """tests/golden/body_math.npz (the reference's integrate through glibc) under the same rule, through one
    gravity-free, contact-free step per dt of the fixture."""
    bm = np.load(os.path.join(GOLD, "body_math.npz"))
    sel = np.where(bm["dt"] > 0)[0]
    for dt in np.unique(bm["dt"][sel]):
        s = sel[bm["dt"][sel] == dt]
        q, w = bm["q"][s], bm["w"][s]
        world = E.World(len(s), fixed_dt=float(dt))
        world.add_bodies(free_bodies(q, w, np.zeros(len(s), bool)))
        world.step(1)
        got = world.download_state(aabb=False)["orn"]
        world.close()
        check_candidates(f"reference vectors, dt {dt}", got, q, w, f32(dt))
        check_candidates(f"the reference itself, dt {dt}", bm["q_out"][s], q, w, f32(dt))
