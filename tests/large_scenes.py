"""TEST INFRASTRUCTURE.  Scenes with LARGE DYNAMIC bodies: bodies the broadphase keeps in its brute-force list instead of
the cell grid because their bounding diameter is more than 4 x the mean dynamic diameter (b2d_api.cu reclassify).  A
plank, a crate among marbles, a log under falling spheres.  Each scene isolates one path such a body takes: its
manifold with a static / kinematic partner (filed under the large body, in the large body's tile), manifolds between
two large dynamic bodies (found from the brute-force side only), a manifold of a two-point island growing past 2
points, one body at the 64-colour and the restitution-group limits, and the classification flipping between steps.

`large_dynamic(bodies)` restates the host's rule; every scene lists the bodies it was built to make large (`large`),
and the tests assert the two agree before running it.  Consumers: tests/test_gpu_large_bodies.py (-m gpu),
tests/emu/lockstep.py `large` (the CPU emulation) and tests/test_ref_stepper.py (the reference's real stepper)."""
import numpy as np

f32 = np.float32
PLANE = -1


def diameters(bodies):
    """The bounding diameter class_add receives (b2d_api.cu shape_diameter), in float: inf for planes, 0 without shape."""
    from edyn_b200.rigidbody import SHAPE_BOX, SHAPE_CAPSULE, SHAPE_NONE, SHAPE_SPHERE
    sk = np.asarray(bodies["shape_kind"])
    p = np.asarray(bodies["shape_params"], f32).reshape(-1, 4)
    d = np.full(len(sk), np.inf, f32)
    d[sk == SHAPE_SPHERE] = f32(2) * p[sk == SHAPE_SPHERE, 0]
    d[sk == SHAPE_CAPSULE] = f32(2) * (p[sk == SHAPE_CAPSULE, 0] + p[sk == SHAPE_CAPSULE, 1])
    b = p[sk == SHAPE_BOX]
    d[sk == SHAPE_BOX] = f32(2) * np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])
    d[sk == SHAPE_NONE] = 0
    return d


def large_dynamic(bodies, kind=None):
    """Ids of the dynamic bodies in the brute-force list: diameter > 4 x the mean diameter of the dynamic bodies (kind
    overrides the scene's kinds, e.g. after a kind patch)."""
    d = diameters(bodies)
    dyn = np.asarray(bodies["kind"] if kind is None else kind) == 0
    counted = dyn & (d > 0) & np.isfinite(d)
    big = f32(4.0 * d[counted].astype(np.float64).sum() / counted.sum())
    return np.nonzero(dyn & (d > 0) & (~np.isfinite(d) | (d > big)))[0]


def _quat(axis, angle):
    """Rotation quaternion (x, y, z, w) in float that normalisation leaves unchanged (the reference normalises static
    bodies' orientations in its position solver; see tests/test_ref_stepper.py _unit_quat): the angle is nudged until it is."""
    ax = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    while True:
        q = np.concatenate([ax * np.sin(angle / 2), [np.cos(angle / 2)]]).astype(f32)
        n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
        if n == f32(1) and np.array_equal(q / n, q):
            return q
        angle += 1e-4


def _rotate(q, v):
    x, y, z, w = (float(c) for c in q)
    u = np.array([x, y, z])
    v = np.asarray(v, np.float64)
    return v + 2 * np.cross(u, np.cross(u, v) + w * v)


class Builder:
    """Bodies as RigidBodyDefs, a ground plane through the origin, fillers: small spheres resting far away (one-body
    islands) that keep the mean dynamic diameter small."""

    def __init__(self):
        from edyn_b200 import rigidbody as R
        self.R, self.defs, self.large, self.roots, self.touch = R, [], [], {}, []

    def add(self, name=None, large=False, **kw):
        self.defs.append(self.R.RigidBodyDef(**kw))
        i = len(self.defs) - 1
        if large:
            self.large.append(i)
        if name:
            self.roots[name] = i
        return i

    def touches(self, a, others):
        """The scene is built for body `a` to touch one of `others` (PLANE: the ground plane) at some step."""
        self.touch.append((a, list(others)))

    def box(self, he, pos, large=False, name=None, **kw):
        return self.add(name, large, shape=self.R.box_shape(tuple(he)), position=tuple(pos), **kw)

    def sphere(self, r, pos, **kw):
        return self.add(shape=self.R.sphere_shape(r), position=tuple(pos), **kw)

    def fillers(self, n=12, r=0.2, x=-9.0):
        for k in range(n):
            self.sphere(r, (x, r, 1.5 * k - 0.75 * n))

    def build(self, name, vi=10, pi=3, plane=True):
        R = self.R
        ground = len(self.defs)
        if plane:
            self.defs.append(R.RigidBodyDef(kind=R.STATIC, shape=R.plane_shape((0, 1, 0), 0.0)))
        b = R.bodies_soa(self.defs)
        touch = [(a, [ground if o == PLANE else o for o in others]) for a, others in self.touch]
        return dict(name=name, bodies=b, hinges=None, exclusions=None, dynamic=int((np.asarray(b["kind"]) == 0).sum()),
                    settings=dict(velocity_iterations=vi, position_iterations=pi), large=list(self.large), roots=dict(self.roots),
                    touch=touch)


# ---------------------------------------------------------------------------------------------------------- scenes 1-5

def plank_alone(E):
    """A plank 5 cm above the plane, twelve spheres resting 6 m away: the plank is a one-body island whose only manifold
    has a static partner."""
    s = Builder()
    s.touches(s.box((2, 0.25, 2), (0, 0.3, 0), large=True, name="plank", mass=4.0), [PLANE])
    for k in range(12):
        s.sphere(0.2, (6.0, 0.2, 0.5 * k - 3.0))
    return s.build("plank_alone")


def plank_tipping(E):
    """A plank standing on one long edge, tilted 25 degrees: its plane manifold starts with 2 points (a two-point tile)
    and grows to 4 as the plank falls onto its face (a generic tile from the rebuild of that step on)."""
    s = Builder()
    he, q = np.array([2.0, 0.1, 0.6]), _quat((1, 0, 0), 0.44)
    low = max(abs(_rotate(q, he * np.array(c))[1]) for c in [(1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1)])
    s.touches(s.box(he, (0, low + 0.004, 0), large=True, name="plank", orientation=tuple(q), mass=3.0), [PLANE])
    s.fillers()
    return s.build("plank_tipping")


def log_spheres(E):
    """Two-point island with a large body: a capsule log on the plane, five spheres dropped onto it (capsule-plane,
    sphere-capsule and sphere-plane manifolds have at most 2 points)."""
    s = Builder()
    log = s.add("log", True, shape=s.R.capsule_shape(0.25, 2.5, 0), position=(0, 0.25, 0), mass=5.0)
    s.touches(log, [s.sphere(0.15, (k - 2.0, 0.9 + 0.1 * k, 0.05 * (k - 2)), mass=0.5) for k in range(5)])
    s.touches(log, [PLANE])
    s.fillers(r=0.15)
    return s.build("log_spheres")


def plank_boxes(E):
    """Generic island with a large body: a plank resting on the plane, four small boxes dropped onto it."""
    s = Builder()
    plank = s.box((2, 0.25, 2), (0, 0.25, 0), large=True, name="plank", mass=4.0)
    s.touches(plank, [s.box((0.2, 0.2, 0.2), (x, 1.0 + 0.15 * k, z), orientation=tuple(_quat((1, 2, 3), 0.3 * k)), mass=0.5)
                      for k, (x, z) in enumerate([(-1, -1), (1, -1), (-1, 1), (1, 1)])])
    s.touches(plank, [PLANE])
    s.fillers()
    return s.build("plank_boxes")


def crates_on_statics(E):
    """Large dynamic against large static: a crate sliding into a big static wall box, and a crate resting on a tilted
    static slab, sliding down it.  Crates, wall and slab are all in the brute-force list."""
    from edyn_b200.rigidbody import Material, STATIC
    s = Builder()
    a = s.box((1.2, 1.2, 1.2), (0, 1.2, 0), large=True, name="sliding", linvel=(3.0, 0, 0), material=Material(friction=0.3))
    s.touches(a, [s.box((0.5, 2.0, 4.0), (2.6, 2.0, 0), kind=STATIC)])
    q = _quat((0, 0, 1), 0.2)
    slab = np.array([0.0, 1.5, 12.0])
    b = s.box((3.0, 0.5, 3.0), slab, kind=STATIC, orientation=tuple(q))
    s.touches(s.box((1.0, 1.0, 1.0), slab + _rotate(q, (0, 0.5 + 1.0 + 0.002, 0)), large=True, name="tilted", orientation=tuple(q),
                    material=Material(friction=0.1)), [b])
    s.fillers(r=0.1)
    return s.build("crates_on_statics")


def crate_on_kinematic(E):
    """Large dynamic against kinematic: a crate riding a moving, turning kinematic platform (both in the brute-force
    list)."""
    from edyn_b200.rigidbody import KINEMATIC
    s = Builder()
    k = s.box((3.0, 0.1, 3.0), (0, 0.3, 0), kind=KINEMATIC, linvel=(0.6, 0, 0.2), angvel=(0, 0.25, 0))
    s.touches(s.box((0.8, 0.4, 0.8), (0.3, 0.8, -0.2), large=True, name="crate", mass=2.0), [k])
    s.fillers(r=0.1)
    return s.build("crate_on_kinematic")


def two_crates(E):
    """Large dynamic against large dynamic: a crate dropped onto a resting crate, and a third crate sliding into the pair.
    Which body of a large-large pair is body[0] is decided from the brute-force side alone."""
    s = Builder()
    a = s.box((1.0, 1.0, 1.0), (0, 1.0, 0), large=True, name="bottom")
    s.touches(s.box((1.0, 1.0, 1.0), (0.3, 3.1, 0.1), large=True, name="top", orientation=tuple(_quat((0, 1, 0), 0.3))), [a])
    s.touches(s.box((0.9, 0.9, 0.9), (3.0, 0.9, 0.2), large=True, name="slider", linvel=(-4.0, 0, 0)), [a])
    s.fillers(16, r=0.1)
    return s.build("two_crates")


SCENES = {"plank_alone": plank_alone, "plank_tipping": plank_tipping, "log_spheres": log_spheres, "plank_boxes": plank_boxes,
          "crates_on_statics": crates_on_statics, "crate_on_kinematic": crate_on_kinematic, "two_crates": two_crates}


# --------------------------------------------------------------------------------------- limits: colours, restitution

GRID = [(0.45 * (i - 3.5), 0.45 * (j - 3.5)) for i in range(8) for j in range(8)]       # never closer than 0.45 m: spheres never touch


def plank_degree(E, manifolds):
    """A plank on the plane carrying `manifolds` manifolds: the plane and manifolds - 1 spheres resting on an 8 x 8 grid.
    Every manifold of the plank takes its own colour, so the colours run 0 .. manifolds - 1; 65 overflows the 64."""
    assert 1 <= manifolds <= 65
    s = Builder()
    plank = s.box((2, 0.1, 2), (0, 0.1, 0), large=True, name="plank", mass=8.0)
    for x, z in GRID[:manifolds - 1]:
        s.touches(plank, [s.sphere(0.1, (x, 0.3, z), mass=0.2)])
    s.touches(plank, [PLANE])
    return s.build(f"plank_degree_{manifolds}")


def plank_bounce(E, n, boxes=False):
    """`n` spheres (boxes: n small boxes, 4 points each) touching a resting plank and closing on it at 1 m/s, all with
    restitution: the restitution solver's walk solves them as ONE group at the plank (minus the one it starts from)."""
    from edyn_b200.rigidbody import Material
    mat = Material(restitution=0.5, friction=0.5)
    s = Builder()
    s.box((2, 0.1, 2), (0, 0.1, 0), large=True, name="plank", mass=8.0, material=mat)
    for x, z in GRID[:n]:
        if boxes:
            s.box((0.15, 0.1, 0.15), (x, 0.3, z), mass=0.2, linvel=(0, -1.0, 0), material=mat)
        else:
            s.sphere(0.1, (x, 0.3, z), mass=0.2, linvel=(0, -1.0, 0), material=mat)
    return s.build(f"plank_bounce_{n}{'_boxes' if boxes else ''}")


# -------------------------------------------------------------------------------------------------- population drift

def drift_scene(E):
    """A crate among four big spheres: NOT large (2.4 m against 4 x 0.96 m)."""
    s = Builder()
    s.box((0.8, 0.4, 0.8), (0, 0.4, 0), name="crate", mass=2.0)
    for k in range(4):
        s.sphere(0.3, (3.0, 0.3, 1.0 * k - 1.5))
    return s.build("drift")


def drift_arrivals(E, n=20):
    """Small spheres dropped onto and beside the crate: with them in the world the crate is large (2.4 m against
    4 x 0.35 m)."""
    R = E.rigidbody
    defs = [R.RigidBodyDef(shape=R.sphere_shape(0.1), position=(0.6 * (k % 5) - 1.2, 1.2 + 0.3 * (k // 5), 0.5 * (k % 3) - 0.5), mass=0.2)
            for k in range(n)]
    return R.bodies_soa(defs)
