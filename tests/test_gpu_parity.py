"""GPU parity tests proper: the CUDA path, called through the C ABI, against (a) the committed golden vectors generated
from the real reference functions, (b) the CPU oracle on identical seeded inputs, and (c) size-independent properties
at BASELINE.json's full sizes.  Bar (tests/parity.py): bit-exact for pair lists, island partitions, contact sets,
velocities, hinge impulses, AABBs and inverse world inertias, and for poses outside the trig set -- the bodies whose
step may have taken integrate()'s sinf / cosf, which may differ from glibc's by an ulp or two (the library is built with
-fmad=false and otherwise restated operation for operation)."""
import os

import numpy as np
import pytest

from tests import parity as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32


# ----------------------------------------------------------------------------- golden vectors from the reference

def test_narrowphase_matches_reference_vectors(gpu, E):
    """Device collide() for all 15 ordered shape pairs == the reference's collide() (2 400 committed cases), bit for bit."""
    g = np.load(os.path.join(GOLD, "collide.npz"))
    n = len(g["num"])
    kinds = g["kinds"].reshape(-1)
    b = dict(pos=g["pos"].reshape(-1, 3), orn=g["orn"].reshape(-1, 4), linvel=np.zeros((2 * n, 3), f32), angvel=np.zeros((2 * n, 3), f32),
             inv_mass=np.ones(2 * n, f32), inv_inertia=np.tile(np.eye(3, dtype=f32).reshape(9), (2 * n, 1)), gravity=np.zeros((2 * n, 3), f32),
             kind=np.where(kinds == 6, 2, 0).astype(np.uint32), shape_kind=kinds.astype(np.uint32), shape_params=g["params"].reshape(-1, 4),
             friction=np.full(2 * n, 0.5, f32), restitution=np.zeros(2 * n, f32), group=None, mask=None)
    w = E.World(2 * n, max_manifolds=2 * n)
    w.add_bodies(b)
    pairs = np.stack([2 * np.arange(n), 2 * np.arange(n) + 1], axis=1).astype(np.uint32)
    w.upload_contacts(pairs, np.zeros(n, np.uint32), np.zeros((n, 4, 18), f32), np.zeros((n, 4), np.uint32))
    w.run_phases(E.world.PH_NARROW)
    c = w.contacts()
    idx = {tuple(p): k for k, p in enumerate(c["pairs"].tolist())}
    bad = 0
    for i in range(n):
        k = idx[(2 * i, 2 * i + 1)]
        m = int(g["num"][i])
        assert int(c["num"][k]) == m, f"case {i} kinds {g['kinds'][i]}: {c['num'][k]} points, reference {m}"
        # new points are pushed at the list head: slot order is the reverse of creation order
        got = c["pts"][k, :m][::-1]
        ref_pts = g["pts"][i, :m]
        same = (np.array_equal(got[:, 0:9], ref_pts[:, 0:9]) and np.array_equal(got[:, 12], ref_pts[:, 9])
                and np.array_equal(c["att"][k, :m][::-1], g["att"][i, :m]))
        bad += 0 if same else 1
    assert bad == 0, f"{bad} of {n} cases differ from the reference vectors"


def test_refresh_matches_reference_vectors(gpu, E):
    """AABBs (util/aabb_util.cpp) and inertia_world_inv (sys/update_inertias.cpp) computed on the device."""
    g = np.load(os.path.join(GOLD, "aabb.npz"))
    m = len(g["kind"])
    np_ = len(g["planes"])
    bm = np.load(os.path.join(GOLD, "body_math.npz"))
    b = dict(pos=np.concatenate([g["pos"], np.zeros((np_, 3), f32)]), orn=np.concatenate([g["orn"], np.tile([0, 0, 0, 1], (np_, 1)).astype(f32)]),
             linvel=np.zeros((m + np_, 3), f32), angvel=np.zeros((m + np_, 3), f32), inv_mass=np.ones(m + np_, f32),
             inv_inertia=np.concatenate([bm["inv_inertia"][:m], np.zeros((np_, 9), f32)]), gravity=np.zeros((m + np_, 3), f32),
             kind=np.concatenate([np.zeros(m), np.full(np_, 2)]).astype(np.uint32), shape_kind=np.concatenate([g["kind"], np.full(np_, 6)]).astype(np.uint32),
             shape_params=np.concatenate([g["params"], g["planes"]]), friction=np.full(m + np_, 0.5, f32), restitution=np.zeros(m + np_, f32), group=None, mask=None)
    w = E.World(m + np_)
    w.add_bodies(b)
    st = w.download_state(aabb=True, inv_IW=True)
    assert np.array_equal(st["aabb"][:m], g["aabb"])
    assert np.array_equal(st["aabb"][m:], g["plane_aabb"])
    # inertia_world_inv for the fixture's orientations: upload them, refresh, compare
    w2 = E.World(m)
    b2 = {k: (v[:m] if v is not None else None) for k, v in b.items()}
    b2["orn"] = bm["q"][:m]
    w2.add_bodies(b2)
    assert np.array_equal(w2.download_state(inv_IW=True)["inv_IW"], bm["inv_inertia_world"][:m])


def test_integrate_matches_reference_vectors(gpu, E):
    """integrate(q, w, dt) (math/quaternion.cpp:7-22) through one gravity-free, contact-free step."""
    bm = np.load(os.path.join(GOLD, "body_math.npz"))
    sel = np.where(bm["dt"] > 0)[0]
    m = len(sel)
    b = dict(pos=np.zeros((m, 3), f32), orn=bm["q"][sel], linvel=np.zeros((m, 3), f32), angvel=bm["w"][sel], inv_mass=np.ones(m, f32),
             inv_inertia=np.tile(np.eye(3, dtype=f32).reshape(9), (m, 1)), gravity=np.zeros((m, 3), f32), kind=np.zeros(m, np.uint32),
             shape_kind=np.full(m, 255, np.uint32), shape_params=np.zeros((m, 4), f32), friction=np.zeros(m, f32), restitution=np.zeros(m, f32), group=None, mask=None)
    w = E.World(m)
    w.add_bodies(b)
    w.step(1)
    q = w.download_state(aabb=False)["orn"]
    # sinf/cosf on the device may differ from glibc's by an ulp; everything else in the expression is exact
    assert np.abs(q - bm["q_out"][sel]).max() <= 2.4e-7
    assert (q == bm["q_out"][sel]).mean() > 0.9


def test_broadphase_matches_reference_tree_vectors(gpu, E):
    """Device broadphase (uniform grid) == the pair lists the reference's own dynamic AABB trees produce
    (tests/golden/broadphase.npz, generated with oracle/_ref): ordered pairs, 12 crowded scenes."""
    g = np.load(os.path.join(GOLD, "broadphase.npz"))
    keys = [k[4:] for k in g.files if k.startswith("soa_")]
    off = po = 0
    for i, (n, c) in enumerate(zip(g["sizes"].tolist(), g["counts"].tolist())):
        soa = {k: g["soa_" + k][off:off + n] for k in keys}
        w = E.World(n, max_manifolds=max(4096, 4 * c))
        w.add_bodies(soa)
        assert np.array_equal(w.download_state(aabb=True)["aabb"], g["aabb1"][off:off + n])
        w.run_phases(E.world.PH_BROAD)
        P.check_pairs(f"0 of scene {i}", w.pairs(), g["pairs"][po:po + c])
        assert w.stats()["error_flags"] == 0
        off += n; po += c


# ----------------------------------------------------------------------------- lock-step against the oracle

SCENES = {
    "hello_world": (lambda E: E.scenes.hello_world(), 150),
    "boxes_64": (lambda E: E.scenes.boxes_on_plane(4, jitter=0.01), 100),
    "spheres_144": (lambda E: E.scenes.spheres_in_box(6, 4, 6), 100),
    "mixed_216": (lambda E: E.scenes.mixed_pile(6), 160),
    "chains_64": (lambda E: E.scenes.hinge_chains(4, 4), 80),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_lockstep_phase_parity(gpu, E, O, name):
    """Every phase of every step against the oracle on the same inputs: ORDERED broadphase pair list (which body is
    body[0] included), contact points, island labels, and the post-solve state with the oracle replaying the device's
    Gauss-Seidel order (the coloured parallel solve is a permutation of the sequential sweep)."""
    make, steps = SCENES[name]
    scene = make(E)
    w = E.scenes.build_world(scene)
    o = P.oracle_for(O, scene)
    res = None
    for s in range(steps):
        # every step a fresh single-step comparison: the oracle continues from the device's bodies, contacts and joints
        res = P.tally(res, P.phase_step(E, O, w, o, s))
    P.report(name, res)
    assert w.stats()["error_flags"] == 0
    assert res["bitwise"] > 0, res


def test_solver_only_parity_from_injected_contacts(gpu, E, O):
    """Row preparation + warm start + velocity iterations + integration + position iterations in isolation: the same
    manifolds (with non-zero warm-start impulses) are injected on both sides."""
    scene = E.scenes.mixed_pile(5)
    o = P.oracle_for(O, scene)
    o.step(60)
    st, c = o.state(), o.contacts()
    assert c["num"].sum() > 100
    w = E.scenes.build_world(scene)
    w.upload_state(st["pos"], st["orn"], st["linvel"], st["angvel"])
    w.upload_contacts(c["pairs"], c["num"], c["pts"], c["att"], c["lifetime"])
    P.islands(E, O, w, o, 0)
    # the settled pile is one island with spinning bodies in it, so every pose is in the trig set: what this holds to
    # bits is the velocities, the applied impulses and the AABBs and inertias of the device's poses
    g, _ = P.solve(E, O, w, o, 0)
    P.resync(o, w, 0, g)


# ----------------------------------------------------------------------------- free-running trajectories

def test_hello_world_1000_steps(gpu, E, O):
    """BASELINE.json: positions within 1e-4 relative of the CPU stepper after 1000 steps (config 1).  The oracle runs
    FREE here, in its own natural Gauss-Seidel order."""
    scene = E.scenes.hello_world()
    w = E.scenes.build_world(scene)
    o = P.oracle_for(O, scene)
    w.step(1000); o.step(1000)
    g, c = w.download_state(), o.state()
    rel = np.abs(g["pos"][0] - c["pos"][0]).max() / max(1.0, np.abs(c["pos"][0]).max())
    assert rel <= 1e-4, rel
    assert abs(g["pos"][0, 1] - 0.5) < 1e-3 and w.contacts()["num"].tolist() == [4]


def test_box_stacks_1000_steps(gpu, E, O):
    """Config 2 in miniature (27 stacks of 3 boxes) against the FREE-running CPU stepper, which sweeps rows in a different
    Gauss-Seidel order.  Heights agree to 1e-6; the residual is a lateral drift of ~4e-4 m picked up while the stacks
    settle (any two row orders differ by that much, the reference against itself included), hence 5e-4 here and 1e-4 only
    for the order-independent single-body case above."""
    scene = E.scenes.boxes_on_plane(3)
    w = E.scenes.build_world(scene)
    o = P.oracle_for(O, scene)
    w.step(1000); o.step(1000)
    g, c = w.download_state(), o.state()
    n = scene["dynamic"]
    rel = np.abs(g["pos"][:n] - c["pos"][:n]).max() / np.abs(c["pos"][:n]).max()
    assert rel <= 5e-4, rel
    assert np.abs(g["pos"][:n, 1] - c["pos"][:n, 1]).max() <= 1e-5


# ----------------------------------------------------------------------------- properties at BASELINE.json's full sizes

def _check_world_invariants(E, w, scene, nsteps):
    n = scene["dynamic"]
    w.step(nsteps)
    st = w.download_state(aabb=True)
    assert np.isfinite(st["pos"]).all() and np.isfinite(st["linvel"]).all()
    assert np.abs(np.linalg.norm(st["orn"][:n], axis=1) - 1).max() < 1e-5
    s = w.stats()
    assert s["error_flags"] == 0
    pairs = w.pairs()
    keys = np.sort(np.minimum(pairs[:, 0], pairs[:, 1]).astype(np.uint64) << np.uint64(32) | np.maximum(pairs[:, 0], pairs[:, 1]).astype(np.uint64))
    assert len(np.unique(keys)) == len(keys), "duplicate manifolds for one body pair"
    # every surviving manifold satisfies the non-separation predicate it was kept under (broadphase.cpp:119-134);
    # AABBs moved after the broadphase ran, so allow the distance travelled in one step
    a, b = st["aabb"][pairs[:, 0]], st["aabb"][pairs[:, 1]]
    gap = np.maximum(a[:, 0:3] - b[:, 3:6], b[:, 0:3] - a[:, 3:6]).max(axis=1)
    assert gap.max() < 0.026 + 0.25
    # island labels: a partition whose representative is the smallest member; manifolds between dynamic bodies never cross
    lab = w.islands()
    dyn = scene["bodies"]["kind"] == 0
    assert (lab[dyn] <= np.arange(len(lab))[dyn]).all() and (lab[lab[dyn]] == lab[dyn]).all()
    both = dyn[pairs[:, 0]] & dyn[pairs[:, 1]]
    assert (lab[pairs[both, 0]] == lab[pairs[both, 1]]).all()
    # exported Gauss-Seidel order: a permutation of the manifolds that carry points
    hi, pr = w.solver_order()
    c_keys = np.minimum(pr[:, 0], pr[:, 1]).astype(np.uint64) << np.uint64(32) | np.maximum(pr[:, 0], pr[:, 1]).astype(np.uint64)
    assert len(np.unique(c_keys)) == len(c_keys) and np.isin(c_keys, keys).all()
    return st, s


def test_full_size_mixed_pile_properties(gpu, E):
    """Config 4 at full size (262 144 bodies): determinism (two worlds, identical bits), idempotent broadphase,
    structural invariants, bounded penetration."""
    scene = E.scenes.mixed_pile(64)
    w1 = E.scenes.build_world(scene)
    st1, s1 = _check_world_invariants(E, w1, scene, 120)
    w2 = E.scenes.build_world(scene)
    w2.step(120)
    st2 = w2.download_state(aabb=True)
    for k in ("pos", "orn", "linvel", "angvel"):
        assert np.array_equal(st1[k], st2[k]), f"non-deterministic {k}"
    w1.run_phases(E.world.PH_BROAD)                 # bring the manifold set up to date with the moved AABBs ...
    before = w1.pairs()
    w1.run_phases(E.world.PH_BROAD)                 # ... then a second pass over the same AABBs must change nothing
    P.check_pairs("after a second broadphase", w1.pairs(), before)
    n = scene["dynamic"]
    assert st1["pos"][:n, 1].min() > -0.05, "bodies sank through the floor"
    assert s1["contact_points"] > n // 2


def test_full_size_hinge_chains_properties(gpu, E):
    """Config 5 at full size (1 048 576 bodies in 262 144 four-link chains): every chain is one island of 4 bodies, the
    hinges hold (pivot gap small) and the chains rest on the plane."""
    scene = E.scenes.hinge_chains(512, 512)
    w = E.scenes.build_world(scene, max_manifolds=3 * scene["dynamic"])
    st, s = _check_world_invariants(E, w, scene, 40)
    n = scene["dynamic"]
    lab = w.islands()[:n].reshape(-1, 4)
    assert (lab == lab[:, :1]).all() and len(np.unique(lab[:, 0])) == n // 4
    assert s["islands"] == n // 4 and s["hinge_colors"] == 2
    pos = st["pos"][:n].reshape(-1, 4, 3)
    gap = np.linalg.norm(pos[:, 1:] - pos[:, :-1], axis=2)
    assert np.abs(gap - 0.7).max() < 5e-3
    assert np.abs(st["pos"][:n, 1] - 0.1).max() < 5e-3


def test_spheres_65536_rest_in_box(gpu, E):
    """Config 3 at full size: nothing escapes the five planes, energy decays."""
    scene = E.scenes.spheres_in_box()
    w = E.scenes.build_world(scene)
    st, s = _check_world_invariants(E, w, scene, 150)
    n = scene["dynamic"]
    p = st["pos"][:n]
    assert p[:, 1].min() > 0.2 and p[:, 0].min() > -0.3 and p[:, 2].min() > -0.3
    assert np.linalg.norm(st["linvel"][:n], axis=1).mean() < 1.0


# ----------------------------------------------------------------------------- C ABI behaviour

def test_state_round_trip_and_errors(gpu, E):
    scene = E.scenes.boxes_on_plane(3)
    w = E.scenes.build_world(scene)
    st = w.download_state(aabb=False)
    w.upload_state(st["pos"], st["orn"], st["linvel"], st["angvel"])
    st2 = w.download_state(aabb=False)
    for k in ("pos", "orn", "linvel", "angvel"):
        assert np.array_equal(st[k], st2[k])
    bad = dict(scene["bodies"])
    bad["shape_kind"] = bad["shape_kind"].copy(); bad["shape_kind"][0] = 1         # cylinder: out of scope -> error, no fallback
    w3 = E.World(64)
    with pytest.raises(E.B2DError, match="scope"):
        w3.add_bodies(bad)
    with pytest.raises(E.B2DError, match="max_bodies"):
        E.World(4).add_bodies(scene["bodies"])


def test_manifold_capacity_overflow_is_reported(gpu, E):
    scene = E.scenes.spheres_in_box(8, 4, 8, jitter=0.0)
    w = E.scenes.build_world(scene, max_manifolds=64)
    w.step(60)
    assert w.stats()["error_flags"] & 1
