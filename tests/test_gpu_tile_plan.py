"""The island tiles' lane plan (k_tile_plan) is written by the island rebuild and read by the tile kernels on every step, so
a CUDA-graph step that skips the rebuild solves from the plan of the last step that ran it.  After every event that
must rebuild it, the reused steps must give the bits of graphs without reuse and of plain launches, which rebuild every
step, and solve every constraint in the same order."""
import numpy as np
import pytest

from tests.parity import build_world, same_state

pytestmark = pytest.mark.gpu

LINKS = 4
KEYS = ("pos", "orn", "linvel", "angvel", "aabb", "inv_IW")
TIP_DEG = 40.0          # the tipping box stands on one edge, off balance: 2 contact points until it lands on a face


def _scene(E):
    """A slice of the chains workload (two-point islands in two-point tiles) and one box on an edge that tips onto a
    face: its manifold with the plane grows from 2 points to 4, and its island moves to a generic tile."""
    from edyn_b200.rigidbody import DYNAMIC, SHAPE_BOX
    scene = E.scenes.hinge_chains(16, 16, LINKS)
    a = np.radians(TIP_DEG)
    tip = np.array([[12.0, 0.5 * (np.sin(a) + np.cos(a)) + 0.002, 14.0]])
    orn = np.array([[0, 0, np.sin(a / 2), np.cos(a / 2)]], np.float32)
    box = E.scenes._assemble(tip, orn, np.full(1, SHAPE_BOX, np.uint32), np.array([[0.5, 0.5, 0.5, 0]], np.float32),
                             np.full(1, DYNAMIC, np.uint32))
    b = scene["bodies"]
    scene["bodies"] = {k: np.concatenate([b[k], box[k]]) for k in b}
    return scene, len(b["kind"])


def _per_body(w, dynamic):
    """The solver order as each dynamic body sees it: its hinges, then its manifolds (by partner), in the order they are
    solved.  Constraints of one colour touch disjoint dynamic bodies, so their order in the export is immaterial and
    differs with the tile an island sits in; the order per dynamic body decides the results."""
    hi, pr = w.solver_order()
    ends = w.hinge_defs()
    seq = {}
    for h in hi.tolist():
        for b in (int(ends["a"][h]), int(ends["b"][h])):
            seq.setdefault(b, []).append(("h", h))
    for a, b in pr.tolist():
        seq.setdefault(a, []).append(("m", b))
        seq.setdefault(b, []).append(("m", a))
    return {b: s for b, s in seq.items() if b in dynamic}


def _same(worlds, dynamic):
    """State (with AABBs and inverse world inertias), contacts and per-body solver order of every world equal to the
    first's."""
    same_state(*worlds, keys=KEYS)
    ref_c, ref_o = worlds[0].contacts(), _per_body(worlds[0], dynamic)
    for w in worlds[1:]:
        c = w.contacts()
        for k in ref_c:
            np.testing.assert_array_equal(c[k], ref_c[k], err_msg=f"contacts[{k}]")
        assert _per_body(w, dynamic) == ref_o, "solver order"


def _run(worlds, steps, dynamic):
    for _ in range(steps):
        for w in worlds:
            w.step(1)
        _same(worlds, dynamic)


def _points(w, body):
    c = w.contacts()
    hit = np.nonzero((c["pairs"] == body).any(axis=1))[0]
    return int(c["num"][hit].max()) if len(hit) else 0


def test_plan_follows_every_rebuild(gpu, E):
    scene, box = _scene(E)
    reuse = build_world(E, scene, "graph")
    full = build_world(E, scene, "graph", env=dict(B2D_GRAPH_REUSE="0"))
    plain = build_world(E, scene, "plain")
    worlds = (reuse, full, plain)
    dynamic = set(np.nonzero(scene["bodies"]["kind"] == 0)[0].tolist())

    def rebuilt():
        return reuse.stats()["steps_rebuilt"]

    # the box tips over while the chains settle: a two-point manifold grows past 2 points
    history = []
    for _ in range(150):
        r0 = rebuilt()
        _run(worlds, 1, dynamic)
        history.append((_points(reuse, box), rebuilt() - r0))
    assert history[0][0] == 2 and history[-1][0] == 4, [h[0] for h in history]
    grew = next(i for i in range(1, len(history)) if history[i - 1][0] <= 2 < history[i][0])
    assert history[grew][1] == 1, history[grew - 2:grew + 2]

    def event(name, apply, steps=30, min_rebuilt=1):
        r0, u0 = rebuilt(), reuse.stats()["steps_reused"]
        for w in worlds:
            apply(w)
        _run(worlds, steps, dynamic)
        assert rebuilt() - r0 >= min_rebuilt, name
        assert reuse.stats()["steps_reused"] - u0 > 0, name         # the plan was reused after the event

    # a chain thrown upwards: its manifolds with the plane are destroyed, then created again when it lands
    up = np.tile(np.array([0.0, 3.0, 0.0], np.float32), (LINKS, 1))
    event("thrown chain", lambda w: w.upload_bodies(np.arange(37 * LINKS, 38 * LINKS, dtype=np.uint32), linvel=up),
          steps=70, min_rebuilt=2)
    # a middle link removed: its manifold and both its hinges go
    dynamic -= {101 * LINKS + 2, 150 * LINKS}
    event("body and hinges removed", lambda w: w.remove_bodies(np.array([101 * LINKS + 2], np.uint32)))
    # an end link removed: one hinge goes, the rest of the chain keeps its island
    event("hinge removed", lambda w: w.remove_bodies(np.array([150 * LINKS], np.uint32)))
    # a link turned kinematic and back: the body tags and record slots of its constraints change
    link = np.array([201 * LINKS + 1], np.uint32)
    dynamic.discard(int(link[0]))
    event("kind patched to kinematic", lambda w: w.upload_bodies(link, kind=np.array([1], np.uint32)))
    defs = reuse.body_defs(link)
    dynamic.add(int(link[0]))
    event("kind patched to dynamic", lambda w: w.upload_bodies(link, kind=np.array([0], np.uint32), inv_mass=defs["inv_mass"],
                                                               inv_inertia=np.asarray(defs["inv_inertia"]).reshape(1, 9)))

    for w in worlds:
        assert w.stats()["error_flags"] == 0
    assert full.stats()["steps_reused"] == 0 and plain.stats()["steps_reused"] == 0


def test_plan_follows_sleeping(gpu, E):
    """An island falls asleep (its constraints leave the tiles) and is woken by a falling box (they come back)."""
    scene = E.scenes.sleep_and_wake()
    worlds = (build_world(E, scene, "graph", flags=E.world.FLAG_SLEEPING),
              build_world(E, scene, "graph", env=dict(B2D_GRAPH_REUSE="0"), flags=E.world.FLAG_SLEEPING),
              build_world(E, scene, "plain", flags=E.world.FLAG_SLEEPING))
    dynamic = set(np.nonzero(scene["bodies"]["kind"] == 0)[0].tolist())
    asleep = []
    for _ in range(240):
        _run(worlds, 1, dynamic)
        asleep.append(bool(worlds[0].sleeping()[0]))
    fell = asleep.index(True)
    woke = asleep.index(False, fell)
    assert fell < woke, asleep
    for w in worlds:
        assert w.stats()["error_flags"] == 0
