"""Large DYNAMIC bodies on the device, in lock step with the oracle.  A body more than 4 x the mean dynamic diameter is
searched brute force (F_LARGE); its constraints are filed under it, or under its small dynamic partner (key_body), and
must sort into its island's tile like everybody else's.  Scenes (tests/large_scenes.py): a plank alone on the plane, a
plank tipping from an edge onto its face (its plane manifold grows from 2 to 4 points in a two-point tile), a log under
falling spheres (two-point tile), a plank under falling boxes (generic tile), crates against a static wall and on a
tilted static slab, a crate on a moving kinematic platform, three crates touching each other, a plank at 32 / 33 / 63 /
64 manifolds (the colour limit), the restitution solver at its group limits (32 manifolds, 96 points) and a crate whose
class flips between steps (bodies added, a kind patch to static and back).

Every step, in three modes (plain launches, CUDA graphs with rebuild reuse, dataflow only) and with both neighbourhood
searches (warp per body, and thread per body: B2D_BP_WARP_MAX=0): the tile packing against its restatement
(tests/tile_packing.py), the oracle lock step of tests/parity.py, and all runs bit-identical to each other (state
and ordered pair set).  Each test first asserts that its scene has the large dynamic bodies it was built for, by the
host's rule restated in numpy.  Also runs against the CPU emulation (B2D_EMU=1: no graphs, fewer steps); the cases
beyond the limits run there only (tests/test_emu_device.py)."""
import os

import numpy as np
import pytest

from tests import large_scenes as L
from tests import tile_packing as TP
from tests.parity import lockstep, oracle_for, load, report, same_digests

pytestmark = pytest.mark.gpu

EMU = os.environ.get("B2D_EMU") == "1"
STEPS = 40 if EMU else 100
MODES = ("plain", "dataflow") if EMU else ("plain", "graph", "dataflow")
SEARCH = {"warp": None, "thread": {"B2D_BP_WARP_MAX": "0"}}


class Recorder(TP.PackingCheck):
    """The packing check, plus per step: the points of every manifold (unordered pair -> count) and the tile of each
    large body."""

    def __init__(self, scene, large):
        super().__init__(scene)
        self.large, self.points, self.tiles = list(large), [], []

    def __call__(self, step, w):
        p = super().__call__(step, w)
        c = w.contacts()
        self.points.append({tuple(sorted(q)): int(n) for q, n in zip(c["pairs"].tolist(), c["num"].tolist()) if n})
        m = w.debug_tile_map()
        self.tiles.append([(int(m["btile"][b]), int(m["ntiles2"])) for b in self.large])
        return p


def assert_large(scene):
    got = L.large_dynamic(scene["bodies"]).tolist()
    assert got and got == scene["large"], f"{scene['name']}: large dynamic bodies {got}, built for {scene['large']}"


def assert_touches(scene, rec):
    for a, others in scene["touch"]:
        hit = [o for o in others if any(tuple(sorted((a, o))) in pts for pts in rec.points)]
        assert hit, f"{scene['name']}: body {a} never touched any of {others}"


def run_all(E, O, scene, steps=STEPS, modes=MODES, search=("warp", "thread"), **kw):
    """Every (search, mode) run of `scene`; asserts the lock step, the packing and that all runs are bit-identical.
    Returns {(search, mode): (result, recorder)}."""
    out = {}
    for s in search:
        for mode in modes:
            rec = Recorder(scene, scene["large"])
            res = lockstep(E, O, scene, steps, mode=mode, hook=rec, env=SEARCH[s], **kw)
            assert res["ok"], (s, mode, res)
            report(f"{scene['name']} {s} {mode}", res)
            assert res["bitwise"] > 0, (s, mode, res["bitwise"], res["trig"])
            assert rec.rebuilt + rec.reused == steps
            if mode == "dataflow":
                assert rec.tiled_steps == 0
            out[(s, mode)] = (res, rec)
    same_digests({f"{scene['name']} {k}": res["digests"] for k, (res, _) in out.items()})
    return out


@pytest.mark.parametrize("name", list(L.SCENES))
def test_large_dynamic_bodies_lockstep(gpu, E, O, name):
    scene = L.SCENES[name](E)
    assert_large(scene)
    out = run_all(E, O, scene)
    rec = out[("warp", "plain")][1]
    assert_touches(scene, rec)
    # in plain mode every large body with a manifold is in a tile: its constraints with static / kinematic partners too
    for s, step_tiles in enumerate(rec.tiles):
        for b, (t, _) in zip(scene["large"], step_tiles):
            if any(b in q for q in rec.points[s]):
                assert t != TP.TILE_NONE, f"{name} step {s}: large body {b} has contacts but no tile"
    if name == "plank_tipping":
        plank, ground = scene["roots"]["plank"], len(scene["bodies"]["kind"]) - 1
        n = [pts.get((plank, ground), 0) for pts in rec.points]
        first = next(i for i, k in enumerate(n) if k)
        assert n[first] == 2 and max(n) == 4, n
        cls = [t < n2 for t, n2 in (st[0] for st in rec.tiles)]
        assert cls[first] and not cls[-1], "the plank should move from a two-point tile to a generic one"
    if name == "log_spheres":
        assert all(t < n2 for t, n2 in (st[0] for st in rec.tiles) if t != TP.TILE_NONE)


def test_large_dynamic_bodies_without_position_iterations(gpu, E, O):
    """The tile kernel without position iterations: it writes back the integrated pose and k_integrate refreshes the
    tiled bodies' inertia and AABB."""
    for name in L.SCENES:
        scene = L.SCENES[name](E)
        assert_large(scene)
        run_all(E, O, scene, steps=STEPS // 2, search=("warp",), pos_iters=0)


@pytest.mark.parametrize("manifolds", [32, 33, 63, 64])
def test_plank_at_the_colour_limit(gpu, E, O, manifolds):
    """One body carrying 32 / 33 / 63 / 64 manifolds: its colours run 0 .. manifolds - 1, so at 64 the colour masks, the
    8-bit ticket fields and the tile key's 6 colour bits are full.  In a tile and on the dataflow path."""
    scene = L.plank_degree(E, manifolds)
    assert_large(scene)
    out = run_all(E, O, scene, steps=STEPS // 2, search=("warp",))
    for (s, mode), (res, rec) in out.items():
        assert res["colors"] == manifolds, (mode, res["colors"])
        assert_touches(scene, rec)
        if mode == "plain":
            assert all(st[0][0] != TP.TILE_NONE for st in rec.tiles)


@pytest.mark.parametrize("n,boxes", [(32, False), (24, True)], ids=["32_manifolds", "96_points"])
def test_restitution_solver_at_its_group_limits(gpu, E, O, n, boxes):
    """FLAG_RESTITUTION_SOLVER, bodies closing on a resting plank at 1 m/s: the walk starts at one of them and solves the
    plank's closing manifolds as one group -- the other n - 1 and the plane's: 32 manifolds (spheres), or 23 x 4 + 4 = 96
    points (boxes).  One body more overflows the group (tests/test_emu_device.py)."""
    scene = L.plank_bounce(E, n, boxes=boxes)
    assert_large(scene)
    run_all(E, O, scene, steps=STEPS // 2, search=("warp",), restitution_solver=True)


def drift_events(E, O, scene, arrivals, log):
    """before(step, world, oracle) of the drift test: at step 5 the arrivals land (the crate becomes large), at step 25
    the crate is patched static, at step 40 dynamic again.  The oracle has no kind patch: it is rebuilt from the device's
    state with the new kinds and continues from the device's manifolds, as it does every step."""
    from edyn_b200.rigidbody import DYNAMIC, STATIC
    crate = scene["roots"]["crate"]
    bodies = {k: np.concatenate([np.asarray(scene["bodies"][k]), np.asarray(arrivals[k])]) for k in scene["bodies"]}
    n0 = len(scene["bodies"]["kind"])

    def rebuilt(w, kind):
        g = w.download_state()
        b = {k: v.copy() for k, v in bodies.items()}
        b.update(pos=g["pos"], orn=g["orn"], linvel=g["linvel"], angvel=g["angvel"], kind=kind)
        if kind[crate] != DYNAMIC:
            b["inv_mass"][crate], b["inv_inertia"][crate] = 0, 0
        o = oracle_for(O, dict(scene, bodies=b))
        load(o, w, g)
        return o

    def before(s, w, o):
        kind = bodies["kind"].copy()
        if s == 5:
            w.add_bodies(arrivals); o.add_bodies(arrivals)
        if s in (25, 40):
            kind[crate] = STATIC if s == 25 else DYNAMIC
            patch = dict(kind=[kind[crate]])
            if s == 40:
                patch.update(inv_mass=bodies["inv_mass"][[crate]], inv_inertia=bodies["inv_inertia"][[crate]].reshape(1, 9))
            w.upload_bodies([crate], **patch)
            o = rebuilt(w, kind)
        if s in (0, 5, 25, 40):
            n = n0 if s == 0 else len(kind)
            log.append((s, L.large_dynamic({k: v[:n] for k, v in bodies.items()}, kind=kind[:n]).tolist()))
        return o
    return before


def test_large_class_flips_between_steps(gpu, E, O):
    """classify_arrivals / reclassify move a crate into the brute-force list when small bodies arrive, and the class
    follows a kind patch to static and back; the lock step holds through every change."""
    scene, arrivals = L.drift_scene(E), L.drift_arrivals(E)
    crate, steps = scene["roots"]["crate"], 60
    digests = {}
    for s in SEARCH:
        for mode in MODES:
            log = []
            res = lockstep(E, O, scene, steps, mode=mode, hook=TP.PackingCheck(scene), env=SEARCH[s], max_bodies=len(scene["bodies"]["kind"]) + len(arrivals["kind"]),
                           before=drift_events(E, O, scene, arrivals, log))
            assert res["ok"], (s, mode, res)
            assert [(k, crate in lg) for k, lg in log] == [(0, False), (5, True), (25, False), (40, True)], log
            digests[(s, mode)] = res["digests"]
    same_digests(digests)
