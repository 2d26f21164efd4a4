"""TEST INFRASTRUCTURE.  The library's CUDA kernels, executed by the CPU emulation (tests/emu), in lock step with the
oracle through the normal Python adapter and C ABI -- the same comparison tests/test_gpu_parity.py makes on the GPU: ordered
pair lists identical as multisets (a pair with two manifolds is a difference), post-solve state within 1e-5 (here: identical, glibc's sinf / cosf on both sides) with the oracle
replaying the device's Gauss-Seidel order, manifolds and joint impulses re-synchronised every step.  The -m gpu lock-step
tests (test_gpu_tile_edges.py, test_gpu_random_lockstep.py) call `lockstep` in-process, on the GPU or the emulation.

    python tests/emu/lockstep.py fixed|narrow|wide|large|beyond FIRST LAST [--tiles 0|1] [--steps N] [--restitution] [--mutate]
                                 [--bp-warp-max N]     -> one JSON line
large: scenes with large dynamic bodies (tests/large_scenes.py), within every limit; beyond: the same content past the
64 colours and the restitution group's 32 manifolds / 96 points, flags only (tiles on: a colour clash on the dataflow
path would spend the waits' whole spin budget).
Runs in its own process because B2D_LIB has to be set before edyn_b200 is imported."""
import json
import os
import sys
import time
from collections import Counter

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


# How the device runs the step: plain launches that rebuild the islands every step, CUDA graphs that skip the rebuild while
# the constraint graph is unchanged, and everything on the dataflow path (no island tiles).  The emulation launches plainly.
MODES = {"plain": dict(B2D_GRAPH="0", B2D_GRAPH_REUSE="1", B2D_TILES="1"),
         "graph": dict(B2D_GRAPH="1", B2D_GRAPH_REUSE="1", B2D_TILES="1"),
         "dataflow": dict(B2D_GRAPH="0", B2D_GRAPH_REUSE="1", B2D_TILES="0")}
STATE_KEYS = ("pos", "orn", "linvel", "angvel", "aabb")


def build_world(E, scene, mode=None, env=None, **kw):
    """E.scenes.build_world with the environment of `mode` (read when the world is created) and the extra variables `env`;
    None: as the environment is."""
    env = {**(MODES[mode] if mode is not None else {}), **(env or {})}
    if not env:
        return E.scenes.build_world(scene, **kw)
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return E.scenes.build_world(scene, **kw)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def lockstep(E, O, scene, steps, restitution_solver=False, mode=None, hook=None, vel_iters=None, pos_iters=None, env=None,
             before=None, max_bodies=None):
    """One device world in `mode` (a key of MODES; None: as the environment says) against the oracle, `steps` single
    steps.  vel_iters / pos_iters override the scene's settings on both sides; env: more environment variables for the
    world's creation; hook(step, world) runs after each step's comparison (and may assert); before(step, world, oracle)
    runs before each step, may change both worlds and returns the oracle to continue with; max_bodies reserves room for
    bodies added on the way.  Returns ok, worst (largest state difference), exact (bit-identical steps), points (contact
    points at the end), max_points (most points in one manifold at any step), flags, and digests: one hash of the device
    state and ordered pair set per step, for comparing modes."""
    import hashlib
    import numpy as np
    st = dict(scene["settings"])
    if vel_iters is not None:
        st["velocity_iterations"] = vel_iters
    if pos_iters is not None:
        st["position_iterations"] = pos_iters
    w = build_world(E, scene, mode, env, flags=E.world.FLAG_RESTITUTION_SOLVER if restitution_solver else 0, max_bodies=max_bodies, **st)
    o = O.OracleWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"])
    if restitution_solver:
        o.set_restitution_iterations(8, 3)          # no graph order handed over: the oracle's defaults are the device's conventions
    o.add_bodies(scene["bodies"])
    if scene["hinges"]:
        h = scene["hinges"]
        o.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    if scene["exclusions"] is not None:
        o.add_exclusions(*scene["exclusions"])
    worst, exact, max_points, digests = 0.0, 0, 0, []
    for s in range(steps):
        if before is not None:
            o = before(s, w, o)
        w.step(1)
        hi, pr = w.solver_order()
        o.run_phases(O.PH_BROAD | O.PH_NARROW | O.PH_ISLANDS)
        o.set_order(hi, pr)
        o.run_phases(O.PH_SOLVE)
        g, c = w.download_state(), o.state()
        wp = w.pairs()
        if Counter(map(tuple, wp.tolist())) != Counter(map(tuple, o.pairs().tolist())):
            return dict(ok=False, step=s, why="ordered broadphase pair lists differ")
        if not np.array_equal(w.islands(), o.islands()):
            return dict(ok=False, step=s, why="island labels differ")
        err = max(float(np.abs(g[k] - c[k]).max()) for k in STATE_KEYS)
        worst = max(worst, err)
        exact += err == 0.0
        if err > 1e-5:
            return dict(ok=False, step=s, why=f"state differs by {err:.3e}")
        wp = wp[np.lexsort((wp[:, 1], wp[:, 0]))] if len(wp) else wp
        digests.append(hashlib.sha1(b"".join(np.ascontiguousarray(x).tobytes() for x in [g[k] for k in STATE_KEYS] + [wp])).hexdigest())
        o.set_state(g["pos"], g["orn"], g["linvel"], g["angvel"])
        gc = w.contacts()
        max_points = max(max_points, int(gc["num"].max(initial=0)))
        o.set_contacts(gc["pairs"], gc["num"], gc["pts"], gc["att"], gc["lifetime"])
        if scene["hinges"]:
            o.set_hinge_impulses(w.hinge_impulses())
        if hook is not None:
            hook(s, w)
    stats = w.stats()
    w.close()
    return dict(ok=stats["error_flags"] == 0, worst=worst, exact=exact, points=int(stats["contact_points"]), max_points=max_points,
                flags=int(stats["error_flags"]), reused=int(stats["steps_reused"]), colors=int(stats["contact_colors"]), digests=digests)


def over_the_limit(E, scene, steps, restitution_solver=False):
    """The device alone, `steps` steps of a scene beyond one of its limits: the error flags and what World.sync() raises
    (None: nothing).  No oracle: past a limit the state is not meant to match."""
    w = build_world(E, scene, None, flags=E.world.FLAG_RESTITUTION_SOLVER if restitution_solver else 0, **scene["settings"])
    w.step(steps)
    flags = int(w.stats()["error_flags"])
    try:
        w.sync()
        raised = None
    except E.world.B2DError as e:
        raised = str(e)
    w.close()
    return dict(ok=True, flags=flags, raised=raised)


def lockstep_with_mutations(E, O, scene, steps, seed):
    """Same comparison while user code interferes every 13th step: b2d_remove_bodies, b2d_remove_exclusions, b2d_add_bodies,
    b2d_upload_bodies (a patched velocity)."""
    import numpy as np
    R = E.rigidbody
    rng = np.random.default_rng(seed)
    st = scene["settings"]
    nb = len(scene["bodies"]["kind"])
    w = E.scenes.build_world(scene, max_bodies=nb + 16)
    o = O.OracleWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"])
    o.add_bodies(scene["bodies"])
    if scene["hinges"]:
        h = scene["hinges"]
        o.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    if scene["exclusions"] is not None:
        o.add_exclusions(*scene["exclusions"])
    kind = np.asarray(scene["bodies"]["kind"]).copy()
    alive = np.ones(len(kind), bool)
    excluded = list(zip(*[x.tolist() for x in scene["exclusions"]])) if scene["exclusions"] is not None else []
    events = 0
    for s in range(steps):
        if s and s % 13 == 0:
            what, movable = rng.integers(4), np.where(alive & (kind == 0))[0]
            if what == 0 and len(movable) > 4:
                b = int(rng.choice(movable))
                w.remove_bodies([b]); o.remove_bodies([b]); alive[b] = False
            elif what == 1 and excluded:
                a, b = excluded.pop()
                if alive[a] and alive[b]:
                    w.remove_exclusions([a], [b]); o.remove_exclusions([a], [b])
            elif what == 3 and len(kind) < nb + 16:
                d = R.RigidBodyDef(position=tuple(rng.uniform([-1, 2, -1], [1, 4, 1])), mass=float(rng.choice([0.5, 1.0, 2.0])), linvel=tuple(rng.uniform(-2, 2, 3)),
                                   shape=[R.sphere_shape(0.3), R.box_shape((0.3, 0.2, 0.25)), R.capsule_shape(0.15, 0.3, 1)][rng.integers(3)])
                soa = R.bodies_soa([d])
                w.add_bodies(soa); o.add_bodies(soa)
                kind, alive = np.append(kind, 0), np.append(alive, True)
            else:
                b = int(rng.choice(movable))
                lv, av = rng.uniform(-3, 3, (1, 3)).astype(np.float32), rng.uniform(-3, 3, (1, 3)).astype(np.float32)
                w.upload_bodies([b], linvel=lv, angvel=av)
                x = o.state()
                x["linvel"][b], x["angvel"][b] = lv[0], av[0]
                o.set_state(x["pos"], x["orn"], x["linvel"], x["angvel"])
            events += 1
        w.step(1)
        hi, pr = w.solver_order()
        o.run_phases(O.PH_BROAD | O.PH_NARROW | O.PH_ISLANDS)
        o.set_order(hi, pr)
        o.run_phases(O.PH_SOLVE)
        g, c = w.download_state(), o.state()
        if Counter(map(tuple, w.pairs().tolist())) != Counter(map(tuple, o.pairs().tolist())):
            return dict(ok=False, step=s, why="ordered broadphase pair lists differ")
        err = max(float(np.abs(g[k][alive] - c[k][alive]).max()) for k in ("pos", "orn", "linvel", "angvel"))
        if err > 1e-5:
            return dict(ok=False, step=s, why=f"state differs by {err:.3e}")
        o.set_state(g["pos"], g["orn"], g["linvel"], g["angvel"])
        gc = w.contacts()
        o.set_contacts(gc["pairs"], gc["num"], gc["pts"], gc["att"], gc["lifetime"])
        if scene["hinges"]:
            o.set_hinge_impulses(w.hinge_impulses())
    flags = int(w.stats()["error_flags"])
    w.close()
    return dict(ok=flags == 0, worst=0.0, points=events, flags=flags)


def free_run_against_real_stepper(E, O):
    """No oracle in between: the kernels (emulated) and the reference's real stepper, both free-running from the same scene.
    Hinge chains are insensitive to the sweep order (tiny islands at rest), so the two must simply agree; hello_world must be
    identical while the box falls.  The reference's side is its recorded states (tests/golden/free_run.npz)."""
    import numpy as np
    from tests.golden import make_whole_step as G
    out = []
    for name in ("chains_64", "hello_world"):
        scene, marks = G.free_run_scene(E, name), G.FREE_RUN[name][2]
        w = E.scenes.build_world(scene)
        n, done = scene["dynamic"], 0
        for m in marks:
            w.step(m - done); done = m
            g, c = w.download_state(), G.reference_free_run(name, m)
            out.append(dict(scene=name, step=m, dpos=float(np.abs(g["pos"][:n] - c["pos"][:n]).max()), dvel=float(np.abs(g["linvel"][:n] - c["linvel"][:n]).max())))
        w.close()
    return out


def main():
    kind, first, last = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    tiles = sys.argv[sys.argv.index("--tiles") + 1] if "--tiles" in sys.argv else "1"
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 100
    restitution = "--restitution" in sys.argv
    from tests.emu import build
    os.environ["B2D_LIB"] = build.build()
    mode = "dataflow" if tiles == "0" else "plain"
    import edyn_b200 as E
    from oracle import oracle as O
    from tests.test_ref_stepper import random_scene, random_scene_wide
    from tests import large_scenes as L
    env = {"B2D_BP_WARP_MAX": sys.argv[sys.argv.index("--bp-warp-max") + 1]} if "--bp-warp-max" in sys.argv else None
    large = [lambda name=name: L.SCENES[name](E) for name in L.SCENES] + [lambda k=k: L.plank_degree(E, k) for k in (32, 33, 63, 64)]
    beyond = [(lambda: L.plank_degree(E, 65), False), (lambda: L.plank_bounce(E, 33), True), (lambda: L.plank_bounce(E, 25, boxes=True), True)]
    fixed = [lambda: E.scenes.hello_world(), lambda: E.scenes.boxes_on_plane(3), lambda: E.scenes.spheres_in_box(4, 6, 4),
             lambda: E.scenes.mixed_pile(5, jitter=0.01), lambda: E.scenes.hinge_chains(2, 2)]
    out, t0 = [], time.time()
    if kind == "vsref":
        print(json.dumps(dict(results=free_run_against_real_stepper(E, O), seconds=0.0)))
        return
    for i in range(first, last):
        if kind == "beyond":
            make, rest = beyond[i]
            scene = make()
            res = over_the_limit(E, scene, steps, rest)
        elif kind == "large":
            scene = large[i]()
            res = lockstep(E, O, scene, steps, restitution, mode, env=env)
            res["large"], res["want"] = L.large_dynamic(scene["bodies"]).tolist(), scene["large"]
        else:
            scene = fixed[i]() if kind == "fixed" else (random_scene_wide if kind == "wide" else random_scene)(E, O, i)
            res = lockstep_with_mutations(E, O, scene, steps, i) if "--mutate" in sys.argv else lockstep(E, O, scene, steps, restitution, mode)
        res.pop("digests", None)
        res["scene"] = scene["name"]
        out.append(res)
    print(json.dumps(dict(results=out, seconds=time.time() - t0)))


if __name__ == "__main__":
    main()
