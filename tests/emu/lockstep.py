"""TEST INFRASTRUCTURE.  The command-line driver of the CPU emulation (tests/emu): the library's CUDA kernels, executed by
the emulation, in lock step with the oracle through the normal Python adapter and C ABI -- the comparison of
tests/parity.py, which the -m gpu tests make on the GPU (here everything is bit-identical, the trig set's poses and
contact normals included: glibc's sinf / cosf on both sides).

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

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.parity import build_world, lockstep  # noqa: E402


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


def mutations(E, scene, seed, events):
    """before(step, world, oracle) for `lockstep`: user code interferes every 13th step with b2d_remove_bodies,
    b2d_remove_exclusions, b2d_add_bodies or b2d_upload_bodies (a patched velocity), on both sides; each is appended to
    `events`.  Needs room for 16 more bodies."""
    import numpy as np
    R = E.rigidbody
    rng = np.random.default_rng(seed)
    nb = len(scene["bodies"]["kind"])
    kind = np.asarray(scene["bodies"]["kind"]).copy()
    alive = np.ones(len(kind), bool)
    excluded = list(zip(*[x.tolist() for x in scene["exclusions"]])) if scene["exclusions"] is not None else []

    def before(s, w, o):
        nonlocal kind, alive
        if not s or s % 13:
            return o
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
        events.append((s, int(what)))
        return o
    return before


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
    os.environ["B2D_EMU"] = "1"            # tests/parity.py: nothing is exempt from bit equality
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
            if "--mutate" in sys.argv:
                events = []
                res = lockstep(E, O, scene, steps, restitution, mode, before=mutations(E, scene, i, events),
                               max_bodies=len(scene["bodies"]["kind"]) + 16)
                res["events"] = len(events)
            else:
                res = lockstep(E, O, scene, steps, restitution, mode)
        res.pop("digests", None)
        res["scene"] = scene["name"]
        out.append(res)
    print(json.dumps(dict(results=out, seconds=time.time() - t0)))


if __name__ == "__main__":
    main()
