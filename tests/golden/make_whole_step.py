"""Regenerates tests/golden/whole_step.npz: trajectories of the reference's OWN stepper_sequential
(/root/reference/src/edyn/simulation/stepper_sequential.cpp:71-102, compiled unmodified into oracle/_ref/libedyn_stepper.so
against oracle/entt_lite -- `make -C oracle stepper`) on five small scenes of the four BASELINE workload families, with
the order in which its island solver swept the constraint rows every step (dynamics/island_solver.cpp:181-222 walks
island.edges; that order is EnTT pool order after entity_graph traversals, so it is recorded rather than re-derived).

    python tests/golden/make_whole_step.py          # needs /root/reference at build time; the .npz travels, the reference does not

Consumer: tests/test_ref_stepper.py::test_oracle_replays_reference_trajectories (CPU, runs without the library).
It also writes tests/golden/free_run.npz, the reference's free-running end states that the device (and its CPU emulation)
is compared with: tests/test_zz_gpu_stepper_b2d.py, tests/test_emu_device.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

STEPS = 120
KEEP_EVERY = 10
# name -> (edyn_b200.scenes factory, args)
SCENES = {
    "hello_world": ("hello_world", ()),
    "boxes_27": ("boxes_on_plane", (3,)),
    "spheres_96": ("spheres_in_box", (4, 6, 4)),
    "mixed_125": ("mixed_pile", (5,)),
    "chains_16": ("hinge_chains", (2, 2)),
}
SCENE_KW = {"mixed_125": {"jitter": 0.01}}
# free_run.npz: the reference's state, nothing replayed, after the listed step counts.  name -> (factory, args, steps)
FREE_RUN = {
    "chains_64": ("hinge_chains", (4, 4), (60, 300)),
    "hello_world": ("hello_world", (), (24,)),
    "chains_256": ("hinge_chains", (8, 8), (1000,)),
}
FREE_RUN_PATH = os.path.join(ROOT, "tests", "golden", "free_run.npz")


def free_run_scene(E, name):
    fn, a, _ = FREE_RUN[name]
    return getattr(E.scenes, fn)(*a)


def reference_free_run(name, step):
    """pos and linvel of the scene's dynamic bodies after `step` free-running steps of the reference's own stepper."""
    g = np.load(FREE_RUN_PATH)
    return {k: g[f"{name}.{step}.{k}"] for k in ("pos", "linvel")}


def build_scene(E, name):
    fn, a = SCENES[name]
    return getattr(E.scenes, fn)(*a, **SCENE_KW.get(name, {}))


def populate(world, scene):
    world.add_bodies(scene["bodies"])
    if scene["hinges"]:
        h = scene["hinges"]
        world.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    if scene["exclusions"] is not None:
        world.add_exclusions(*scene["exclusions"])


def main():
    import edyn_b200 as E
    from oracle import oracle as O
    O.build()
    assert O.ref_stepper() is not None, "oracle/_ref/libedyn_stepper.so missing: make -C oracle stepper"
    out = {}
    for name in SCENES:
        scene = build_scene(E, name)
        st = scene["settings"]
        r = O.RefWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"])
        populate(r, scene)
        oh, oc, oh_off, oc_off, kept = [], [], [0], [0], []
        for s in range(STEPS):
            r.step(1)
            hi, ct = r.solver_order()
            oh.append(np.asarray(hi, np.uint32).reshape(-1)); oc.append(np.asarray(ct, np.uint32).reshape(-1, 3))
            oh_off.append(oh_off[-1] + len(oh[-1])); oc_off.append(oc_off[-1] + len(oc[-1]))
            if (s + 1) % KEEP_EVERY == 0:
                x = r.state()
                kept.append(np.concatenate([x["pos"], x["orn"], x["linvel"], x["angvel"]], axis=1))
        c = r.contacts()
        out[f"{name}.order_h"] = np.concatenate(oh) if oh else np.zeros(0, np.uint32)
        out[f"{name}.order_c"] = np.concatenate(oc)
        out[f"{name}.order_h_off"] = np.asarray(oh_off, np.uint32)
        out[f"{name}.order_c_off"] = np.asarray(oc_off, np.uint32)
        out[f"{name}.states"] = np.stack(kept)                               # (STEPS / KEEP_EVERY, bodies, 13)
        out[f"{name}.final_pairs"] = c["pairs"]
        out[f"{name}.final_num"] = c["num"]
        out[f"{name}.islands"] = r.islands()
        print(f"{name}: {r.num_bodies} bodies, {oc_off[-1]} contact rows and {oh_off[-1]} joint rows over {STEPS} steps, "
              f"{int(c['num'].sum())} points at the end")
    out["steps"] = np.asarray([STEPS, KEEP_EVERY], np.uint32)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "whole_step.npz"), **out)
    write_free_run(E, O)


def write_free_run(E, O):
    free = {}
    for name, (_, _, marks) in FREE_RUN.items():
        scene = free_run_scene(E, name)
        st = scene["settings"]
        r = O.RefWorld(vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"])
        populate(r, scene)
        n, done = scene["dynamic"], 0
        for m in marks:
            r.step(m - done); done = m
            x = r.state()
            free[f"{name}.{m}.pos"], free[f"{name}.{m}.linvel"] = x["pos"][:n].copy(), x["linvel"][:n].copy()
    np.savez_compressed(FREE_RUN_PATH, **free)


if __name__ == "__main__":
    main()
