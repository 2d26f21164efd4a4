"""Raycast throughput on the benchmark workloads (include/b2d.h b2d_raycast).

    python tools/raycast_bench.py [--rays 1048576] [--reps 10] [--workloads a,b] [--out DIR]

Each workload is settled as bench.py does (150 steps), then, with CUDA events on the world's stream:
  * build_ms  -- the raycast index (k_bp_cells into the index's own buffers, k_ray_classify, the key sort, cell starts),
                 rebuilt after one more step each repetition;
  * down / across -- casts of --rays segments through the device-pointer path (b2d_raycast_device): short downward probes
                 from above the scene, and horizontal segments across the whole scene;
  * host_ms   -- the same downward batch through the host-array path (b2d_raycast: copies in, cast, copies out; wall clock).
A CPU arm times the reference's own edyn::raycast (tests/raycast/ref_raycast.cpp) on the 4 096 boxes of boxes_4096, where
the reference's object files exist (--cpu-only runs just that arm, without a GPU).
Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception as e:  # noqa: BLE001
        return [f"unknown ({e})"]


def bounds(st, kind):
    dyn = np.asarray(kind) == 0
    bb = st["aabb"][:len(dyn)][dyn]
    return bb[:, :3].min(0), bb[:, 3:].max(0)


def device_arm(E, name, nrays, reps):
    import torch
    import bench as B
    scene = B.make_scene(name)
    n = len(scene["bodies"]["kind"])
    w = E.scenes.build_world(scene, max_manifolds=B.capacity(name, n))
    w.step(B.SETTLE_STEPS)
    w.sync()
    lo, hi = bounds(w.download_state(), scene["bodies"]["kind"])
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(w.stream, device=0)
    res = dict(bodies=n)

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); fn(); b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)

    build = []
    for _ in range(reps):
        w.step(1)
        w.sync()
        build.append(timed(lambda: w.raycast_device(0, 0, 0)))
    res["build_ms"] = float(np.median(build))
    out = [torch.empty(nrays, dtype=torch.int32, device=dev), torch.empty(nrays, dtype=torch.float32, device=dev),
           torch.empty((nrays, 3), dtype=torch.float32, device=dev), torch.empty(nrays, dtype=torch.int32, device=dev)]
    for kind in ("down", "across"):
        p0, p1 = E.scenes.raycast_segments(lo, hi, nrays, kind=kind, seed=1)
        t0, t1 = torch.from_numpy(p0).to(dev), torch.from_numpy(p1).to(dev)
        torch.cuda.synchronize()
        cast = lambda: w.raycast_device(nrays, t0.data_ptr(), t1.data_ptr(), *[o.data_ptr() for o in out])   # noqa: E731
        timed(cast)                                                               # warm-up
        ms = [timed(cast) for _ in range(reps)]
        hit = float((out[0] != -1).float().mean().item())
        res[kind] = dict(ms=float(np.median(ms)), spread_ms=float(np.max(ms) - np.min(ms)),
                         rays_per_s=nrays / (float(np.median(ms)) * 1e-3), hit_fraction=hit)
        if kind == "down":
            w.raycast(p0, p1)
            host = []
            for _ in range(max(3, reps // 2)):
                t = time.perf_counter(); w.raycast(p0, p1); host.append((time.perf_counter() - t) * 1e3)
            res["host_ms"] = float(np.median(host))
            res["host_rays_per_s"] = nrays / (res["host_ms"] * 1e-3)
    assert w.stats()["error_flags"] == 0
    w.close()
    return res


def cpu_reference_arm(E, nrays):
    """edyn::raycast itself (the reference's dynamic AABB trees, tests/raycast/ref_raycast.cpp), one segment per call, one
    thread, on the boxes_4096 bodies at their starting positions (a 16 x 16 x 16 grid, all static).  Runs where the
    reference's object files exist (oracle/_ref/edyn_obj, built where /root/reference is); the host CPU is reported."""
    from tests import raycast_support as S
    import bench as B
    import platform
    if S.ref() is None:
        return dict(skipped="the reference's object files (oracle/_ref/edyn_obj) are not available")
    scene = B.make_scene("boxes_4096")
    b = scene["bodies"]
    rw = S.RefWorld(b["pos"], b["orn"], b["shape_kind"], b["shape_params"])
    dyn = np.asarray(b["kind"]) == 0
    pos = np.asarray(b["pos"], np.float32)[dyn]
    p0, p1 = E.scenes.raycast_segments(pos.min(0) - 0.5, pos.max(0) + 0.5, nrays, kind="down", seed=1)
    hits = 0
    t = time.perf_counter()
    for i in range(nrays):
        hits += int(rw.raycast(p0[i], p1[i])[0] != S.MISS)
    dt = time.perf_counter() - t
    rw.close()
    cpu = next((ln.split(":", 1)[1].strip() for ln in open("/proc/cpuinfo") if ln.startswith("model name")), platform.processor())
    return dict(bodies=len(b["kind"]), rays=nrays, s=dt, rays_per_s=nrays / dt, hit_fraction=hits / nrays, threads=1, cpu=cpu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--workloads", default="boxes_4096,spheres_65536,mixed_262144,chains_1048576")
    ap.add_argument("--cpu-rays", type=int, default=1 << 15)
    ap.add_argument("--cpu-only", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import edyn_b200 as E
    res = dict(card=None if args.cpu_only else card(), rays=args.rays, workloads={})
    for name in ([] if args.cpu_only else args.workloads.split(",")):
        res["workloads"][name] = device_arm(E, name, args.rays, args.reps)
    res["cpu_reference_boxes_4096"] = cpu_reference_arm(E, args.cpu_rays)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raycast_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
