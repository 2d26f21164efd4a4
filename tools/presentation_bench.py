"""Cost of the presentation transforms on the benchmark workloads (include/b2d.h b2d_update_presentation).

    python tools/presentation_bench.py [--workloads chains_1048576,mixed_262144] [--calls 200] [--steps 30] [--out DIR]

Each workload is built as bench.py builds it, with presentation on every dynamic body, and stepped --steps times.  Then,
with CUDA events on the world's stream, the mean time per call of:
  * update_ms      b2d_update_presentation alone;
  * update_dev_ms  b2d_update_presentation followed by b2d_download_presentation_device into torch CUDA tensors
                   (a frame that never leaves the GPU);
  * snap_ms        b2d_snap_presentation;
and, on the host clock, host_ms: b2d_update_presentation + b2d_download_presentation into host arrays (blocking).
bytes_per_body gives the traffic the kernel needs with the float4 layout: 68 B read and 32 B written per interpolated
body, 28 B more written per body for the packed device output.  Prints one JSON line with the card's name and power limit
read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.raycast_bench import card  # noqa: E402


def events_ms(torch, stream, fn, calls):
    s = torch.cuda.ExternalStream(stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        fn()
    e0.record(s)
    for _ in range(calls):
        fn()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def run(name, calls, steps):
    import torch
    import bench
    import edyn_b200 as E
    scene = bench.make_scene(name)
    b = dict(scene["bodies"], presentation=(scene["bodies"]["kind"] == 0).astype(np.uint32))
    n = len(b["kind"])
    w = E.scenes.build_world(dict(scene, bodies=b), max_manifolds=bench.capacity(name, n))
    w.set_timing(False)
    w.step(steps)
    w.sync()
    pos = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    orn = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    dt = -1.0 / 120
    upd = events_ms(torch, w.stream, lambda: w.update_presentation(dt), calls)
    dev = events_ms(torch, w.stream, lambda: (w.update_presentation(dt), w.presentation_device(pos.data_ptr(), orn.data_ptr())), calls)
    snap = events_ms(torch, w.stream, w.snap_presentation, calls)
    w.presentation()
    hcalls = max(5, calls // 10)
    t0 = time.perf_counter()
    for _ in range(hcalls):
        w.update_presentation(dt)
        w.presentation()
    host = (time.perf_counter() - t0) * 1e3 / hcalls
    dyn = int(b["presentation"].sum())
    nbytes = dyn * (68 + 32) + (n - dyn) * 4
    w.close()
    return dict(workload=name, bodies=n, presented=dyn, update_ms=round(upd, 4), update_dev_ms=round(dev, 4),
                snap_ms=round(snap, 4), host_ms=round(host, 3), update_GBps=round(nbytes / upd / 1e6, 1),
                bytes_per_body=dict(update=100, snap=68, device_output=28))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="chains_1048576,mixed_262144")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card(), results=[run(n, a.calls, a.steps) for n in a.workloads.split(",")])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "presentation_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
