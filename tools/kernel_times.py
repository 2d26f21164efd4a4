"""Per-kernel device time of one simulation step of a bench.py workload, from torch.profiler (CUPTI).

    python tools/kernel_times.py WORKLOAD [--steps N] [--warmup W] [--graph]
                                 [--velocity-iterations V] [--position-iterations P] --out DIR

The scene is built and settled as bench.py does it (same generator, capacity and settle steps).  The step time is
taken first with CUDA events and the profiler off; then N steps run under torch.profiler with CUDA activities and
every kernel's summed duration is divided by N.  By default the world steps without its CUDA graph (B2D_GRAPH=0), so
every kernel is its own launch in the trace and the island rebuild runs on every step; kernel durations do not depend
on that, the gaps between them do.  --graph replays the step graph as bench.py does: the rebuild's kernels then only
appear on the steps that ran it (the header gives how many did).  --velocity-iterations / --position-iterations
replace the workload's solver settings (settling included), so the difference of two runs is the cost of the
iterations left out; the files then carry the setting in their name (_v<V>, _p<P>).

Writes DIR/kernel_times_<WORKLOAD>.txt (table, largest first) and DIR/kernel_times_<WORKLOAD>.json."""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--graph", action="store_true", help="step through the CUDA graph (island rebuild reuse on)")
    ap.add_argument("--velocity-iterations", type=int, help="override the workload's velocity iterations")
    ap.add_argument("--position-iterations", type=int, help="override the workload's position iterations")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.environ["B2D_GRAPH"] = "1" if args.graph else "0"

    import torch
    import edyn_b200 as E
    from torch.profiler import profile, ProfilerActivity

    scene = bench.make_scene(args.workload)
    override = {}
    if args.velocity_iterations is not None:
        override["velocity_iterations"] = args.velocity_iterations
    if args.position_iterations is not None:
        override["position_iterations"] = args.position_iterations
    w = E.scenes.build_world(scene, device=0, max_manifolds=bench.capacity(args.workload, len(scene["bodies"]["kind"])),
                             **override)
    iters = dict(scene["settings"], **override)
    tag = "".join(f"_{k[0]}{override[k]}" for k in ("velocity_iterations", "position_iterations") if k in override)
    w.step(bench.SETTLE_STEPS)
    w.step(args.warmup)
    w.sync()

    stream = torch.cuda.ExternalStream(w.stream, device=0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    w.step(args.steps)
    e1.record(stream)
    w.sync()
    step_ms = e0.elapsed_time(e1) / args.steps

    st0 = w.stats()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        w.step(args.steps)
        w.sync()
    per = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name.split("(")[0].split("<")[0] or ev.name
        per[name][0] += 1
        per[name][1] += ev.time_range.elapsed_us()
    st = w.stats()
    w.close()
    if not per:
        raise SystemExit("kernel_times: the profiler recorded no device activity")

    rows = sorted(((n, c / args.steps, us / args.steps) for n, (c, us) in per.items()), key=lambda r: -r[2])
    total_us = sum(r[2] for r in rows)
    gpu = torch.cuda.get_device_name(0)
    rebuilt = st["steps_rebuilt"] - st0["steps_rebuilt"]
    mode = "CUDA graph" if args.graph else "no graph"
    head = (f"{args.workload} on {gpu}: {args.steps} profiled steps after {bench.SETTLE_STEPS} + {args.warmup} untimed; "
            f"step {step_ms * 1e3:.1f} us (CUDA events, profiler off, {mode}); island rebuild on {rebuilt} of the {args.steps} "
            f"profiled steps; {iters['velocity_iterations']} velocity / {iters['position_iterations']} position iterations; "
            f"kernels {total_us:.1f} us per step; "
            f"{st['contact_points']} contact points, {st['hinges']} hinges, {st['manifolds']} manifolds")
    lines = [head, f"{'us/step':>10} {'%kern':>6} {'launches':>8}  kernel"]
    lines += [f"{us:10.1f} {100 * us / total_us:6.1f} {c:8.1f}  {n}" for n, c, us in rows]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"kernel_times_{args.workload}{tag}.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    with open(os.path.join(args.out, f"kernel_times_{args.workload}{tag}.json"), "w") as f:
        json.dump({"workload": args.workload, "gpu": gpu, "graph": args.graph, "steps": args.steps, "steps_rebuilt": rebuilt, "step_us": step_ms * 1e3, "kernel_us": total_us,
                   "velocity_iterations": iters["velocity_iterations"], "position_iterations": iters["position_iterations"],
                   "kernels": [{"name": n, "launches_per_step": c, "us_per_step": us} for n, c, us in rows]}, f, indent=1)
    print("\n".join(lines))


if __name__ == "__main__":
    main()
