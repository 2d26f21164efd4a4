"""How much resident warps and register spills are worth to the island-tile kernel, on one GPU call.

    python tools/tile_residency.py --out DIR [--workload chains_1048576]

Builds three variants of the tree's library into a temporary directory and times the tile kernel of each with
tools/kernel_times.py --graph (B2D_LIB selects the build):
  tree    the sources as they are;
  cap128  -DB2D_TILE_CAP=128 and __launch_bounds__(TILE_CAP, 4) on the tile kernels: 128-lane tiles at the same
          register cap, so the same warps per SM hold twice as many independent tiles;
  lb1     __launch_bounds__(TILE_CAP, 1): half the resident warps, but no register cap and no spills.
For each it prints ptxas's resources for the tile kernels and the occupancy API's resident CTAs / warps per SM
(tools/tile_occupancy.cu, built with the same switches), then the card, its power limit and SM clocks.
Writes DIR/tile_residency.json and DIR/<variant>/kernel_times_<workload>.{txt,json}."""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from edyn_b200 import _lib  # noqa: E402

NVCC = os.environ.get("NVCC", "nvcc")
TILE_BOUNDS = re.compile(r"__launch_bounds__\(TILE_CAP, 2\)(\s+k_island_tiles)")     # the tree's bound of the tile kernels


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    if not shutil.which("nvidia-smi"):
        return "nvidia-smi not found"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or r.stderr.strip()


def source_tree(tmp, name, min_blocks):
    """A copy of the sources (csrc, include, tools/tile_occupancy.cu); with min_blocks, the tile kernels' launch bounds
    ask for that many resident CTAs per SM."""
    top = os.path.join(tmp, name)
    shutil.copytree(os.path.join(ROOT, "edyn_b200", "csrc"), os.path.join(top, "edyn_b200", "csrc"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(top, "include"))
    os.makedirs(os.path.join(top, "tools"))
    shutil.copy(os.path.join(ROOT, "tools", "tile_occupancy.cu"), os.path.join(top, "tools"))
    if min_blocks:
        k = os.path.join(top, "edyn_b200", "csrc", "b2d_kernels.cuh")
        src = open(k).read()
        new, n = TILE_BOUNDS.subn(rf"__launch_bounds__(TILE_CAP, {min_blocks})\1", src)
        if n == 0:
            raise SystemExit("tile_residency: no `__launch_bounds__(TILE_CAP, 2) k_island_tiles` to change")
        open(k, "w").write(new)
    return top


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--workload", default="chains_1048576")
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    variants = [("tree", [], None), ("cap128", ["-DB2D_TILE_CAP=128"], 4), ("lb1", [], 1)]
    res = {"workload": args.workload, "gpu_before": gpu_info(), "variants": {}}
    print("gpu:", res["gpu_before"], flush=True)
    with tempfile.TemporaryDirectory(prefix="tile_residency_") as tmp:
        jobs = []
        for name, defs, min_blocks in variants:
            top = source_tree(tmp, name, min_blocks)
            lib = os.path.join(tmp, f"libb2d_{name}.so")
            occ = os.path.join(tmp, f"occ_{name}")
            flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared",)]
            jobs.append((name, lib, occ, subprocess.Popen(
                [NVCC] + _lib.NVCC_FLAGS + defs + ["-Xptxas", "-v", "-o", lib, os.path.join(top, "edyn_b200", "csrc", "b2d_api.cu")],
                stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True),
                subprocess.Popen([NVCC] + [f for f in flags if f not in ("-Xcompiler", "-fPIC")] + defs + ["-o", occ, os.path.join(top, "tools", "tile_occupancy.cu")],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        for name, lib, occ, p_lib, p_occ in jobs:
            log, olog = p_lib.communicate()[0], p_occ.communicate()[0]
            if p_lib.returncode or p_occ.returncode:
                raise SystemExit(f"tile_residency: build of {name} failed\n{log[-4000:]}\n{olog[-4000:]}")
            lines = log.splitlines()
            ptx = []
            for i, l in enumerate(lines):
                m = re.search(r"Function properties for (_ZN3b2d\d*k_island_tiles\S*)", l)
                if m and i + 2 < len(lines):
                    ptx.append(f"{m.group(1)}: {lines[i + 1].strip()}; {lines[i + 2].split(':', 1)[1].strip()}")
            o = subprocess.run([occ], capture_output=True, text=True)
            v = {"ptxas": ptx, "occupancy": (o.stdout + o.stderr).strip()}
            res["variants"][name] = v
            for line in ptx + v["occupancy"].splitlines():
                print(f"[{name}] {line}", flush=True)
        for name, lib, _, _, _ in jobs:
            odir = os.path.join(args.out, name)
            env = dict(os.environ, B2D_LIB=lib)
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "kernel_times.py"), args.workload, "--graph",
                                "--steps", str(args.steps), "--out", odir], env=env, capture_output=True, text=True)
            if r.returncode:
                raise SystemExit(f"tile_residency: kernel_times for {name} failed\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
            kt = json.load(open(os.path.join(odir, f"kernel_times_{args.workload}.json")))
            tiles = {k["name"]: k["us_per_step"] for k in kt["kernels"] if "island_tiles" in k["name"]}
            res["variants"][name].update({"step_us": kt["step_us"], "tile_kernels_us": tiles})
            print(f"[{name}] step {kt['step_us']:.1f} us, " + ", ".join(f"{k} {us:.1f} us" for k, us in tiles.items()), flush=True)
    res["gpu_after"] = gpu_info()
    print("gpu:", res["gpu_after"])
    with open(os.path.join(args.out, "tile_residency.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
