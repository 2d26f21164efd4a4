"""TEST INFRASTRUCTURE.  Builds tests/emu/_build/libb2d_emu.so: the library's CUDA sources compiled for the CPU emulation of
tests/emu/include/cuda_runtime.h.  The sources are used as they are except for what C++ cannot parse:
  * kernel<<<grid, block, smem, stream>>>(args)  ->  EMU_LAUNCH(kernel, grid, block, smem, stream, args)      (5 sites)
  * cudaLaunchCooperativeKernel(...)             ->  the same kernel on ONE block                             (1 site)
  * extern __shared__ T name[];                  ->  T *name = emu::dynamic_smem()                            (1 site)
  * the seven inline-PTX lines (acquire / relaxed polls, fences, prefetch, register pinning) -> plain loads / stores / no-ops,
    every poll yielding to the other fibers.
    python tests/emu/build.py        # g++ only, ~1 minute
"""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(ROOT, "edyn_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libb2d_emu.so")

ASM = [  # (substring identifying the line, replacement for the whole line)
    ('ld.acquire.gpu.global.u32', '            do { v = *(volatile unsigned *)ctr; if (v < target) emu::yield(); } while (v < target);'),
    ('fence.acq_rel.gpu', 'B2D_D void fence_gpu() {}'),
    ('void keep(float x)', 'B2D_D void keep(float) {}'),
    ('void keep(uint32_t x)', 'B2D_D void keep(uint32_t) {}'),
    ('asm volatile(B2D_LD_POLL', '    emu::yield(); return *p;'),
    ('asm volatile(B2D_ST_POLL', '    *p = v;'),
    ('prefetch.global.L2', 'B2D_D void prefetch_L2(const void *) {}'),
]


def transform(text, name):
    n_launch = len(re.findall(r"<<<", text))
    text = re.sub(r"(\w+)<<<(.*?)>>>\((.*?)\);", lambda m: f"EMU_LAUNCH({m.group(1)}, {m.group(2)}{', ' + m.group(3) if m.group(3).strip() else ''});", text)
    assert "<<<" not in text, f"{name}: a launch was not rewritten"
    text = re.sub(r"return cudaLaunchCooperativeKernel\(.*?\);", "emu::launch(kernel, dim3(1), dim3(threads), 0, args...); return cudaSuccess;", text)
    text = text.replace("__noinline__", "EMU_NOINLINE")
    text = re.sub(r"extern __shared__ (\w+) (\w+)\[\];", r"\1 *\2 = static_cast<\1 *>(emu::dynamic_smem());", text)
    lines, n_asm = text.split("\n"), 0
    for i, ln in enumerate(lines):
        if "asm volatile" in ln or "asm(" in ln:
            for key, repl in ASM:
                if key in ln:
                    lines[i] = repl
                    n_asm += 1
                    break
            else:
                raise SystemExit(f"{name}:{i + 1}: inline assembly without an emulation: {ln.strip()}")
    return "\n".join(lines), n_launch, n_asm


def build(force=False):
    srcs = [os.path.join(SRC, f) for f in sorted(os.listdir(SRC)) if f.endswith((".cu", ".cuh"))]
    deps = srcs + [os.path.join(HERE, "include", "cuda_runtime.h"), os.path.join(HERE, "include", "cooperative_groups.h"),
                   os.path.join(HERE, "include", "cub", "cub.cuh"), os.path.join(HERE, "emu_runtime.cpp"), os.path.abspath(__file__),
                   os.path.join(ROOT, "include", "b2d.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    gen = os.path.join(OUT, "src", "edyn_b200", "csrc")
    os.makedirs(gen, exist_ok=True)
    os.makedirs(os.path.join(OUT, "src", "include"), exist_ok=True)
    with open(os.path.join(ROOT, "include", "b2d.h")) as f, open(os.path.join(OUT, "src", "include", "b2d.h"), "w") as g:
        g.write(f.read())
    total = [0, 0]
    for s in srcs:
        text, nl, na = transform(open(s).read(), os.path.basename(s))
        total[0] += nl; total[1] += na
        dst = os.path.join(gen, os.path.basename(s).replace("b2d_api.cu", "b2d_api.cpp"))
        open(dst, "w").write(text)
    cxx = os.environ.get("CXX", "g++")
    cmd = [cxx, "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-DB2D_EMU",
           "-I" + os.path.join(HERE, "include"), os.path.join(gen, "b2d_api.cpp"), os.path.join(HERE, "emu_runtime.cpp"), "-o", LIB]
    subprocess.run(cmd, check=True)
    print(f"tests/emu: {total[0]} launch sites and {total[1]} inline-PTX lines rewritten -> {LIB}")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
