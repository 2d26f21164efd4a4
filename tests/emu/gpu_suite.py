"""TEST INFRASTRUCTURE / development aid.  Runs the `-m gpu` tests that do not need torch's CUDA tensors against the CPU
emulation (tests/emu) instead of a GPU: the kernels' logic, the C ABI, the Python adapter, the C++ EnTT binding.

    python tests/emu/gpu_suite.py [extra pytest args]

Not run: the full-size configs and the 1000-step box stack (hours under emulation), the hand-over tests (their payloads live
in torch CUDA tensors), the NCCL tests, the C++ adapter's hello_world (links libb2d.so by name).
State at the end of round 2: 32 tests, all green (the same tests were green on a GPU before the last kernel clean-up;
tests/test_zz_gpu_stepper_b2d.py has only ever run here).  The tile-edge, random and large-body lock-step files run here with
fewer steps and seeds and without their CUDA-graph mode (the emulation launches plainly)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

SELECT = "not full_size and not box_stacks_1000 and not spheres_65536 and not two_gpus and not nccl and not two_ranks_on_one_device " \
         "and not chain_handover and not cpp_hello_world and not free_running_steps"


def main():
    from tests.emu import build
    lib = build.build()
    if os.path.isdir("/root/reference/include/edyn"):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "integration"), "emu"], check=True)
    os.environ.update(B2D_EMU="1", B2D_LIB=lib, B2D_GRAPH="0")
    import pytest
    import tests.test_stepper_b2d as T
    real_load = T.load

    def load(O, variant):                  # the binding harness linked against the emulation instead of libb2d.so
        if variant != "dev":
            return real_load(O, variant)
        saved, T.BUILD = T.BUILD, os.path.join(HERE, "_build")
        try:
            return real_load(O, "emu")
        finally:
            T.BUILD = saved
    T.load = load
    import tests.test_zz_gpu_stepper_b2d as Z
    Z.load = load
    files = [os.path.join(ROOT, "tests", f) for f in ("test_gpu_parity.py", "test_gpu_dist.py", "test_gpu_handover.py", "test_zz_gpu_stepper_b2d.py",
                                                      "test_gpu_tile_edges.py", "test_gpu_random_lockstep.py", "test_gpu_large_bodies.py",
                                                      "test_gpu_merge.py", "test_gpu_point_transitions.py", "test_gpu_broadphase_edges.py")]
    return pytest.main(["-q", "-m", "gpu", "-k", SELECT, "-p", "no:cacheprovider"] + files + sys.argv[1:])


if __name__ == "__main__":
    sys.exit(main())
