"""ctypes binding of libb2d.so (include/b2d.h).  No fallback: a missing library or GPU is a hard error."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2D_LIB") or os.path.join(HERE, "libb2d.so")     # B2D_LIB: development builds
SRC = os.path.join(HERE, "csrc", "b2d_api.cu")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
              "-Xcompiler", "-fPIC", "-shared"]


class B2DError(RuntimeError):
    pass


def build(force=False):
    """nvcc cross-compiles the whole CUDA path for sm_90a into edyn_b200/libb2d.so (in-tree)."""
    srcs = [os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc")) if f.endswith((".cu", ".cuh"))]
    srcs.append(os.path.join(HERE, "..", "include", "b2d.h"))
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(s) <= os.path.getmtime(LIB_PATH) for s in srcs):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    subprocess.run([nvcc] + NVCC_FLAGS + ["-o", LIB_PATH, SRC], check=True)
    return LIB_PATH


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_bodies", C.c_uint32), ("max_manifolds", C.c_uint32),
                ("max_hinges", C.c_uint32), ("fixed_dt", C.c_float), ("velocity_iterations", C.c_uint32),
                ("position_iterations", C.c_uint32), ("flags", C.c_uint32)]


class Bodies(C.Structure):
    _fields_ = [("count", C.c_uint32)] + [(n, C.c_void_p) for n in (
        "pos", "orn", "linvel", "angvel", "inv_mass", "inv_inertia", "gravity", "kind", "shape_kind",
        "shape_params", "friction", "restitution", "group", "mask", "material", "presentation")]


class BodyPatch(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("pos", "orn", "linvel", "angvel", "inv_mass", "inv_inertia", "gravity",
                                          "friction", "restitution", "kind", "material")]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("bodies", "manifolds", "contact_points", "hinges", "contact_colors",
                                         "hinge_colors", "islands", "manifold_high_water")] + \
               [("kernel_launches", C.c_uint64), ("steps", C.c_uint64), ("last_step_ms", C.c_float),
                ("solve_ms", C.c_float), ("integrate_ms", C.c_float), ("error_flags", C.c_uint32),
                ("steps_rebuilt", C.c_uint64), ("steps_reused", C.c_uint64)]


EXPORTS = ["b2d_create", "b2d_destroy", "b2d_last_error", "b2d_add_bodies", "b2d_remove_bodies", "b2d_wake_bodies", "b2d_download_sleeping", "b2d_add_hinges", "b2d_add_exclusions", "b2d_remove_exclusions",
           "b2d_step", "b2d_run_phases", "b2d_upload_state", "b2d_download_state", "b2d_num_manifolds",
           "b2d_download_pairs", "b2d_download_contacts", "b2d_upload_contacts", "b2d_download_islands",
           "b2d_download_solver_order", "b2d_download_hinge_impulses", "b2d_get_stats", "b2d_reset_timers", "b2d_debug_counters", "b2d_debug_tiles", "b2d_debug_newcount", "b2d_debug_tile_map", "b2d_device_bounds", "b2d_set_halo_margin", "b2d_sync", "b2d_stream",
           "b2d_upload_bodies", "b2d_set_entities", "b2d_download_entities", "b2d_island_halo", "b2d_handover_plan",
           "b2d_handover_bytes", "b2d_handover_pack", "b2d_handover_unpack", "b2d_set_timing", "b2d_raycast", "b2d_raycast_device",
           "b2d_set_material_mixing", "b2d_remove_material_mixing", "b2d_update_presentation", "b2d_snap_presentation",
           "b2d_download_presentation", "b2d_download_presentation_device"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B2DError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`. "
                           "There is no CPU fallback.")
        l = C.CDLL(LIB_PATH)
        l.b2d_create.restype = C.c_void_p
        l.b2d_create.argtypes = [C.POINTER(Config)]
        l.b2d_destroy.argtypes = [C.c_void_p]
        l.b2d_last_error.restype = C.c_char_p
        l.b2d_last_error.argtypes = [C.c_void_p]
        l.b2d_stream.restype = C.c_void_p
        l.b2d_stream.argtypes = [C.c_void_p]
        l.b2d_handover_bytes.restype = C.c_uint64
        l.b2d_handover_bytes.argtypes = [C.c_void_p]
        _lib = l
    return _lib
