"""edyn_b200 -- H100-native replacement for Edyn's per-step rigid-body hot path.

Host adapter (this package) -> C ABI (include/b2d.h, edyn_b200/libb2d.so) -> hand-written sm_90a kernels
(edyn_b200/csrc).  See DESIGN.md.  Importing this package never imports oracle/.
"""
from ._lib import B2DError, build  # noqa: F401
from .rigidbody import (DYNAMIC, KINEMATIC, MATERIAL_NONE, MATERIAL_UNASSIGNED, STATIC, Material, RigidBodyDef, Shape, bodies_soa, box_shape,  # noqa: F401
                        capsule_shape, plane_shape, sphere_shape)
from .world import (RAY_CAPSULE_SIDE, RAY_FEATURE_NONE, RAY_MISS, RaycastResult, World, attach,  # noqa: F401
                    clear_collision_exclusion, detach, exclude_collision, insert_material_mixing, make_hinge, make_rigidbody, raycast,
                    remove_collision_exclusion, set_paused, step_simulation, update)
from . import scenes  # noqa: F401
