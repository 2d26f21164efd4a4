/*
 * b2d.h -- C ABI of the GPU-native Edyn step ("b2d": the project's original name).
 *
 * Drop-in boundary (SURVEY.md section 8b, DESIGN.md section 2).  The reference has no FFI; its boundary is
 * four C++ objects called in fixed order from
 *     edyn::stepper_sequential::update / step_simulation
 *         /root/reference/src/edyn/simulation/stepper_sequential.cpp:71-102, :121-147
 *             bphase.update(mt)        src/edyn/collision/broadphase.cpp:177
 *             nphase.update(mt)        src/edyn/collision/narrowphase.cpp:21
 *             m_island_manager.update  src/edyn/simulation/island_manager.cpp:533
 *             m_solver.update(mt)      src/edyn/dynamics/solver.cpp:387
 * A device world is "a simulation_worker whose registry lives in HBM": the host adapter
 * (edyn_b200/csrc/host/edyn_adapter.hpp for C++17/EnTT users, edyn_b200/world.py for Python) stages
 * components into the SoA arrays below, calls b2d_step(), and reads results back.
 *
 * Every function returns 0 on success or a negative b2d_status; b2d_last_error() gives the text.
 * Unsupported content is an error, never a CPU fallback.  All pointers are HOST pointers
 * (pinned memory recommended); arrays are densely packed float / uint32_t / uint64_t.
 * One world per registry; calls on one world are not re-entrant.
 */
#ifndef B2D_H
#define B2D_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* shape_index values of the reference (include/edyn/shapes/shapes.hpp:23-37). */
#define B2D_SHAPE_SPHERE  0u
#define B2D_SHAPE_CAPSULE 2u
#define B2D_SHAPE_BOX     3u
#define B2D_SHAPE_PLANE   6u
#define B2D_SHAPE_NONE    255u

/* rigidbody_kind (include/edyn/util/rigidbody.hpp): dynamic_tag / kinematic_tag / static_tag. */
#define B2D_DYNAMIC   0u
#define B2D_KINEMATIC 1u
#define B2D_STATIC    2u

/* contact_normal_attachment (include/edyn/collision/contact_normal_attachment.hpp:16-20). */
#define B2D_ATTACH_NONE 0u
#define B2D_ATTACH_A    1u
#define B2D_ATTACH_B    2u

/* b2d_bodies.material / b2d_body_patch.material values besides a material::id 0..0xFFFE (include/edyn/comp/material.hpp). */
#define B2D_MATERIAL_UNASSIGNED 0xFFFFu      /* material::UnassignedID: the body has a material without an id */
#define B2D_MATERIAL_NONE 0xFFFFFFFFu        /* no material component: the body is a sensor */

/* b2d_run_phases() mask: the four calls of stepper_sequential.cpp:82-91. */
#define B2D_PHASE_BROAD   1u
#define B2D_PHASE_NARROW  2u
#define B2D_PHASE_ISLANDS 4u
#define B2D_PHASE_SOLVE   8u
#define B2D_PHASE_ALL     15u

typedef enum b2d_status {
    B2D_OK = 0,
    B2D_ERR_CUDA = -1,         /* a CUDA runtime call failed */
    B2D_ERR_CAPACITY = -2,     /* max_bodies / max_manifolds / max_hinges exceeded */
    B2D_ERR_UNSUPPORTED = -3,  /* shape / constraint / setting outside the hot-path scope */
    B2D_ERR_ARGUMENT = -4
} b2d_status;

typedef struct b2d_world b2d_world;

/* edyn::init_config + settings (include/edyn/edyn.hpp:39-60, include/edyn/context/settings.hpp:21-57). */
typedef struct b2d_config {
    int32_t  device;               /* CUDA ordinal */
    uint32_t max_bodies;
    uint32_t max_manifolds;        /* device-resident contact manifolds (4 point slots each) */
    uint32_t max_hinges;
    float    fixed_dt;             /* settings.fixed_dt, default 1/60 */
    uint32_t velocity_iterations;  /* settings.num_solver_velocity_iterations, default 8 */
    uint32_t position_iterations;  /* settings.num_solver_position_iterations, default 3 */
    uint32_t flags;                /* B2D_FLAG_* */
} b2d_config;

#define B2D_FLAG_RECOLOR_EACH_STEP 1u  /* recompute the constraint colouring from scratch every step */
#define B2D_FLAG_RESTITUTION_SOLVER 4u /* settings.num_restitution_iterations = 8, num_individual_restitution_iterations = 3 (the
                                          reference's defaults, include/edyn/context/settings.hpp:29-30): the restitution solver
                                          (src/edyn/dynamics/restitution_solver.cpp:86-408) runs before gravity, the rows then carry no
                                          restitution.  Off = set_solver_restitution_iterations(0): restitution through the row rhs */
#define B2D_FLAG_SLEEPING 2u           /* island sleeping (src/edyn/simulation/island_manager.cpp:541-623).  Off = every
                                          body carries sleeping_disabled_tag, as the benchmark configurations prescribe */

/* make_rigidbody() output for n bodies (src/edyn/util/rigidbody.cpp:47-185), SoA.
 * inv_inertia = inertia_inv component, row-major 3x3 in body space (ignored unless dynamic).
 * gravity = gravity component (zero if absent).  group/mask may be NULL (= no collision_filter).
 * material: n values or NULL (= every body B2D_MATERIAL_UNASSIGNED).  A material id, B2D_MATERIAL_UNASSIGNED, or
 *   B2D_MATERIAL_NONE: an empty rigidbody_def::material, a sensor (util/collision_util.cpp:358-384,
 *   util/constraint_util.cpp:82-85).  A sensor's pairs get manifolds and contact points like any other pair, join and keep
 *   awake islands like them, but get no contact constraint: nothing pushes or bounces on a sensor, and its friction and
 *   restitution are not read.  Other values: B2D_ERR_ARGUMENT.
 * presentation: n values or NULL (= none).  Non-zero: the body has present_position and present_orientation
 *   (rigidbody_def::presentation, util/rigidbody.cpp:99-102), both starting at pos / orn.  make_rigidbody emplaces them on
 *   dynamic bodies only; a non-zero value on a kinematic or static body is accepted and that body is snapped by
 *   b2d_snap_presentation but never interpolated, as the reference's views would treat it. */
typedef struct b2d_bodies {
    uint32_t count;
    const float *pos;          /* 3n  position */
    const float *orn;          /* 4n  orientation x,y,z,w */
    const float *linvel;       /* 3n */
    const float *angvel;       /* 3n */
    const float *inv_mass;     /* n   mass_inv */
    const float *inv_inertia;  /* 9n  inertia_inv */
    const float *gravity;      /* 3n */
    const uint32_t *kind;      /* n   B2D_DYNAMIC.. */
    const uint32_t *shape_kind;/* n   B2D_SHAPE_.. */
    const float *shape_params; /* 4n  sphere{r} capsule{r,half_length,axis} box{half_extents} plane{n,constant} */
    const float *friction;     /* n   material.friction */
    const float *restitution;  /* n   material.restitution */
    const uint64_t *group;     /* n or NULL  collision_filter.group */
    const uint64_t *mask;      /* n or NULL  collision_filter.mask */
    const uint32_t *material;  /* n or NULL  material.id, B2D_MATERIAL_UNASSIGNED or B2D_MATERIAL_NONE (sensor) */
    const uint32_t *presentation; /* n or NULL  has present_position / present_orientation */
} b2d_bodies;

/* profile_counters + profile_timers analogue (include/edyn/context/profile.hpp:8-27). */
typedef struct b2d_stats {
    uint32_t bodies, manifolds, contact_points, hinges;
    uint32_t contact_colors, hinge_colors, islands, manifold_high_water;
    uint64_t kernel_launches;      /* kernels launched by this world since creation */
    uint64_t steps;
    float last_step_ms;            /* CUDA-event time of the last b2d_step() call */
    float solve_ms;                /* mean CUDA-event time of the velocity-solve kernel per step since b2d_reset_timers */
    float integrate_ms;            /* ... of the integrate kernel (means cover at most the last 256 steps) */
    uint32_t error_flags;          /* device-side overflow flags, 0 if none */
    /* Steps that ran the island rebuild (connected components, colouring, tile packing, solver order) and steps that
       reused the previous one because the constraint graph had not changed (CUDA graphs only; B2D_GRAPH_REUSE=0 turns
       reuse off).  kernel_launches counts the rebuild's kernels either way. */
    uint64_t steps_rebuilt, steps_reused;
} b2d_stats;

b2d_world  *b2d_create(const b2d_config *cfg);
void        b2d_destroy(b2d_world *w);
const char *b2d_last_error(const b2d_world *w);   /* w may be NULL: error of the last failed b2d_create */

/* Appends bodies; ids are consecutive, *first_id receives the id of bodies[0]. */
int b2d_add_bodies(b2d_world *w, const b2d_bodies *bodies, uint32_t *first_id);
/* make_constraint<hinge_constraint> + set_axes (src/edyn/constraints/hinge_constraint.cpp:11-17). */
int b2d_add_hinges(b2d_world *w, uint32_t n, const uint32_t *body_a, const uint32_t *body_b,
                   const float *pivot_a, const float *pivot_b, const float *axis_a, const float *axis_b);
/* registry.destroy(body): the body leaves the broadphase (src/edyn/collision/broadphase.cpp:54-68) and the entity graph
 * together with every manifold and joint attached to it (src/edyn/simulation/island_manager.cpp:47-66).  Ids are not
 * recycled; state downloads keep reporting the slot (as a static body without shape).  Used by island migration
 * between GPUs (SURVEY section 8e). */
int b2d_remove_bodies(b2d_world *w, const uint32_t *body_ids, uint32_t n);
/* wake_up_entity (src/edyn/util/island_util.cpp): clears sleeping_tag; the body's island follows at the next island
 * update.  ids == NULL wakes every body.  b2d_download_sleeping: 1 per body that carries sleeping_tag. */
int b2d_wake_bodies(b2d_world *w, const uint32_t *body_ids, uint32_t n);
int b2d_download_sleeping(b2d_world *w, uint32_t *asleep);
/* exclude_collision (src/edyn/util/exclude_collision.cpp): pairs that never collide. */
int b2d_add_exclusions(b2d_world *w, uint32_t n, const uint32_t *body_a, const uint32_t *body_b);
/* remove_collision_exclusion (src/edyn/util/exclude_collision.cpp); unknown pairs are ignored. */
int b2d_remove_exclusions(b2d_world *w, uint32_t n, const uint32_t *body_a, const uint32_t *body_b);

/* Dirty-subset staging (SURVEY.md section 8b): the reference's remote-replica contract -- users write through
 * registry.patch / replace and only the touched entities travel (include/edyn/comp/shared_comp.hpp:36-86,
 * include/edyn/replication/registry_operation_observer.hpp:49-82).  Arrays are packed per listed body (3n, 4n, ...);
 * a NULL array leaves that component untouched.  kind may change (dynamic <-> kinematic <-> static: a kinematic body
 * keeps its velocity but has no mass, src/edyn/dynamics/solver.cpp:101-147).  AABB and inertia_world_inv follow. */
typedef struct b2d_body_patch {
    const float *pos, *orn, *linvel, *angvel;   /* 3n 4n 3n 3n */
    const float *inv_mass, *inv_inertia;        /* n  9n */
    const float *gravity;                       /* 3n */
    const float *friction, *restitution;        /* n  n  */
    const uint32_t *kind;                       /* n  */
    const uint32_t *material;                   /* n  material.id; a change between B2D_MATERIAL_NONE and a material
                                                      (sensor <-> non-sensor) is B2D_ERR_UNSUPPORTED */
} b2d_body_patch;
int b2d_upload_bodies(b2d_world *w, uint32_t n, const uint32_t *body_ids, const b2d_body_patch *patch);

/* insert_material_mixing / material_mix_table::remove (util/insert_material_mixing.cpp:9-22, dynamics/material_mixing.hpp:36-80)
 * for n unordered id pairs (id0[i], id1[i]).  An insert overwrites an existing entry; removing an absent pair is ignored.
 * Ids >= 0xFFFF are B2D_ERR_ARGUMENT (the reference asserts on them).  When a contact point is created and both bodies
 * have materials, the entry of their two ids replaces the mixed friction sqrt(fA fB) and restitution min(rA, rB)
 * (collision_util.cpp:282-317); existing points keep theirs, as in the reference.  The table is per world: a host
 * framework that spreads a scene over several worlds (island hand-over) sets the same table on every one.
 * Known difference: whether the restitution solver (B2D_FLAG_RESTITUTION_SOLVER) treats a manifold as one with
 * restitution is evaluated every step from the table and the bodies' materials; the reference fixes it when the manifold
 * is created (constraint_util.cpp:90-101).  A table edit or a restitution patch reaches existing manifolds at once here,
 * only new ones in the reference. */
int b2d_set_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1, const float *friction,
                            const float *restitution);
int b2d_remove_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1);

/* n fixed steps: broadphase -> narrowphase -> islands -> solve/integrate (step_simulation semantics). */
int b2d_step(b2d_world *w, uint32_t num_steps);
/* Selected phases of ONE step, in stepper order (parity tests of individual phases). */
int b2d_run_phases(b2d_world *w, uint32_t phase_mask);

/* Overwrite position/orientation/linvel/angvel of ALL bodies from host arrays (full resync after the
 * user wrote components directly); AABB and inertia_world_inv are refreshed as solver.cpp:453-465 does. */
int b2d_upload_state(b2d_world *w, const float *pos, const float *orn, const float *linvel, const float *angvel);
/* Any output may be NULL.  aabb: 6 floats per body (min, max); inv_inertia_world: 9 per body. */
int b2d_download_state(b2d_world *w, float *pos, float *orn, float *linvel, float *angvel,
                       float *aabb, float *inv_inertia_world);

/* Contact manifolds (contact_manifold / contact_point*, include/edyn/collision/contact_point.hpp:17-58).
 * pairs: 2 uint32 per manifold (body[0], body[1]).  num: points per manifold.  Per point slot
 * (4 per manifold, list order, slot 0 = newest): pt18 = pivotA(3) pivotB(3) normal(3) local_normal(3)
 * distance friction restitution normal_impulse friction_impulse[2]; pt_u2 = {normal_attachment, lifetime}.
 * A point stores its attachment and lifetime in one 32-bit word: b2d_upload_contacts returns B2D_ERR_ARGUMENT for a
 * normal_attachment > 2 or a lifetime >= 2^30 in any of the first num slots.  The step counts a lifetime modulo 2^30
 * (about 207 days at 60 Hz) where the reference's uint32 would go on; nothing in the step reads it.
 * A sensor's points (B2D_MATERIAL_NONE on either body) have no contact_point_material and no contact_point_impulse: their
 * friction, restitution and impulses are reported as 0. */
int b2d_num_manifolds(b2d_world *w, uint32_t *n);
int b2d_download_pairs(b2d_world *w, uint32_t capacity, uint32_t *pairs, uint32_t *n);
int b2d_download_contacts(b2d_world *w, uint32_t capacity, uint32_t *pairs, uint32_t *num,
                          float *pt18, uint32_t *pt_u2, uint32_t *n);
/* Replaces all manifolds (solver-only and narrowphase-only parity tests; EnTT -> device mirroring). */
int b2d_upload_contacts(b2d_world *w, uint32_t n, const uint32_t *pairs, const uint32_t *num,
                        const float *pt18, const uint32_t *pt_u2);

/* island_resident analogue: label[i] = smallest body id of i's island, 0xFFFFFFFF for static/kinematic. */
int b2d_download_islands(b2d_world *w, uint32_t *label);
/* The sequential Gauss-Seidel order equivalent to the device's coloured solve in the last step:
 * hinge ids, then manifold body pairs.  Capacities in *nh / *nm on entry, counts on exit. */
int b2d_download_solver_order(b2d_world *w, uint32_t *hinge_ids, uint32_t *nh, uint32_t *pairs, uint32_t *nm);
/* applied_impulse.linear[3], .hinge[2] per hinge (constraints/hinge_constraint.hpp:63-70). */
int b2d_download_hinge_impulses(b2d_world *w, float *imp5);

int b2d_get_stats(b2d_world *w, b2d_stats *out);
/* Restart the per-kernel timing averages reported by b2d_get_stats. */
int b2d_reset_timers(b2d_world *w);
/* Development aid: raw copy of the device-side counter block (layout private to the library).  Not part of the reference-facing surface. */
int b2d_debug_counters(b2d_world *w, void *out, uint32_t bytes);
/* Development aid: the island tiles of the last step (DESIGN.md section 2): out6 = tiles, manifolds / hinges solved in
 * tiles, manifolds / hinges with rows, most bodies in one tile. */
int b2d_debug_tiles(b2d_world *w, uint32_t *out6);
/* Development aid: the new pairs the last broadphase counted per body (each pair at its query body), one word per body. */
int b2d_debug_newcount(b2d_world *w, uint32_t *counts);
/* Development aid: the island-tile packing of the last island rebuild, which later steps reuse while the constraint graph
 * is unchanged.  counts5 = tiles (two-point tiles first), two-point tiles, manifolds / hinges solved in tiles, tile
 * capacity of the world.  Each of the other outputs may be NULL: btile / bslot (one word per body: its tile and record
 * slot, 0xFFFFFFFF / 0xFFFF when it is not in a tile), tiles5 (5 x tiles words, row-major: bodies, then the
 * [c0, c1) and [h0, h1) ranges into the tiled constraints), tiled_pairs (2 x manifolds in tiles: the body pairs of the
 * tiled manifolds in that order), tiled_hinges (hinges in tiles: hinge ids in that order).  Call with NULLs first for
 * the sizes. */
int b2d_debug_tile_map(b2d_world *w, uint32_t *counts5, uint32_t *btile, uint32_t *bslot, uint32_t *tiles5,
                       uint32_t *tiled_pairs, uint32_t *tiled_hinges);
/* Multi-GPU exchange (SURVEY.md section 8e): enqueue, on the world's stream, the reduction of all dynamic AABBs into
 * device_out8 = {min xyz, max xyz, speed, 0} -- a DEVICE pointer (e.g. a buffer owned by the host framework) the adapter
 * then all-gathers over NCCL to detect island groups of different ranks coming within the broadphase margin of each
 * other.  speed = the fastest any point of any dynamic body moves (|v| + |w| r, m/s): an adapter that overlaps the
 * exchange with the next step widens its margins by what the bodies can travel in that step. */
int b2d_device_bounds(b2d_world *w, float *device_out8);
/* Distance below which an island counts as touching a peer's box / island in b2d_island_halo and b2d_handover_plan
 * (never below the manifold separation threshold 0.026, broadphase.hpp:18, which is the default). */
int b2d_set_halo_margin(b2d_world *w, float margin);
/* ---- Island hand-over between the worlds of different GPUs (SURVEY.md section 8e).  The host framework owns the
 * transport (NCCL send/recv of DEVICE buffers); every payload is produced and consumed on the device.
 *   b2d_set_entities   scene-global name per body (the entt::entity of the EnTT binding); default = local id.
 *   b2d_island_halo    update_island_aabbs (src/edyn/sys/update_aabbs.cpp:106-138) on the device, then the islands whose
 *                      AABB, inflated by the manifold separation threshold, reaches into the box of a peer in peer_mask
 *                      are appended to device_records: 8 words each {min xyz, max xyz, island label, self}.
 *                      device_boxes: nboxes x 6 floats (the all-gathered b2d_device_bounds of all ranks).
 *   b2d_handover_plan  device_records = the halo records of ALL ranks concatenated in rank order, [my_begin, my_end)
 *                      being this world's.  An island that touches an island of a lower rank moves there, whole
 *                      (merge_islands: "move into the other island", src/edyn/simulation/island_manager.cpp:297-350).
 *                      counts: nranks x 4 = bodies, manifolds, joints, exclusions leaving for each rank (host array).
 *   b2d_handover_pack  everything rank dst needs to continue those islands -- body components with their current state,
 *                      manifolds with points, lifetimes and warm-start impulses, joints, exclusions, all named by
 *                      entity -- into device_blob (b2d_handover_bytes(counts + 4 * dst) bytes); the local copies are
 *                      destroyed (b2d_remove_bodies semantics).
 *   b2d_handover_unpack  appends a received blob; counts_out (4 words, may be NULL) = what it held. */
int b2d_set_entities(b2d_world *w, uint32_t first_body, uint32_t n, const uint32_t *entity);
int b2d_download_entities(b2d_world *w, uint32_t *entity);
int b2d_island_halo(b2d_world *w, const float *device_boxes, uint32_t nboxes, uint32_t self, uint64_t peer_mask,
                    void *device_records, uint32_t capacity, uint32_t *device_count);
int b2d_handover_plan(b2d_world *w, const void *device_records, uint32_t my_begin, uint32_t my_end, uint32_t nranks,
                      uint32_t *counts);
uint64_t b2d_handover_bytes(const uint32_t *counts4);
int b2d_handover_pack(b2d_world *w, uint32_t dst, void *device_blob, uint64_t capacity);
int b2d_handover_unpack(b2d_world *w, const void *device_blob, uint64_t bytes, uint32_t *counts_out);

/* ---- Raycast: edyn::raycast(registry, p0, p1, ignore_entities) (include/edyn/collision/raycast.hpp:157-168,
 * src/edyn/collision/raycast.cpp:20-56) for a batch of n segments p0[i] -> p1[i] (3 floats each).
 *   Candidates  every body with a shape that is not removed and not ignored: dynamic, kinematic, static and sleeping.
 *   Hit         the reference's shape_raycast (raycast.cpp:58-109 box, :182-195 sphere, :197-257 capsule, :356-378 plane)
 *               gives a fraction f per body; it counts if 0 <= f <= 1 (NaN never does).  The answer is the body with the
 *               smallest f; equal fractions (==) go to the smaller body id.  So the result is the brute-force minimum over
 *               all candidates, whatever the spatial index does.  fraction, normal and feature are the reference's bits,
 *               except the capsule hemisphere normal: normalize(lerp(p0, p1, f) - hemisphere centre).  Consequences: a
 *               segment that starts inside a sphere reports it at 0; one that starts inside a box or a capsule's side
 *               reports nothing from that body; a zero-length segment, or one with a non-finite coordinate, hits nothing.
 *   State       what every step, upload, add or remove enqueued before it on the world's stream left, with the AABBs
 *               b2d_download_state returns.  A raycast writes nothing a step reads.
 *   Output      body: local id or B2D_RAY_MISS; fraction: FLT_MAX on a miss; normal: 3 floats, zero on a miss (NaN
 *               where the reference's is: a segment through a sphere's centre or a capsule's axis);
 *               feature: box face 0-5 (box_raycast_info), capsule hemisphere 0 / 1 or B2D_RAY_CAPSULE_SIDE
 *               (capsule_raycast_info), B2D_RAY_FEATURE_NONE for spheres, planes and misses.  Any output may be NULL.
 *   Ignoring    ignore_list: nignore body ids ignored by every segment (host array, may be NULL when nignore = 0);
 *               ignore_body: n ids, one per segment (e.g. the agent casting it), or NULL.
 * b2d_raycast takes and returns HOST arrays and returns when the results are there.  b2d_raycast_device takes DEVICE
 * pointers for p0 .. feature (ignore_list stays a host array) and only enqueues the work on b2d_stream(w). */
#define B2D_RAY_MISS 0xFFFFFFFFu
#define B2D_RAY_FEATURE_NONE 0xFFFFFFFFu
#define B2D_RAY_CAPSULE_SIDE 2u
int b2d_raycast(b2d_world *w, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body,
                const uint32_t *ignore_list, uint32_t nignore, uint32_t *body, float *fraction, float *normal, uint32_t *feature);
int b2d_raycast_device(b2d_world *w, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body,
                       const uint32_t *ignore_list, uint32_t nignore, uint32_t *body, float *fraction, float *normal,
                       uint32_t *feature);

/* ---- Presentation transforms: update_presentation / snap_presentation (src/edyn/sys/update_presentation.cpp:56-93), which
 * stepper_sequential::update runs after its steps (src/edyn/simulation/stepper_sequential.cpp:37-43, :104-105).  Only bodies
 * added with a non-zero b2d_bodies.presentation have the two components; they live on the device next to the state.
 *   b2d_update_presentation  for every body with presentation that is dynamic and not sleeping:
 *                            present_position = pos + linvel * interpolation_dt,
 *                            present_orientation = integrate(orn, angvel, interpolation_dt) (math/quaternion.cpp:7-22).
 *                            The caller computes interpolation_dt as the reference does: min(float(time - fixed_dt -
 *                            sim_time), fixed_dt), usually negative.  Sleeping, kinematic and static bodies keep theirs.
 *   b2d_snap_presentation    for every body with presentation: present_position = pos, present_orientation = orn (what
 *                            update() does while paused).
 * Both only enqueue work on b2d_stream(w); no step reads or writes the presentation.
 *   b2d_download_presentation         pos3n / orn4n: HOST arrays (either may be NULL, not both); returns when they are filled.
 *   b2d_download_presentation_device  the same into DEVICE pointers (e.g. a graphics-interop buffer the caller
 *                                     owns); only enqueues on b2d_stream(w).
 * In both downloads a body without presentation reports its current pos / orn, and a removed body what
 * b2d_download_state reports for it. */
int b2d_update_presentation(b2d_world *w, float interpolation_dt);
int b2d_snap_presentation(b2d_world *w);
int b2d_download_presentation(b2d_world *w, float *pos3n, float *orn4n);
int b2d_download_presentation_device(b2d_world *w, float *device_pos3n, float *device_orn4n);

/* Per-kernel CUDA-event timing of the velocity solve and the integrator (b2d_get_stats).  On (default): a step is
 * replayed as three CUDA graphs with the events in between; off: as one graph. */
int b2d_set_timing(b2d_world *w, int enabled);
/* Blocks until all queued device work of this world has finished; device-side overflow flags (b2d_stats.error_flags)
 * come back as B2D_ERR_CAPACITY / B2D_ERR_UNSUPPORTED / B2D_ERR_CUDA with the text in b2d_last_error. */
int b2d_sync(b2d_world *w);
/* The CUDA stream (cudaStream_t) the world launches on, for event timing by the caller. */
void *b2d_stream(b2d_world *w);

#ifdef __cplusplus
}
#endif
#endif /* B2D_H */
