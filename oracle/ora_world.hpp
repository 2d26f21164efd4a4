// TEST INFRASTRUCTURE -- CPU oracle (see ora_math.hpp header).
// World state + one fixed step of the sequential stepper restated without EnTT:
//   src/edyn/simulation/stepper_sequential.cpp:71-102  (order of phases)
//   src/edyn/collision/broadphase.cpp:119-195, src/edyn/collision/narrowphase.cpp:21-40,
//   include/edyn/util/collision_util.hpp:105-276, src/edyn/dynamics/solver.cpp:387-468,
//   src/edyn/dynamics/island_solver.cpp:76-111,263-376,521-543.
// Also restated: island sleeping (island_manager.cpp:541-623) and the restitution solver
// (dynamics/restitution_solver.cpp:86-408; off unless restitution_iters > 0 -- the device path and the benchmark
// configurations run with restitution iterations = 0, restitution through the row rhs).
// Not restated (out of scope, SURVEY.md section 2): center_of_mass/origin offsets, contact_extras.
// PINNED: leaf functions against the reference's object code (tests/test_oracle_fixtures.py), whole steps bit for bit
// against the reference's real stepper_sequential (oracle/_ref/libedyn_stepper.so, tests/test_ref_stepper.py and
// tests/golden/whole_step.npz) with the reference's row order replayed through set_point_order().
#pragma once
#include "ora_collide.hpp"
#include <unordered_map>
#include <unordered_set>
#include <algorithm>
#include <cmath>
#include <vector>

namespace ora {

enum body_kind : uint32_t { BK_DYNAMIC = 0, BK_KINEMATIC = 1, BK_STATIC = 2 };

struct Body {
    vec3 pos; quat orn;
    vec3 linvel, angvel, dv, dw;
    scalar inv_m;
    mat3 inv_I, inv_IW;
    vec3 gravity;
    shape sh;
    aabb bb;
    uint32_t kind;
    scalar friction, restitution;
    bool rolling;            // rolling_tag: dynamic sphere/cylinder/capsule (util/rigidbody.cpp:120-130)
    bool has_filter; uint64_t group, mask;
    bool asleep = false;     // sleeping_tag (island_manager.cpp:541-566): excluded from every per-step view
    bool procedural() const { return kind == BK_DYNAMIC; }
    bool awake() const { return kind == BK_DYNAMIC && !asleep; }
};

struct Point {               // contact_point + _geometry + _material + _impulse (collision/contact_point.hpp:17-58)
    vec3 pivotA, pivotB, normal, local_normal;
    scalar distance;
    uint32_t att;
    scalar friction, restitution;
    uint32_t lifetime;
    scalar imp_n, imp_t[2];
};

struct Manifold {            // contact_manifold + state; pt[0] is the linked-list head (newest point)
    uint32_t a, b;
    uint32_t num;
    Point pt[4];
};

// Branches of process_collision (World::narrowphase), one bit each in World::merge_trace when trace_merge is on.  Test
// infrastructure: tests/golden/make_merge.py samples cases until each branch is covered, and the merge tests assert that
// coverage on the cases they run.  "Slot" is a point's position in the list when the step starts (the device's storage
// slot), "index" its position once the removals of the first pass closed the gaps.
enum merge_branch : uint32_t {
    MB_SETTLED,             // persisted points present, every result point merged into one in the first pass
    MB_EARLY_RETURN,        // no persisted point, empty result
    MB_EMPTY_KEEP,          // empty result, a persisted point kept (distance updated)
    MB_EMPTY_REMOVE,        // empty result, a persisted point removed
    MB_NEAREST_A,           // merged into the result point nearest through pivot A
    MB_NEAREST_B,           // ... through pivot B
    MB_ROLL_A,              // merged through the rolling search on body A
    MB_ROLL_B,              // ... on body B (pivotB, B's pose, the result's pivotA)
    MB_ROLL_BOTH,           // both bodies rolling: B's search ran after A's found nothing
    MB_TAKEN,               // the nearest result point was already merged: falls through to the removal test
    MB_REMOVE_NORMAL,       // removed: separation along the normal
    MB_REMOVE_TANGENT,      // removed: tangential drift only
    MB_REMOVE_FIRST,        // removed slot 0 of 2+ points
    MB_REMOVE_MIDDLE,       // removed a slot between the first and the last
    MB_REMOVE_LAST,         // removed the last slot of 2+ points
    MB_REMOVE_GAP,          // removed two slots with a kept one between them
    MB_REMOVE_ALL4,         // removed all of 4 points
    MB_KEPT,                // unmatched point kept, distance updated
    MB_INS1_APPEND, MB_INS1_SIMILAR,
    MB_INS2_APPEND, MB_INS2_SIMILAR, MB_INS2_REPLACE0, MB_INS2_REPLACE1, MB_INS2_NONE,
    MB_INS3_NONE,           // in the triangle
    MB_INS3_APPEND,
    MB_INS3_COL1, MB_INS3_COL0, MB_INS3_COL2, MB_INS3_SHORTEST,     // collinear triple: replace index 1, 0, 2, shortest edge
    MB_INS4_SIMILAR, MB_INS4_REPLACE0, MB_INS4_REPLACE1, MB_INS4_REPLACE2, MB_INS4_REPLACE3, MB_INS4_NONE,
    MB_PIVOT_B,             // pivots B tried after pivots A found no place, and found one
    MB_SIMILAR_INPLACE,     // SIMILAR onto a persisted point that stays in its slot
    MB_SIMILAR_MOVED,       // SIMILAR onto a persisted point that changes slot (with its impulse)
    MB_SIMILAR_CREATED,     // SIMILAR onto a point inserted this pass: created
    MB_REPLACE_PERSISTED,   // REPLACE of a persisted point
    MB_REPLACE_AFTER_GAP,   // ... that sat after a removed slot
    MB_REPLACE_THEN_SIMILAR,// one index of the list written twice in one pass: REPLACE, then SIMILAR
    MB_SIMILAR_THEN_REPLACE,//                                                     SIMILAR, then REPLACE
    MB_FULL4,               // the rearranged list holds 4 points
    MB_MOVE_UP,             // a persisted point moves to a later slot
    MB_MOVE_DOWN,           // ... to an earlier slot
    MB_MOVE_BOTH,           // both in one manifold
    MB_COUNT
};

struct Hinge {               // constraints/hinge_constraint.hpp:22-93 without limits/springs/torque
    uint32_t a, b;
    vec3 pivot[2];
    mat3 frame[2];
    scalar imp_lin[3], imp_hinge[2];
};

struct World {
    scalar dt = scalar(1.0 / 60);
    int vel_iters = 8, pos_iters = 3;          // context/settings.hpp:22-30
    std::vector<Body> bodies;
    std::vector<Manifold> manifolds;
    std::vector<Hinge> hinges;
    std::unordered_map<uint64_t, uint32_t> manifold_map;   // contact_manifold_map
    std::unordered_set<uint64_t> exclusions;               // collision_exclusion (pair form)
    std::vector<uint32_t> island;                           // label per body (min procedural id), ~0u if none
    // Sleeping (island_manager.cpp:541-623, thresholds config/constants.hpp:41-48).  Off by default = every body
    // carries sleeping_disabled_tag, which is what the benchmark configurations prescribe.
    bool sleeping_enabled = false;
    uint64_t updates = 0;                                   // island_manager::update calls so far
    std::vector<uint32_t> prev_island;                      // label of the previous update (~0u: none)
    std::vector<uint32_t> isl_size;                         // per previous label: number of procedural bodies
    std::vector<double> isl_sleep_ts;                       // per previous label: island::sleep_timestamp, < 0 = unset
    void update_sleep();
    void wake_body(uint32_t i) { bodies[i].asleep = false; }
    bool trace_merge = false;                               // record merge_trace in the next narrowphase
    std::vector<uint64_t> merge_trace;                      // per manifold: bit b = merge_branch b was taken
    // Optional injected Gauss-Seidel order (see ora_api.cpp: ora_set_order).
    bool use_order = false;
    std::vector<uint32_t> hinge_order;
    std::vector<uint64_t> manifold_order;                   // pair keys
    bool position_contacts_first = false;                   // position iterations: sweep contacts before joints (GCC argument order, see step())
    std::vector<uint32_t> point_order;                      // optional, one per entry of manifold_order: which point of the manifold's list
                                                            // the row is (0xFFFFFFFF = all its points, in list order)
    int threads = 1;                                        // island-parallel solve (run_island_solver_seq_mt analogue)
    // Which body of a new pair becomes body[0] = which of the two issues its broadphase query first = iteration order of
    // view<AABB, procedural_tag> (broadphase.cpp:183), i.e. of the procedural_tag pool: newest first.  Without removals
    // that is descending body index (default, and what the device does).  registry.destroy(body) is a swap-and-pop in
    // the pool -- the newest body takes the removed one's place in the iteration -- which proc_pool reproduces when
    // emulate_pool_order is on (comparisons with the real stepper after bodies were destroyed).
    bool emulate_pool_order = false;
    std::vector<uint32_t> proc_pool;                        // packed array of the procedural_tag pool
    // Restitution solver (dynamics/restitution_solver.cpp:86-408; settings.hpp:29-30: 8 iterations by default in the
    // reference, 0 here = restitution goes through the row rhs).  It walks the entity graph breadth first, so its result
    // depends on the graph's adjacency order and on island.edges order; both are supplied by the caller
    // (ora_set_graph_order): adj_off / adj_nbr = per body the neighbours in adjacency-list order, bit 31 set when the
    // adjacency holds a contact manifold; rest_edge_order = the manifolds tagged contact_manifold_with_restitution in
    // island.edges iteration order (pair keys).  Without them: ascending neighbour id / manifold order.
    int restitution_iters = 0, individual_restitution_iters = 3;
    std::vector<uint32_t> adj_off, adj_nbr;
    std::vector<uint64_t> rest_edge_order;
    bool graph_order_set = false;
    void solve_restitution();
    scalar manifold_min_relvel(const Manifold &m) const;
    void solve_restitution_group(const std::vector<uint32_t> &group);
    bool restitution_iteration(const std::vector<uint32_t> &tagged);

    static uint64_t key(uint32_t a, uint32_t b) { return a < b ? (uint64_t(a) << 32) | b : (uint64_t(b) << 32) | a; }

    uint32_t add_body(const Body &b);
    void remove_body(uint32_t i);              // registry.destroy(body): broadphase.cpp:54-68, island_manager.cpp:47-66
    void refresh_body(uint32_t i);             // AABB + inv_IW from current transform
    void broadphase();
    void narrowphase();
    void islands();
    void solve();
    void step() { broadphase(); narrowphase(); islands(); solve(); }      // islands() ends with update_sleep()
    bool should_collide(uint32_t a, uint32_t b) const;
};

// dynamics/material_mixing.hpp:12-18
inline scalar material_mix_restitution(scalar a, scalar b) { return std::min(a, b); }
inline scalar material_mix_friction(scalar a, scalar b) { return std::sqrt(a * b); }

// Row-level helpers exposed for pinning against the reference's constraint_row.cpp
struct Row {
    vec3 J[4];
    scalar eff_mass, rhs, lo, hi, impulse;
};
void prepare_row(Row &row, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                 scalar error, scalar erp, scalar restitution, vec3 vA, vec3 wA, vec3 vB, vec3 wB);
scalar solve_row(Row &row, vec3 dvA, vec3 dwA, vec3 dvB, vec3 dwB);
mat3 moment_of_inertia(const shape &sh, scalar mass);
// constraint_row_friction (constraints/constraint_row_friction.hpp:12-24) and its two functions, pinned against the
// reference's solve_friction / warm_start (constraint_row_friction.cpp:11-66) by tests/test_oracle_fixtures.py
struct FrictionPair { vec3 J[2][4]; scalar eff_mass[2], rhs[2], impulse[2]; scalar mu; };
// contact_constraint::prepare (constraints/contact_constraint.cpp:15-56): builds the normal row (not yet passed through
// prepare_row: `error` and the point's restitution are what constraint_row_options would carry) and the friction pair.
// Pinned against the reference's own object code by tests/test_oracle_fixtures.py.
void prepare_contact(const Point &cp, scalar dt, vec3 posA, quat ornA, vec3 posB, quat ornB,
                     vec3 vA, vec3 wA, scalar inv_mA, const mat3 &inv_IA, vec3 vB, vec3 wB, scalar inv_mB, const mat3 &inv_IB,
                     Row &normal_row, scalar &error, FrictionPair &f);
// position_solver::solve (dynamics/position_solver.hpp:16-51) and contact_constraint::solve_position
// (contact_constraint.cpp:58-90) on two bodies; returns false when the point is not penetrating (nothing solved)
extern bool position_renormalize_all;   // position_solver.hpp:26-32 also normalises non-procedural bodies' orientation: off by default
void position_solve(Body &A, Body &B, const vec3 J[4], scalar error, scalar &max_error);
bool contact_solve_position(Point &cp, Body &A, Body &B, scalar &max_error);
void hinge_solve_position(const Hinge &hc, Body &A, Body &B, scalar &max_error);   // hinge_constraint.cpp:180-213
// the three decisions process_collision takes per persisted point (util/collision_util.cpp:233-280, :397-413), pinned
// against the reference functions cut out of that unit at build time
size_t find_nearest_contact(const Point &cp, const cresult &res, bool *via_B = nullptr);
size_t find_nearest_contact_rolling(const cresult &res, vec3 cp_pivot, vec3 origin, quat orn, vec3 angvel, scalar dt);
bool should_remove_point(const Point &cp, vec3 posA, quat ornA, vec3 posB, quat ornB);
void solve_friction(FrictionPair &f, scalar normal_impulse, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                    vec3 &dvA, vec3 &dwA, vec3 &dvB, vec3 &dwB);
void warm_start_friction(const FrictionPair &f, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                         vec3 &dvA, vec3 &dwA, vec3 &dvB, vec3 &dwB);

} // namespace ora
