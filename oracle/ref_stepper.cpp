// TEST INFRASTRUCTURE.  The reference's REAL sequential stepper -- edyn::attach / make_rigidbody /
// make_constraint<hinge_constraint> / exclude_collision / step_simulation, every translation unit compiled where it lies
// under /root/reference -- behind a small C interface, built against oracle/entt_lite (a from-scratch stand-in for the
// EnTT 3.15 dependency, which this image does not have).  Used as the whole-step oracle for oracle/ (tests/) and as the
// CPU baseline "reference" arm of bench.py.  Nothing under edyn_b200/ links or loads it.
// The restitution solver's result depends on orders inside the entity graph at the moment solver::update starts, so
// refs_step_begin / refs_step_end run stepper_sequential::step_simulation (stepper_sequential.cpp:121-147) in two halves;
// that needs its three members, hence the access hack on this ONE header (object layout is unaffected).
// refs_seed_manifolds / refs_narrowphase / refs_get_seeded run the reference's narrowphase alone on manifolds with given
// points (tests/golden/make_merge.py).
#define private public
#include <edyn/simulation/stepper_sequential.hpp>
#undef private
#include <edyn/edyn.hpp>
#include <edyn/util/rigidbody.hpp>
#include <edyn/util/constraint_util.hpp>
#include <edyn/util/exclude_collision.hpp>
#include <edyn/util/contact_manifold_util.hpp>
#include <edyn/constraints/hinge_constraint.hpp>
#include <edyn/collision/contact_manifold.hpp>
#include <edyn/collision/contact_point.hpp>
#include <edyn/collision/collision_result.hpp>
#include <edyn/util/collision_util.hpp>
#include <edyn/comp/position.hpp>
#include <edyn/comp/orientation.hpp>
#include <edyn/comp/linvel.hpp>
#include <edyn/comp/angvel.hpp>
#include <edyn/comp/aabb.hpp>
#include <edyn/comp/inertia.hpp>
#include <edyn/comp/island.hpp>
#include <edyn/comp/graph_node.hpp>
#include <edyn/core/entity_graph.hpp>
#include <edyn/collision/broadphase.hpp>
#include <edyn/collision/narrowphase.hpp>
#include <edyn/comp/tag.hpp>
#include <edyn/context/settings.hpp>
#include <edyn/dynamics/island_constraint_entities.hpp>
#include <edyn/constraints/constraint.hpp>
#include <edyn/constraints/contact_constraint.hpp>
#include <edyn/util/tuple_util.hpp>
#include <entt/entity/registry.hpp>
#include <cstdint>
#include <cstring>
#include <memory>
#include <optional>
#include <vector>

// Two entry points of the networking layer that the asynchronous stepper's translation units mention; the networking
// sources are not part of this build and the sequential stepper never calls them.
#include <edyn/networking/util/snap_to_pool_snapshot.hpp>
#include <edyn/networking/util/process_extrapolation_result.hpp>
#include <cstdio>
#include <cstdlib>
namespace edyn {
void snap_to_pool_snapshot(entt::registry &, const entity_map &, const std::vector<entt::entity> &, const std::vector<pool_snapshot> &, bool) {
    std::fputs("libedyn_stepper: networking code reached (snap_to_pool_snapshot)\n", stderr); std::abort();
}
void process_extrapolation_result(entt::registry &, entity_map &, const extrapolation_result &) {
    std::fputs("libedyn_stepper: networking code reached (process_extrapolation_result)\n", stderr); std::abort();
}
}

namespace {
struct World {
    entt::registry registry;
    std::vector<entt::entity> bodies, hinges;
    std::vector<entt::entity> seeded;                       // manifolds made by refs_seed_manifolds, in argument order
    double time = 0.0, dt = 1.0 / 60;
    uint64_t steps = 0;
};
edyn::vector3 v3(const float *p) { return {p[0], p[1], p[2]}; }
}

#define REFS_API extern "C" __attribute__((visibility("default")))

// threads == 0: execution_mode::sequential; threads > 0: sequential_multithreaded with that many workers
REFS_API void *refs_create(float dt, int vel_iters, int pos_iters, int restitution_iters, int threads) {
    auto *w = new World();
    w->dt = dt;
    edyn::init_config cfg;
    cfg.fixed_dt = dt;
    cfg.execution_mode = threads > 0 ? edyn::execution_mode::sequential_multithreaded : edyn::execution_mode::sequential;
    cfg.num_worker_threads = threads > 0 ? size_t(threads) : 0;
    cfg.timestamp = 0.0;
    edyn::attach(w->registry, cfg);
    auto &s = w->registry.ctx().get<edyn::settings>();
    s.num_solver_velocity_iterations = unsigned(vel_iters);
    s.num_solver_position_iterations = unsigned(pos_iters);
    s.num_restitution_iterations = unsigned(restitution_iters);
    edyn::set_paused(w->registry, true);                    // steps are driven one at a time (stepper_sequential.cpp:121-147)
    return w;
}
REFS_API void refs_destroy(void *h) {
    auto *w = static_cast<World *>(h);
    edyn::detach(w->registry);
    delete w;
}
// same SoA as b2d_add_bodies (include/b2d.h): kind 0 dynamic / 1 kinematic / 2 static; shape kinds 0 sphere{r}, 2 capsule{r, half_length, axis},
// 3 box{half extents}, 6 plane{normal, constant}, 255 none.  Inertia is left to make_rigidbody (moment_of_inertia of the shape).
REFS_API int refs_add_bodies(void *h, uint32_t n, const float *pos, const float *orn, const float *lv, const float *av, const float *inv_mass,
                             const float *gravity, const uint32_t *kind, const uint32_t *shape_kind, const float *sp,
                             const float *friction, const float *restitution, const uint64_t *group, const uint64_t *mask, int sleeping_disabled) {
    auto *w = static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) {
        edyn::rigidbody_def def;
        def.kind = kind[i] == 0 ? edyn::rigidbody_kind::rb_dynamic : (kind[i] == 1 ? edyn::rigidbody_kind::rb_kinematic : edyn::rigidbody_kind::rb_static);
        def.position = v3(pos + 3 * i);
        def.orientation = {orn[4 * i], orn[4 * i + 1], orn[4 * i + 2], orn[4 * i + 3]};
        def.linvel = v3(lv + 3 * i); def.angvel = v3(av + 3 * i);
        if (kind[i] == 0) def.mass = edyn::scalar(1) / inv_mass[i];
        def.gravity = v3(gravity + 3 * i);
        const float *p = sp + 4 * i;
        switch (shape_kind[i]) {
        case 0: def.shape = edyn::sphere_shape{p[0]}; break;
        case 2: def.shape = edyn::capsule_shape{p[0], p[1], static_cast<edyn::coordinate_axis>(int(p[2]))}; break;
        case 3: def.shape = edyn::box_shape{edyn::vector3{p[0], p[1], p[2]}}; break;
        case 6: def.shape = edyn::plane_shape{edyn::vector3{p[0], p[1], p[2]}, p[3]}; break;
        case 255: break;
        default: return -1;
        }
        edyn::material m; m.friction = friction[i]; m.restitution = restitution[i];
        def.material = m;
        if (group) def.collision_group = group[i];
        if (mask) def.collision_mask = mask[i];
        def.presentation = false;
        def.sleeping_disabled = sleeping_disabled != 0;
        w->bodies.push_back(edyn::make_rigidbody(w->registry, def));
    }
    return 0;
}
REFS_API int refs_add_hinges(void *h, uint32_t n, const uint32_t *a, const uint32_t *b, const float *pivA, const float *pivB, const float *axA, const float *axB) {
    auto *w = static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) {
        if (a[i] >= w->bodies.size() || b[i] >= w->bodies.size()) return -1;
        const auto pa = v3(pivA + 3 * i), pb = v3(pivB + 3 * i), xa = v3(axA + 3 * i), xb = v3(axB + 3 * i);
        w->hinges.push_back(edyn::make_constraint<edyn::hinge_constraint>(w->registry, w->bodies[a[i]], w->bodies[b[i]], [&](edyn::hinge_constraint &c) {
            c.pivot[0] = pa; c.pivot[1] = pb; c.set_axes(xa, xb);
        }));
    }
    return 0;
}
REFS_API int refs_add_exclusions(void *h, uint32_t n, const uint32_t *a, const uint32_t *b) {
    auto *w = static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) edyn::exclude_collision(w->registry, w->bodies[a[i]], w->bodies[b[i]]);
    return 0;
}
REFS_API void refs_step(void *h, uint32_t n) {
    auto *w = static_cast<World *>(h);
    // step j carries the time stepper_sequential::update would give it: sim_time + fixed_dt * i, i.e. j * fixed_dt counted
    // from the attach time 0 (stepper_sequential.cpp:71-75); only island sleeping looks at it (island_manager.cpp:605-623)
    for (uint32_t i = 0; i < n; ++i) { w->time = double(w->steps++) * w->dt; edyn::step_simulation(w->registry, w->time); }
}
// step_simulation in two halves: everything up to and including island_manager.update, then solver.update and the callbacks
REFS_API void refs_step_begin(void *h) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    auto &stepper = r.ctx().get<edyn::stepper_sequential>();
    w->time = double(w->steps++) * w->dt;
    stepper.m_last_time = w->time;
    auto &settings = r.ctx().get<edyn::settings>();
    if (settings.pre_step_callback) (*settings.pre_step_callback)(r);
    stepper.m_poly_initializer.init_new_shapes();
    r.ctx().get<edyn::broadphase>().update(stepper.m_multithreaded);
    r.ctx().get<edyn::narrowphase>().update(stepper.m_multithreaded);
    stepper.m_island_manager.update(stepper.m_last_time);
}
REFS_API void refs_step_end(void *h) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    auto &stepper = r.ctx().get<edyn::stepper_sequential>();
    auto &settings = r.ctx().get<edyn::settings>();
    stepper.m_solver.update(stepper.m_multithreaded);
    if (settings.clear_actions_func) (*settings.clear_actions_func)(r);
    if (settings.post_step_callback) (*settings.post_step_callback)(r);
}
// The orders the restitution solver walks (restitution_solver.cpp:108-124, :352-381): adj_off / adj_nbr = per body its
// neighbours in the entity graph's adjacency-list order (bit 31: the adjacency holds a contact manifold); tagged = the
// manifolds with contact_manifold_with_restitution in island.edges iteration order, island after island, as ordered pairs.
REFS_API int refs_get_graph_order(void *h, uint32_t *adj_off, uint32_t cap_adj, uint32_t *adj_nbr, uint32_t cap_tagged, uint32_t *tagged_pairs, uint32_t *n_tagged) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    auto &graph = r.ctx().get<edyn::entity_graph>();
    std::vector<uint32_t> body_of;
    for (size_t i = 0; i < w->bodies.size(); ++i) { const auto k = entt::to_entity(w->bodies[i]); if (k >= body_of.size()) body_of.resize(k + 1, 0xFFFFFFFFu); body_of[k] = uint32_t(i); }
    uint32_t n = 0;
    for (size_t i = 0; i < w->bodies.size(); ++i) {
        adj_off[i] = n;
        if (!r.valid(w->bodies[i])) continue;
        const auto node0 = r.get<edyn::graph_node>(w->bodies[i]).node_index;
        bool overflow = false;
        graph.visit_neighbors(node0, [&](entt::entity other) {
            if (n >= cap_adj) { overflow = true; return; }
            const auto node1 = r.get<edyn::graph_node>(other).node_index;
            bool has_manifold = false;
            graph.visit_edges(node0, node1, [&](auto edge_index) { if (r.all_of<edyn::contact_manifold>(graph.edge_entity(edge_index))) has_manifold = true; });
            adj_nbr[n++] = body_of[entt::to_entity(other)] | (has_manifold ? 0x80000000u : 0u);
        });
        if (overflow) return -1;
    }
    adj_off[w->bodies.size()] = n;
    uint32_t t = 0;
    for (auto [island_entity, island] : r.view<edyn::island>().each()) {
        for (auto e : island.edges) {
            if (!r.all_of<edyn::contact_manifold_with_restitution>(e)) continue;
            if (t >= cap_tagged) return -1;
            const auto &m = r.get<edyn::contact_manifold>(e);
            tagged_pairs[2 * t] = body_of[entt::to_entity(m.body[0])]; tagged_pairs[2 * t + 1] = body_of[entt::to_entity(m.body[1])];
            ++t;
        }
    }
    *n_tagged = t;
    return 0;
}
REFS_API uint32_t refs_num_bodies(void *h) { return uint32_t(static_cast<World *>(h)->bodies.size()); }
REFS_API void refs_get_state(void *h, float *pos, float *orn, float *lv, float *av, float *aabb) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    for (size_t i = 0; i < w->bodies.size(); ++i) {
        const auto e = w->bodies[i];
        if (!r.valid(e)) {                                  // destroyed by refs_destroy_body: the slot reads as zeros
            for (int k = 0; k < 3; ++k) pos[3 * i + k] = lv[3 * i + k] = av[3 * i + k] = 0;
            for (int k = 0; k < 4; ++k) orn[4 * i + k] = 0;
            if (aabb) for (int k = 0; k < 6; ++k) aabb[6 * i + k] = 0;
            continue;
        }
        const auto &p = r.get<edyn::position>(e); const auto &q = r.get<edyn::orientation>(e);
        pos[3 * i] = p.x; pos[3 * i + 1] = p.y; pos[3 * i + 2] = p.z;
        orn[4 * i] = q.x; orn[4 * i + 1] = q.y; orn[4 * i + 2] = q.z; orn[4 * i + 3] = q.w;
        if (auto *v = r.try_get<edyn::linvel>(e)) { lv[3 * i] = v->x; lv[3 * i + 1] = v->y; lv[3 * i + 2] = v->z; } else lv[3 * i] = lv[3 * i + 1] = lv[3 * i + 2] = 0;
        if (auto *v = r.try_get<edyn::angvel>(e)) { av[3 * i] = v->x; av[3 * i + 1] = v->y; av[3 * i + 2] = v->z; } else av[3 * i] = av[3 * i + 1] = av[3 * i + 2] = 0;
        if (aabb) {
            if (auto *bb = r.try_get<edyn::AABB>(e)) { aabb[6 * i] = bb->min.x; aabb[6 * i + 1] = bb->min.y; aabb[6 * i + 2] = bb->min.z; aabb[6 * i + 3] = bb->max.x; aabb[6 * i + 4] = bb->max.y; aabb[6 * i + 5] = bb->max.z; }
            else for (int k = 0; k < 6; ++k) aabb[6 * i + k] = 0;
        }
    }
}
REFS_API void refs_get_inertia_inv(void *h, float *inv9) {
    auto *w = static_cast<World *>(h);
    for (size_t i = 0; i < w->bodies.size(); ++i) {
        if (auto *m = w->registry.try_get<edyn::inertia_inv>(w->bodies[i])) for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) inv9[9 * i + 3 * r + c] = (*m)[r][c];
        else for (int k = 0; k < 9; ++k) inv9[9 * i + k] = 0;
    }
}
// manifolds: ordered body pairs (body[0], body[1]) as scene indices, point count, and per point (list order, head first)
// pivotA(3) pivotB(3) normal(3) distance normal_impulse friction_impulse(2) lifetime = 14 floats
REFS_API uint32_t refs_num_manifolds(void *h) { return uint32_t(static_cast<World *>(h)->registry.view<edyn::contact_manifold>().size()); }
REFS_API uint32_t refs_get_contacts(void *h, uint32_t capacity, uint32_t *pairs, uint32_t *num, float *pts14) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    std::vector<uint32_t> index;                      // entity index -> scene body index
    for (size_t i = 0; i < w->bodies.size(); ++i) { const auto k = entt::to_entity(w->bodies[i]); if (k >= index.size()) index.resize(k + 1, 0xFFFFFFFFu); index[k] = uint32_t(i); }
    uint32_t n = 0;
    auto cp_view = r.view<edyn::contact_point, edyn::contact_point_list, edyn::contact_point_geometry, edyn::contact_point_impulse>();
    for (auto [entity, manifold, state] : r.view<edyn::contact_manifold, edyn::contact_manifold_state>().each()) {
        if (n >= capacity) break;
        pairs[2 * n] = index[entt::to_entity(manifold.body[0])]; pairs[2 * n + 1] = index[entt::to_entity(manifold.body[1])];
        num[n] = state.num_points;
        uint32_t k = 0;
        for (auto ce = state.contact_entity; ce != entt::null && k < 4; ++k) {
            auto [cp, list, geom, imp] = cp_view.get(ce);
            float *o = pts14 + (size_t(n) * 4 + k) * 14;
            o[0] = cp.pivotA.x; o[1] = cp.pivotA.y; o[2] = cp.pivotA.z; o[3] = cp.pivotB.x; o[4] = cp.pivotB.y; o[5] = cp.pivotB.z;
            o[6] = cp.normal.x; o[7] = cp.normal.y; o[8] = cp.normal.z; o[9] = geom.distance;
            o[10] = imp.normal_impulse; o[11] = imp.friction_impulse[0]; o[12] = imp.friction_impulse[1]; o[13] = float(cp.lifetime);
            ce = list.next;
        }
        ++n;
    }
    return n;
}
// ---- process_collision on given manifolds (tests/golden/make_merge.py).  Layout of b2d_upload_contacts (include/b2d.h):
// per manifold 4 point slots, slot 0 = list head (newest); pt18 = pivotA(3) pivotB(3) normal(3) local_normal(3) distance
// friction restitution normal_impulse friction_impulse[2]; pt_u2 = {normal_attachment, lifetime}.
// Seeds manifolds with make_contact_manifold and their points with create_contact_point, last slot first so that slot 0
// ends up at the head, then patches every persisted field to the given value.  No broadphase runs on these bodies.
REFS_API int refs_seed_manifolds(void *h, uint32_t n, const uint32_t *pairs, const uint32_t *num, const float *pt18, const uint32_t *pt_u2) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    for (uint32_t k = 0; k < n; ++k) {
        if (pairs[2 * k] >= w->bodies.size() || pairs[2 * k + 1] >= w->bodies.size() || num[k] > 4) return -1;
        const auto me = edyn::make_contact_manifold(r, w->bodies[pairs[2 * k]], w->bodies[pairs[2 * k + 1]]);
        w->seeded.push_back(me);
        for (uint32_t s = num[k]; s-- > 0;) {
            const float *f = pt18 + ((size_t)k * 4 + s) * 18;
            const uint32_t *u = pt_u2 + ((size_t)k * 4 + s) * 2;
            auto &manifold = r.get<edyn::contact_manifold>(me);
            auto &state = r.get<edyn::contact_manifold_state>(me);
            edyn::collision_result::collision_point rp;
            rp.pivotA = v3(f); rp.pivotB = v3(f + 3); rp.normal = v3(f + 6); rp.distance = f[12];
            rp.normal_attachment = static_cast<edyn::contact_normal_attachment>(u[0]);
            const auto ce = edyn::create_contact_point(r, me, manifold, state, rp, std::nullopt);
            r.get<edyn::contact_point>(ce).lifetime = u[1];
            auto &geom = r.get<edyn::contact_point_geometry>(ce);
            geom.local_normal = v3(f + 9); geom.normal_attachment = rp.normal_attachment; geom.distance = f[12];
            auto &mat = r.get<edyn::contact_point_material>(ce);
            mat.friction = f[13]; mat.restitution = f[14];
            auto &imp = r.get<edyn::contact_point_impulse>(ce);
            imp.normal_impulse = f[15]; imp.friction_impulse = {f[16], f[17]};
        }
    }
    return 0;
}
// the reference's own narrowphase, as refs_step_begin calls it: update_contact_distances, then detect_collision and
// process_collision with the sequential create / destroy functors on every awake manifold
REFS_API void refs_narrowphase(void *h) {
    auto *w = static_cast<World *>(h);
    w->registry.ctx().get<edyn::narrowphase>().update(false);
}
// the seeded manifolds, in seeding order, in the layout of refs_seed_manifolds (slots past num are zero)
REFS_API int refs_get_seeded(void *h, uint32_t n, uint32_t *num, float *pt18, uint32_t *pt_u2) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    if (n != w->seeded.size()) return -1;
    std::memset(pt18, 0, (size_t)n * 4 * 18 * sizeof(float)); std::memset(pt_u2, 0, (size_t)n * 4 * 2 * sizeof(uint32_t));
    for (uint32_t k = 0; k < n; ++k) {
        const auto &state = r.get<edyn::contact_manifold_state>(w->seeded[k]);
        num[k] = state.num_points;
        uint32_t s = 0;
        for (auto ce = state.contact_entity; ce != entt::null; ce = r.get<edyn::contact_point_list>(ce).next, ++s) {
            if (s >= 4) return -2;
            const auto &cp = r.get<edyn::contact_point>(ce);
            const auto &geom = r.get<edyn::contact_point_geometry>(ce);
            const auto &mat = r.get<edyn::contact_point_material>(ce);
            const auto &imp = r.get<edyn::contact_point_impulse>(ce);
            float *o = pt18 + ((size_t)k * 4 + s) * 18;
            const edyn::vector3 vs[4] = {cp.pivotA, cp.pivotB, cp.normal, geom.local_normal};
            for (int j = 0; j < 4; ++j) { o[3 * j] = vs[j].x; o[3 * j + 1] = vs[j].y; o[3 * j + 2] = vs[j].z; }
            o[12] = geom.distance; o[13] = mat.friction; o[14] = mat.restitution;
            o[15] = imp.normal_impulse; o[16] = imp.friction_impulse[0]; o[17] = imp.friction_impulse[1];
            pt_u2[((size_t)k * 4 + s) * 2] = uint32_t(geom.normal_attachment);
            pt_u2[((size_t)k * 4 + s) * 2 + 1] = cp.lifetime;
        }
        if (s != state.num_points) return -3;
    }
    return 0;
}
// ---- what user code does between steps (plain registry / public API calls)
REFS_API void refs_destroy_body(void *h, uint32_t body) {                      // registry.destroy(entity)
    auto *w = static_cast<World *>(h);
    if (w->registry.valid(w->bodies[body])) w->registry.destroy(w->bodies[body]);
}
REFS_API void refs_remove_exclusion(void *h, uint32_t a, uint32_t b) {
    auto *w = static_cast<World *>(h);
    if (!w->registry.valid(w->bodies[a]) || !w->registry.valid(w->bodies[b])) return;      // one of them was destroyed
    edyn::remove_collision_exclusion(w->registry, w->bodies[a], w->bodies[b]);
}
REFS_API void refs_set_velocity(void *h, uint32_t body, const float *lv, const float *av) {
    auto *w = static_cast<World *>(h);
    w->registry.patch<edyn::linvel>(w->bodies[body], [&](edyn::linvel &v) { v.x = lv[0]; v.y = lv[1]; v.z = lv[2]; });
    w->registry.patch<edyn::angvel>(w->bodies[body], [&](edyn::angvel &v) { v.x = av[0]; v.y = av[1]; v.z = av[2]; });
}
// 1 per body that carries sleeping_tag (island_manager::put_to_sleep, island_manager.cpp:541-566)
REFS_API void refs_get_sleeping(void *h, uint32_t *asleep) {
    auto *w = static_cast<World *>(h);
    for (size_t i = 0; i < w->bodies.size(); ++i) asleep[i] = w->registry.valid(w->bodies[i]) && w->registry.all_of<edyn::sleeping_tag>(w->bodies[i]) ? 1u : 0u;
}
// island label per body: entity index of the island entity for procedural bodies, 0xFFFFFFFF otherwise
REFS_API void refs_get_islands(void *h, uint32_t *label) {
    auto *w = static_cast<World *>(h);
    for (size_t i = 0; i < w->bodies.size(); ++i) {
        auto *res = w->registry.try_get<edyn::island_resident>(w->bodies[i]);
        label[i] = (res && res->island_entity != entt::null) ? entt::to_integral(res->island_entity) : 0xFFFFFFFFu;
    }
}

// The rows of the LAST step in the order the island solver packed them (pack_rows / insert_rows, island_solver.cpp:113-175),
// island after island: hinges as scene hinge indices; contact rows as (body[0], body[1], k) = the k-th point, counted from
// the head of the manifold's point list, of the manifold of that ordered pair.  Returns 0, or -1 if a buffer is too small.
REFS_API int refs_get_solver_order(void *h, uint32_t cap_h, uint32_t *hinge_idx, uint32_t *nh, uint32_t cap_c, uint32_t *contact3, uint32_t *nc) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    std::vector<uint32_t> body_of, hinge_of;
    for (size_t i = 0; i < w->bodies.size(); ++i) { const auto k = entt::to_entity(w->bodies[i]); if (k >= body_of.size()) body_of.resize(k + 1, 0xFFFFFFFFu); body_of[k] = uint32_t(i); }
    for (size_t i = 0; i < w->hinges.size(); ++i) { const auto k = entt::to_entity(w->hinges[i]); if (k >= hinge_of.size()) hinge_of.resize(k + 1, 0xFFFFFFFFu); hinge_of[k] = uint32_t(i); }
    constexpr auto hinge_ix = edyn::tuple_index_of<unsigned, edyn::hinge_constraint>(edyn::constraints_tuple);
    constexpr auto contact_ix = edyn::tuple_index_of<unsigned, edyn::contact_constraint>(edyn::constraints_tuple);
    uint32_t kh = 0, kc = 0;
    auto list_view = r.view<edyn::contact_point_list>();
    for (auto [island_entity, ce] : r.view<edyn::island_constraint_entities>().each()) {
        if (r.any_of<edyn::sleeping_tag>(island_entity)) continue;
        for (auto e : ce.entities[hinge_ix]) { if (kh >= cap_h) return -1; hinge_idx[kh++] = hinge_of[entt::to_entity(e)]; }
        for (auto e : ce.entities[contact_ix]) {
            if (kc >= cap_c) return -1;
            const auto parent = list_view.get<edyn::contact_point_list>(e).parent;
            const auto &manifold = r.get<edyn::contact_manifold>(parent);
            uint32_t k = 0;
            for (auto p = r.get<edyn::contact_manifold_state>(parent).contact_entity; p != entt::null && p != e; p = list_view.get<edyn::contact_point_list>(p).next) ++k;
            contact3[3 * kc] = body_of[entt::to_entity(manifold.body[0])]; contact3[3 * kc + 1] = body_of[entt::to_entity(manifold.body[1])]; contact3[3 * kc + 2] = k;
            ++kc;
        }
    }
    *nh = kh; *nc = kc;
    return 0;
}
