// The reference-side binding of libb2d.so (INTEGRATION.md section 2), written against the reference's OWN headers and an
// entt::registry: edyn::stepper_b2d stands where stepper_sequential stands (src/edyn/simulation/stepper_sequential.cpp:28-147)
// and sends the per-step hot path -- broadphase, narrowphase, islands, solve, integrate -- through the C ABI
// (include/b2d.h).  User code is unchanged Edyn code: make_rigidbody, make_constraint<hinge_constraint>, exclude_collision,
// registry.patch<linvel>(...), registry.destroy(body).
//
// Needs <edyn/...> and <entt/...> on the include path, so it compiles where the reference does.  In this repository it is
// compiled by tests/integration/Makefile against /root/reference/include and oracle/entt_lite (the EnTT stand-in) and
// exercised by tests/test_stepper_b2d.py.  Not part of libb2d.so; there is no CPU fallback in here: if the device world
// cannot be created the constructor throws.
#pragma once
#include <entt/entity/registry.hpp>
#include <edyn/collision/contact_manifold.hpp>
#include <edyn/collision/contact_point.hpp>
#include <edyn/comp/aabb.hpp>
#include <edyn/comp/angvel.hpp>
#include <edyn/comp/collision_exclusion.hpp>
#include <edyn/comp/collision_filter.hpp>
#include <edyn/comp/gravity.hpp>
#include <edyn/comp/inertia.hpp>
#include <edyn/comp/linvel.hpp>
#include <edyn/comp/mass.hpp>
#include <edyn/comp/material.hpp>
#include <edyn/comp/orientation.hpp>
#include <edyn/comp/position.hpp>
#include <edyn/comp/present_orientation.hpp>
#include <edyn/comp/present_position.hpp>
#include <edyn/comp/shape_index.hpp>
#include <edyn/comp/tag.hpp>
#include <edyn/constraints/hinge_constraint.hpp>
#include <edyn/context/settings.hpp>
#include <edyn/dynamics/material_mixing.hpp>
#include <edyn/shapes/shapes.hpp>
#include <edyn/util/visit_component.hpp>
#include "b2d.h"
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <map>
#include <set>
#include <unordered_map>
#include <utility>
#include <vector>

// The mixing-table entry points are referenced weakly: this header-only binding also loads against a libb2d built before
// they existed, and then refuses a registry whose material_mix_table holds entries (sync_material_table).
extern "C" {
int b2d_set_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1, const float *friction,
                            const float *restitution) __attribute__((weak));
int b2d_remove_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1) __attribute__((weak));
}
// So are the presentation entry points: update() calls them only once a staged body has present_position /
// present_orientation, and throws then if the linked libb2d lacks them.
extern "C" {
int b2d_update_presentation(b2d_world *w, float interpolation_dt) __attribute__((weak));
int b2d_snap_presentation(b2d_world *w) __attribute__((weak));
int b2d_download_presentation(b2d_world *w, float *pos3n, float *orn4n) __attribute__((weak));
}

namespace edyn {

struct b2d_capacities {                          // what edyn::init_config would grow by: device + reservations
    int device {0};
    uint32_t max_bodies {1u << 16}, max_manifolds {1u << 19}, max_hinges {1u << 12};
    bool sleeping {false};                       // false = rigidbody_def::sleeping_disabled on every body
};

class stepper_b2d {
    static constexpr uint32_t no_id = 0xFFFFFFFFu;
    entt::registry *m_registry;
    b2d_world *m_world {};
    std::vector<entt::entity> m_entities;                    // body id -> entity (ids are never reused, b2d.h)
    std::vector<uint32_t> m_ids;                             // entt::to_entity(e) -> body id
    std::vector<entt::entity> m_new_bodies, m_new_hinges;    // filled by the construction signals, staged at the next step
    std::vector<entt::entity> m_dirty, m_exclusion_dirty;    // entities the user patched since the last step
    std::vector<std::vector<uint32_t>> m_excluded;           // body id -> ids it is staged as excluded from
    std::vector<uint8_t> m_is_dirty;
    std::vector<uint8_t> m_sensor;                           // body id -> staged without a material (B2D_MATERIAL_NONE)
    std::vector<entt::entity> m_material_toggled;            // material emplaced on / removed from an entity since the last step
    std::set<uint32_t> m_material_ids;                       // material::id values staged so far (UnassignedID excluded)
    std::map<uint32_t, std::pair<float, float>> m_mixing;    // the material_mix_table entries staged: lo << 16 | hi -> (friction, restitution)
    std::vector<uint32_t> m_asleep, m_was_asleep;            // B2D_FLAG_SLEEPING: sleeping_tag per body, this step / last step
    bool m_sleeping {false};
    std::vector<float> m_pos, m_orn, m_lv, m_av, m_aabb;     // download buffers
    std::vector<float> m_ppos, m_porn;                       // presentation download buffers
    std::unordered_map<uint64_t, entt::entity> m_manifold_of;   // (body id 0 << 32 | body id 1) -> mirrored contact_manifold entity
    uint64_t m_steps {0}, m_mirror_step {0};
    double m_last_time;
    double m_accumulated_time {};                            // stepper_sequential::m_accumulated_time
    bool m_presentation {false};                             // a staged body has present_position / present_orientation
    bool m_paused {false};
    bool m_scattering {false};                               // our own component writes are not "dirty"

    void check(int rc, const char *what) const {
        if (rc != B2D_OK) throw std::runtime_error(std::string(what) + ": " + b2d_last_error(m_world));
    }
    uint32_t id_of(entt::entity e) const {
        const auto k = entt::to_entity(e);
        return k < m_ids.size() ? m_ids[k] : no_id;
    }
    static void put3(float *dst, const vector3 &v) { dst[0] = float(v.x); dst[1] = float(v.y); dst[2] = float(v.z); }

public:
    stepper_b2d(entt::registry &registry, double time, const b2d_capacities &cap = {}) : m_registry(&registry), m_last_time(time) {
        const auto &s = registry.ctx().get<settings>();
        b2d_config c {};
        c.device = cap.device; c.max_bodies = cap.max_bodies; c.max_manifolds = cap.max_manifolds; c.max_hinges = cap.max_hinges;
        c.fixed_dt = float(s.fixed_dt);
        c.velocity_iterations = s.num_solver_velocity_iterations;
        c.position_iterations = s.num_solver_position_iterations;
        c.flags = cap.sleeping ? B2D_FLAG_SLEEPING : 0u;
        m_sleeping = cap.sleeping;
        if (s.num_restitution_iterations > 0) {              // the reference's default is 8 x 3 (context/settings.hpp:29-30)
            if (s.num_restitution_iterations != 8 || s.num_individual_restitution_iterations != 3)
                throw std::runtime_error("stepper_b2d: restitution iterations other than the defaults (8 x 3) or 0 are not supported");
            c.flags |= B2D_FLAG_RESTITUTION_SOLVER;
        }
        m_world = b2d_create(&c);
        if (!m_world) throw std::runtime_error(std::string("b2d_create: ") + b2d_last_error(nullptr));
        // make_rigidbody emplaces rigidbody_tag LAST (util/rigidbody.cpp:184): every other component exists by then
        registry.on_construct<rigidbody_tag>().connect<&stepper_b2d::on_construct_body>(*this);
        registry.on_destroy<rigidbody_tag>().connect<&stepper_b2d::on_destroy_body>(*this);
        registry.on_construct<hinge_constraint>().connect<&stepper_b2d::on_construct_hinge>(*this);
        registry.on_construct<collision_exclusion>().connect<&stepper_b2d::on_exclusion_changed>(*this);
        registry.on_update<collision_exclusion>().connect<&stepper_b2d::on_exclusion_changed>(*this);
        registry.on_destroy<collision_exclusion>().connect<&stepper_b2d::on_exclusion_changed>(*this);
        // the patch / replace contract of the reference's replicas (comp/shared_comp.hpp:36-86): what the user touches travels
        registry.on_update<position>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<orientation>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<linvel>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<angvel>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<mass_inv>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<inertia_inv>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<gravity>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_update<material>().connect<&stepper_b2d::on_update_body>(*this);
        registry.on_construct<material>().connect<&stepper_b2d::on_material_toggled>(*this);
        registry.on_destroy<material>().connect<&stepper_b2d::on_material_toggled>(*this);
        for (auto e : registry.view<rigidbody_tag>()) m_new_bodies.push_back(e);       // bodies that predate the stepper,
        std::reverse(m_new_bodies.begin(), m_new_bodies.end());                        // oldest first (views go newest first)
        for (auto e : registry.view<hinge_constraint>()) m_new_hinges.push_back(e);
        std::reverse(m_new_hinges.begin(), m_new_hinges.end());
    }
    stepper_b2d(const stepper_b2d &) = delete;
    stepper_b2d &operator=(const stepper_b2d &) = delete;
    ~stepper_b2d() {
        auto &r = *m_registry;
        r.on_construct<rigidbody_tag>().disconnect<&stepper_b2d::on_construct_body>(*this);
        r.on_destroy<rigidbody_tag>().disconnect<&stepper_b2d::on_destroy_body>(*this);
        r.on_construct<hinge_constraint>().disconnect<&stepper_b2d::on_construct_hinge>(*this);
        r.on_construct<collision_exclusion>().disconnect<&stepper_b2d::on_exclusion_changed>(*this);
        r.on_update<collision_exclusion>().disconnect<&stepper_b2d::on_exclusion_changed>(*this);
        r.on_destroy<collision_exclusion>().disconnect<&stepper_b2d::on_exclusion_changed>(*this);
        r.on_update<position>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<orientation>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<linvel>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<angvel>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<mass_inv>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<inertia_inv>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<gravity>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_update<material>().disconnect<&stepper_b2d::on_update_body>(*this);
        r.on_construct<material>().disconnect<&stepper_b2d::on_material_toggled>(*this);
        r.on_destroy<material>().disconnect<&stepper_b2d::on_material_toggled>(*this);
        b2d_destroy(m_world);
    }

    b2d_world *world() const { return m_world; }
    uint32_t body_id(entt::entity e) const { return id_of(e); }
    uint32_t num_bodies() const { return uint32_t(m_entities.size()); }

    // ---- signals
    void on_construct_body(entt::registry &, entt::entity e) { m_new_bodies.push_back(e); }
    void on_construct_hinge(entt::registry &, entt::entity e) { m_new_hinges.push_back(e); }
    void on_destroy_body(entt::registry &, entt::entity e) {           // island_manager::on_destroy_graph_node does the CPU side
        auto it = std::find(m_new_bodies.begin(), m_new_bodies.end(), e);
        if (it != m_new_bodies.end()) { m_new_bodies.erase(it); return; }      // created and destroyed between two steps
        const uint32_t id = id_of(e);
        if (id == no_id) return;
        check(b2d_remove_bodies(m_world, &id, 1), "b2d_remove_bodies");        // manifolds and joints attached to it go with it
        m_ids[entt::to_entity(e)] = no_id;
        m_entities[id] = entt::null;
        m_excluded[id].clear();
    }
    void on_update_body(entt::registry &, entt::entity e) {
        if (m_scattering) return;
        const uint32_t id = id_of(e);
        if (id == no_id || m_is_dirty[id]) return;                             // not staged yet: staged whole at the next step
        m_is_dirty[id] = 1;
        m_dirty.push_back(e);
    }
    void on_exclusion_changed(entt::registry &, entt::entity e) { m_exclusion_dirty.push_back(e); }
    // checked at the next step (registry.destroy(body) removes the material too, which is no toggle)
    void on_material_toggled(entt::registry &, entt::entity e) { if (id_of(e) != no_id) m_material_toggled.push_back(e); }

    // ---- staging: registry -> device
    void stage_new_bodies() {                                          // make_rigidbody's components -> b2d_bodies (SoA)
        auto &reg = *m_registry;
        m_new_bodies.erase(std::remove_if(m_new_bodies.begin(), m_new_bodies.end(), [&](auto e) { return !reg.valid(e); }), m_new_bodies.end());
        const auto n = uint32_t(m_new_bodies.size());
        if (!n) return;
        std::vector<float> pos(3 * n), orn(4 * n), lv(3 * n), av(3 * n), im(n), iI(9 * n), g(3 * n), sp(4 * n), fr(n), re(n);
        std::vector<uint32_t> kind(n), sk(n);
        std::vector<uint64_t> grp(n, ~0ull), msk(n, ~0ull);
        std::vector<uint32_t> mid(n, B2D_MATERIAL_NONE);                    // no material component: a sensor
        std::vector<uint32_t> pre(n, 0u);
        for (uint32_t i = 0; i < n; ++i) {
            const auto e = m_new_bodies[i];
            const bool has_pp = reg.all_of<present_position>(e), has_po = reg.all_of<present_orientation>(e);
            if (has_pp != has_po) throw std::runtime_error("stepper_b2d: a body with only one of present_position and present_orientation is not supported");
            pre[i] = has_pp ? 1u : 0u;
            m_presentation |= has_pp;
            put3(&pos[3 * i], reg.get<position>(e));
            const auto &q = reg.get<orientation>(e);
            orn[4 * i] = float(q.x); orn[4 * i + 1] = float(q.y); orn[4 * i + 2] = float(q.z); orn[4 * i + 3] = float(q.w);
            kind[i] = reg.all_of<dynamic_tag>(e) ? B2D_DYNAMIC : reg.all_of<kinematic_tag>(e) ? B2D_KINEMATIC : B2D_STATIC;
            if (kind[i] != B2D_STATIC) { put3(&lv[3 * i], reg.get<linvel>(e)); put3(&av[3 * i], reg.get<angvel>(e)); }
            if (kind[i] == B2D_DYNAMIC) {
                im[i] = float(reg.get<mass_inv>(e));
                const auto &I = reg.get<inertia_inv>(e);                       // matrix3x3, rows
                for (int r = 0; r < 3; ++r) put3(&iI[9 * i + 3 * r], I.row[r]);
                if (auto *gr = reg.try_get<gravity>(e)) put3(&g[3 * i], *gr);
            }
            if (auto *m = reg.try_get<material>(e)) {
                fr[i] = float(m->friction); re[i] = float(m->restitution); mid[i] = m->id;
                if (m->id != material::UnassignedID) m_material_ids.insert(m->id);
            }
            sk[i] = B2D_SHAPE_NONE;
            if (auto *si = reg.try_get<shape_index>(e)) {
                sk[i] = uint32_t(si->value);                                   // shapes.hpp:23-37 order == B2D_SHAPE_* values
                float *p = &sp[4 * i];
                if (auto *s = reg.try_get<sphere_shape>(e)) p[0] = float(s->radius);
                else if (auto *c = reg.try_get<capsule_shape>(e)) { p[0] = float(c->radius); p[1] = float(c->half_length); p[2] = float(int(c->axis)); }
                else if (auto *b = reg.try_get<box_shape>(e)) put3(p, b->half_extents);
                else if (auto *pl = reg.try_get<plane_shape>(e)) { put3(p, pl->normal); p[3] = float(pl->constant); }
                // any other shape: b2d_add_bodies answers B2D_ERR_UNSUPPORTED, surfaced below -- never a CPU fallback
            }
            if (auto *f = reg.try_get<collision_filter>(e)) { grp[i] = f->group; msk[i] = f->mask; }
        }
        b2d_bodies b {n, pos.data(), orn.data(), lv.data(), av.data(), im.data(), iI.data(), g.data(), kind.data(), sk.data(), sp.data(),
                      fr.data(), re.data(), grp.data(), msk.data(), mid.data(), pre.data()};
        uint32_t first = 0;
        check(b2d_add_bodies(m_world, &b, &first), "b2d_add_bodies");
        for (uint32_t i = 0; i < n; ++i) {
            const auto e = m_new_bodies[i];
            const auto k = entt::to_entity(e);
            if (k >= m_ids.size()) m_ids.resize(k + 1, no_id);
            m_ids[k] = first + i;
            m_entities.push_back(e);
            if (reg.all_of<collision_exclusion>(e)) m_exclusion_dirty.push_back(e);
        }
        m_excluded.resize(m_entities.size());
        m_is_dirty.resize(m_entities.size(), 0);
        for (uint32_t i = 0; i < n; ++i) m_sensor.push_back(mid[i] == B2D_MATERIAL_NONE ? 1 : 0);
        m_new_bodies.clear();
    }

    void stage_new_hinges() {                                          // make_constraint<hinge_constraint> + set_axes
        auto &reg = *m_registry;
        m_new_hinges.erase(std::remove_if(m_new_hinges.begin(), m_new_hinges.end(), [&](auto e) { return !reg.valid(e); }), m_new_hinges.end());
        const auto n = uint32_t(m_new_hinges.size());
        if (!n) return;
        std::vector<uint32_t> a(n), b(n);
        std::vector<float> pa(3 * n), pb(3 * n), xa(3 * n), xb(3 * n);
        for (uint32_t i = 0; i < n; ++i) {
            const auto &h = reg.get<hinge_constraint>(m_new_hinges[i]);
            a[i] = id_of(h.body[0]); b[i] = id_of(h.body[1]);
            if (a[i] == no_id || b[i] == no_id) throw std::runtime_error("stepper_b2d: hinge between bodies that are not rigid bodies");
            put3(&pa[3 * i], h.pivot[0]); put3(&pb[3 * i], h.pivot[1]);
            put3(&xa[3 * i], h.frame[0].column(0));                            // set_axes: frame = columns(axis, p, q), hinge_constraint.cpp:11-17
            put3(&xb[3 * i], h.frame[1].column(0));
        }
        check(b2d_add_hinges(m_world, n, a.data(), b.data(), pa.data(), pb.data(), xa.data(), xb.data()), "b2d_add_hinges");
        m_new_hinges.clear();
    }

    bool lists(entt::entity e, entt::entity other) const {            // should_exclude, collision/should_collide.cpp:11-21
        if (auto *x = m_registry->try_get<collision_exclusion>(e)) {
            for (unsigned i = 0; i < x->num_entities(); ++i) if (x->entity[i] == other) return true;
        }
        return false;
    }

    // exclude_collision / remove_collision_exclusion: a pair is excluded while EITHER body lists the other
    // (should_collide.cpp); pairs travel once, whichever side changed
    void stage_exclusions() {
        auto &reg = *m_registry;
        std::vector<uint32_t> add_a, add_b, del_a, del_b;
        for (auto e : m_exclusion_dirty) {
            const uint32_t id = reg.valid(e) ? id_of(e) : no_id;
            if (id == no_id) continue;
            std::vector<uint32_t> now;
            if (auto *x = reg.try_get<collision_exclusion>(e)) {
                for (unsigned i = 0; i < x->num_entities(); ++i) { const uint32_t o = id_of(x->entity[i]); if (o != no_id) now.push_back(o); }
            }
            auto &was = m_excluded[id];
            for (uint32_t o : now) {
                if (std::find(was.begin(), was.end(), o) != was.end()) continue;
                auto &theirs = m_excluded[o];                                  // already staged from the other side?
                if (std::find(theirs.begin(), theirs.end(), id) == theirs.end()) { add_a.push_back(id); add_b.push_back(o); }
            }
            for (uint32_t o : was) {
                if (std::find(now.begin(), now.end(), o) != now.end()) continue;
                if (m_entities[o] == entt::null || !lists(m_entities[o], e)) { del_a.push_back(id); del_b.push_back(o); }
            }
            was = std::move(now);
        }
        m_exclusion_dirty.clear();
        if (!del_a.empty()) check(b2d_remove_exclusions(m_world, uint32_t(del_a.size()), del_a.data(), del_b.data()), "b2d_remove_exclusions");
        if (!add_a.empty()) check(b2d_add_exclusions(m_world, uint32_t(add_a.size()), add_a.data(), add_b.data()), "b2d_add_exclusions");
    }

    void upload_dirty() {                                              // only the patched entities travel
        auto &reg = *m_registry;
        std::vector<uint32_t> ids;
        std::vector<float> pos, orn, lv, av, im, iI, g, fr, re;
        std::vector<uint32_t> mid;
        for (auto e : m_dirty) {
            const uint32_t id = reg.valid(e) ? id_of(e) : no_id;
            if (id == no_id) continue;
            m_is_dirty[id] = 0;
            ids.push_back(id);
            float t[9] = {};
            put3(t, reg.get<position>(e)); pos.insert(pos.end(), t, t + 3);
            const auto &q = reg.get<orientation>(e);
            const float qq[4] = {float(q.x), float(q.y), float(q.z), float(q.w)}; orn.insert(orn.end(), qq, qq + 4);
            const bool moves = !reg.all_of<static_tag>(e);
            put3(t, moves ? vector3(reg.get<linvel>(e)) : vector3_zero); lv.insert(lv.end(), t, t + 3);
            put3(t, moves ? vector3(reg.get<angvel>(e)) : vector3_zero); av.insert(av.end(), t, t + 3);
            const bool dyn = reg.all_of<dynamic_tag>(e);
            im.push_back(dyn ? float(reg.get<mass_inv>(e)) : 0.f);
            if (dyn) { const auto &I = reg.get<inertia_inv>(e); for (int r = 0; r < 3; ++r) put3(t + 3 * r, I.row[r]); } else std::fill(t, t + 9, 0.f);
            iI.insert(iI.end(), t, t + 9);
            auto *gr = reg.try_get<gravity>(e);
            put3(t, gr ? vector3(*gr) : vector3_zero); g.insert(g.end(), t, t + 3);
            auto *m = reg.try_get<material>(e);
            fr.push_back(m ? float(m->friction) : 0.f); re.push_back(m ? float(m->restitution) : 0.f);
            mid.push_back(m ? uint32_t(m->id) : B2D_MATERIAL_NONE);
            if (m && m->id != material::UnassignedID) m_material_ids.insert(m->id);
        }
        m_dirty.clear();
        if (ids.empty()) return;
        b2d_body_patch p {pos.data(), orn.data(), lv.data(), av.data(), im.data(), iI.data(), g.data(), fr.data(), re.data(), nullptr, mid.data()};
        check(b2d_upload_bodies(m_world, uint32_t(ids.size()), ids.data(), &p), "b2d_upload_bodies");
    }

    // A staged body cannot gain or lose its material: the device fixes a point's constraint type (contact_constraint or
    // null_constraint) when the point is created, as the reference does, and does not track it per point.
    void check_material_toggles() {
        auto &reg = *m_registry;
        for (auto e : m_material_toggled) {
            const uint32_t id = reg.valid(e) ? id_of(e) : no_id;
            if (id != no_id && reg.all_of<material>(e) == (m_sensor[id] != 0))
                throw std::runtime_error("stepper_b2d: emplacing or removing the material of an existing body (sensor <-> non-sensor) is not supported");
        }
        m_material_toggled.clear();
    }

    // material_mix_table (dynamics/material_mixing.hpp:36-80) has no iteration API and raises no signal: every step probes
    // try_get for each unordered pair of the material ids staged so far (k (k + 1) / 2 pairs for k ids, each looked up in
    // both orders when the first misses), and uploads what
    // changed since the last step.  Entries with contact extras (spin / roll friction, stiffness / damping) are out of scope.
    void sync_material_table() {
        auto *table = m_registry->ctx().find<material_mix_table>();
        if (!table || m_material_ids.empty()) return;
        std::vector<uint32_t> set_a, set_b, del_a, del_b;
        std::vector<float> set_f, set_r;
        for (auto i = m_material_ids.begin(); i != m_material_ids.end(); ++i) {
            for (auto j = i; j != m_material_ids.end(); ++j) {
                const uint32_t key = (*i << 16) | *j;
                // both orders: unordered_pair's operator< (core/unordered_pair.hpp) is no strict weak ordering, so the
                // std::map can miss an entry inserted as (j, i) when it is looked up as (i, j)
                const auto *m = table->try_get({material::id_type(*i), material::id_type(*j)});
                if (!m) m = table->try_get({material::id_type(*j), material::id_type(*i)});
                auto it = m_mixing.find(key);
                if (!m) {
                    if (it != m_mixing.end()) { del_a.push_back(*i); del_b.push_back(*j); m_mixing.erase(it); }
                    continue;
                }
                if (m->spin_friction != 0 || m->roll_friction != 0 || m->stiffness < large_scalar || m->damping < large_scalar)
                    throw std::runtime_error("stepper_b2d: material mixing entries with spin / roll friction, stiffness or damping are not supported");
                const std::pair<float, float> v {float(m->friction), float(m->restitution)};
                if (it != m_mixing.end() && it->second == v) continue;
                m_mixing[key] = v;
                set_a.push_back(*i); set_b.push_back(*j); set_f.push_back(v.first); set_r.push_back(v.second);
            }
        }
        if ((!del_a.empty() || !set_a.empty()) && (!b2d_set_material_mixing || !b2d_remove_material_mixing))
            throw std::runtime_error("stepper_b2d: the linked libb2d has no material mixing (b2d_set_material_mixing)");
        if (!del_a.empty()) check(b2d_remove_material_mixing(m_world, uint32_t(del_a.size()), del_a.data(), del_b.data()), "b2d_remove_material_mixing");
        if (!set_a.empty()) check(b2d_set_material_mixing(m_world, uint32_t(set_a.size()), set_a.data(), set_b.data(), set_f.data(), set_r.data()), "b2d_set_material_mixing");
    }

    // ---- device -> registry: what solver::update writes at the end of a step (island_solver.cpp:358-376,
    // sys/update_aabbs.cpp:53-78); written in place, without signals, like the CPU stepper does
    void scatter_state() {
        auto &reg = *m_registry;
        const auto n = m_entities.size();
        m_pos.resize(3 * n); m_orn.resize(4 * n); m_lv.resize(3 * n); m_av.resize(3 * n); m_aabb.resize(6 * n);
        check(b2d_download_state(m_world, m_pos.data(), m_orn.data(), m_lv.data(), m_av.data(), m_aabb.data(), nullptr), "b2d_download_state");
        m_scattering = true;
        auto body_view = reg.view<position, orientation, linvel, angvel>();
        auto aabb_view = reg.view<AABB>();
        auto static_view = reg.view<static_tag>();
        for (size_t i = 0; i < n; ++i) {
            const auto e = m_entities[i];
            if (e == entt::null || static_view.contains(e)) continue;
            auto [p, q, v, w] = body_view.get(e);
            p.x = m_pos[3 * i]; p.y = m_pos[3 * i + 1]; p.z = m_pos[3 * i + 2];
            q.x = m_orn[4 * i]; q.y = m_orn[4 * i + 1]; q.z = m_orn[4 * i + 2]; q.w = m_orn[4 * i + 3];
            v.x = m_lv[3 * i]; v.y = m_lv[3 * i + 1]; v.z = m_lv[3 * i + 2];
            w.x = m_av[3 * i]; w.y = m_av[3 * i + 1]; w.z = m_av[3 * i + 2];
            if (aabb_view.contains(e)) {
                auto &bb = aabb_view.get<AABB>(e);
                bb.min = {m_aabb[6 * i], m_aabb[6 * i + 1], m_aabb[6 * i + 2]};
                bb.max = {m_aabb[6 * i + 3], m_aabb[6 * i + 4], m_aabb[6 * i + 5]};
            }
        }
        m_scattering = false;
    }

    // ---- device -> registry: present_position / present_orientation after b2d_update_presentation or b2d_snap_presentation,
    // written in place without signals, like update_presentation does
    // b2d_snap_presentation or b2d_update_presentation, then the components; nothing while no body has presentation
    void present(bool snap, float interpolation_dt) {
        if (!m_presentation) return;
        if (!b2d_update_presentation || !b2d_snap_presentation || !b2d_download_presentation)
            throw std::runtime_error("stepper_b2d: the linked libb2d has no presentation transforms (b2d_update_presentation)");
        if (snap) check(b2d_snap_presentation(m_world), "b2d_snap_presentation");
        else check(b2d_update_presentation(m_world, interpolation_dt), "b2d_update_presentation");
        scatter_presentation();
    }
    void scatter_presentation() {
        auto &reg = *m_registry;
        const auto n = m_entities.size();
        m_ppos.resize(3 * n); m_porn.resize(4 * n);
        if (n) check(b2d_download_presentation(m_world, m_ppos.data(), m_porn.data()), "b2d_download_presentation");
        auto view = reg.view<present_position, present_orientation>();
        for (size_t i = 0; i < n; ++i) {
            const auto e = m_entities[i];
            if (e == entt::null || !view.contains(e)) continue;
            auto [p, q] = view.get(e);
            p.x = m_ppos[3 * i]; p.y = m_ppos[3 * i + 1]; p.z = m_ppos[3 * i + 2];
            q.x = m_porn[4 * i]; q.y = m_porn[4 * i + 1]; q.z = m_porn[4 * i + 2]; q.w = m_porn[4 * i + 3];
        }
    }

    // sleeping_tag on the bodies as island_manager::put_to_sleep / wake_up_island leave it (island_manager.cpp:541-566,
    // :257-295); islands fall asleep and wake up on the device
    void sync_sleeping() {
        auto &reg = *m_registry;
        const auto n = m_entities.size();
        m_asleep.resize(n); m_was_asleep.resize(n, 0u);
        check(b2d_download_sleeping(m_world, m_asleep.data()), "b2d_download_sleeping");
        for (size_t i = 0; i < n; ++i) {
            if (m_asleep[i] == m_was_asleep[i] || m_entities[i] == entt::null) continue;
            if (m_asleep[i]) reg.emplace_or_replace<sleeping_tag>(m_entities[i]); else reg.remove<sleeping_tag>(m_entities[i]);
        }
        m_was_asleep = m_asleep;
    }

    // edyn::wake_up_entity for a body of the device world (util/island_util.cpp): its island follows at the next step
    void wake_up(entt::entity e) {
        const uint32_t id = id_of(e);
        if (id == no_id) return;
        check(b2d_wake_bodies(m_world, &id, 1), "b2d_wake_bodies");
        m_registry->remove<sleeping_tag>(e);
        if (id < m_was_asleep.size()) m_was_asleep[id] = 0;
    }

    // everything the user changed in the registry since the last call travels to the device
    void stage() {
        check_material_toggles();
        stage_new_bodies();
        stage_new_hinges();
        stage_exclusions();
        upload_dirty();
        sync_material_table();
    }

    void step_once() {
        auto &s = m_registry->ctx().get<settings>();
        stage();
        if (s.pre_step_callback) (*s.pre_step_callback)(*m_registry);
        check(b2d_step(m_world, 1), "b2d_step");
        ++m_steps;
        scatter_state();                                               // blocks until the step's results are on the host
        if (m_sleeping) sync_sleeping();
        if (s.post_step_callback) (*s.post_step_callback)(*m_registry);
    }

    // ---- stepper_sequential's public surface
    void step_simulation(double time) {                                // stepper_sequential.cpp:121-147 (one fixed step)
        m_last_time = time;
        step_once();
    }

    // stepper_sequential.cpp:28-69, :104-105: the fixed-step accumulator, then the presentation transforms.  Time beyond
    // max_steps_per_update fixed steps is dropped, as the reference drops it.  While paused only snap_presentation runs and
    // the last time stays where it was (:37-43).
    void update(double time) {
        if (m_paused) {
            stage();
            present(true, 0.0f);
            return;
        }
        const auto &s = m_registry->ctx().get<settings>();
        const auto elapsed = std::max(time - m_last_time, 0.0);
        m_accumulated_time += elapsed;
        const auto fixed_dt = s.fixed_dt;
        const auto num_steps = static_cast<uint64_t>(std::floor(m_accumulated_time / fixed_dt));
        const auto advance_dt = static_cast<double>(num_steps) * fixed_dt;
        m_accumulated_time -= advance_dt;
        const auto effective_steps = std::min<uint64_t>(num_steps, s.max_steps_per_update);
        for (uint64_t i = 0; i < effective_steps; ++i) step_once();
        m_last_time = time;
        // update_presentation(registry, get_simulation_timestamp(), time, elapsed, fixed_dt), update_presentation.cpp:70
        const double sim_time = m_last_time - m_accumulated_time;
        const auto interpolation_dt = std::min(static_cast<scalar>(time - double(fixed_dt) - sim_time), s.fixed_dt);
        stage();                                                       // bodies created or patched since the last step count too
        present(false, float(interpolation_dt));
    }

    // ---- contacts, on demand (SURVEY.md section 8 f2).  The device keeps manifolds and points resident; creating and
    // destroying an entity with five components per contact point per step on the host is the cost this design removes.
    // A user who observes contacts calls mirror_contacts() when they want to look: afterwards the registry holds what
    // the CPU stepper would hold -- one contact_manifold + contact_manifold_state entity per touching (AABB-overlapping)
    // pair, and per contact point an entity with contact_point, contact_point_list, contact_point_geometry,
    // contact_point_material and contact_point_impulse -- the last two only where both bodies have a material (a sensor's
    // points have neither, collision_util.cpp:358-384) -- linked newest first (collision_util.cpp:319-395).  A point keeps
    // its entity for as long as it persists on the device (matched through its lifetime counter and its place in the
    // list); new points get contact_started_tag after their components, like narrowphase::patch_new_contacts
    // (narrowphase.cpp:111-130); vanished points and manifolds are destroyed, so on_destroy<contact_point> fires.
    // Not mirrored: the contact_constraint / graph edge of each point (the CPU solver is not running).
    struct mirror_stats { uint32_t manifolds, points, points_created, points_destroyed; };

    mirror_stats mirror_contacts() {
        auto &reg = *m_registry;
        uint32_t n = 0, got = 0;
        check(b2d_num_manifolds(m_world, &n), "b2d_num_manifolds");
        std::vector<uint32_t> pairs(2 * size_t(n) + 2), num(size_t(n) + 1), u2(8 * size_t(n) + 8);
        std::vector<float> pt(72 * size_t(n) + 72);                            // 4 slots x 18 floats per manifold
        if (n) check(b2d_download_contacts(m_world, n, pairs.data(), num.data(), pt.data(), u2.data(), &got), "b2d_download_contacts");
        const uint32_t elapsed = uint32_t(m_steps - m_mirror_step);
        mirror_stats st {};
        std::unordered_map<uint64_t, entt::entity> next;
        next.reserve(got);
        for (uint32_t i = 0; i < got; ++i) {
            const uint32_t a = pairs[2 * i], b = pairs[2 * i + 1];
            if (a >= m_entities.size() || b >= m_entities.size() || m_entities[a] == entt::null || m_entities[b] == entt::null) continue;
            const uint64_t key = (uint64_t(a) << 32) | b;
            entt::entity me;
            if (auto it = m_manifold_of.find(key); it != m_manifold_of.end()) { me = it->second; m_manifold_of.erase(it); }
            else {
                me = reg.create();
                reg.emplace<contact_manifold>(me, contact_manifold{{m_entities[a], m_entities[b]}});
                reg.emplace<contact_manifold_state>(me);
            }
            next.emplace(key, me);
            const bool sensor = m_sensor[a] || m_sensor[b];
            sync_points(me, std::min<uint32_t>(num[i], 4u), &pt[72 * size_t(i)], &u2[8 * size_t(i)], elapsed, sensor, st);
            ++st.manifolds;
        }
        for (auto &gone : m_manifold_of) {                                     // pairs that separated since the last look
            if (!reg.valid(gone.second)) continue;
            sync_points(gone.second, 0, nullptr, nullptr, elapsed, false, st);
            reg.destroy(gone.second);
        }
        m_manifold_of.swap(next);
        m_mirror_step = m_steps;
        return st;
    }

private:
    // sensor: a pair with a body without material, whose points have no contact_point_material and no contact_point_impulse
    // (collision_util.cpp:358-384)
    void sync_points(entt::entity me, uint32_t np, const float *p18, const uint32_t *u2, uint32_t elapsed, bool sensor, mirror_stats &st) {
        auto &reg = *m_registry;
        std::vector<entt::entity> old, now(np, entt::entity{entt::null}), fresh;
        for (auto e = reg.get<contact_manifold_state>(me).contact_entity; e != entt::null; e = reg.get<contact_point_list>(e).next) old.push_back(e);
        size_t j = 0;
        for (uint32_t s = 0; s < np; ++s) {
            const float *p = p18 + 18 * s;
            const uint32_t lifetime = u2[2 * s + 1];
            entt::entity e = entt::null;
            if (lifetime >= elapsed) {                                         // older than the last look: find its entity, in list order
                size_t k = j;
                while (k < old.size() && reg.get<contact_point>(old[k]).lifetime + elapsed != lifetime) ++k;
                if (k < old.size()) {
                    for (; j < k; ++j) { reg.destroy(old[j]); ++st.points_destroyed; }
                    e = old[k]; j = k + 1;
                }
            }
            if (e == entt::null) {
                e = reg.create();
                if (!sensor) { reg.emplace<contact_point_material>(e); reg.emplace<contact_point_impulse>(e); }
                reg.emplace<contact_point_geometry>(e);
                reg.emplace<contact_point_list>(e);
                reg.emplace<contact_point>(e);
                fresh.push_back(e);
                ++st.points_created;
            }
            auto &cp = reg.get<contact_point>(e);
            cp.pivotA = {p[0], p[1], p[2]}; cp.pivotB = {p[3], p[4], p[5]}; cp.normal = {p[6], p[7], p[8]}; cp.lifetime = lifetime;
            auto &geom = reg.get<contact_point_geometry>(e);
            geom.local_normal = {p[9], p[10], p[11]}; geom.distance = p[12];
            geom.normal_attachment = static_cast<contact_normal_attachment>(u2[2 * s]);
            if (!sensor) {
                auto &mat = reg.get<contact_point_material>(e);
                mat.friction = p[13]; mat.restitution = p[14]; mat.spin_friction = 0; mat.roll_friction = 0;
                auto &imp = reg.get<contact_point_impulse>(e);
                imp.normal_impulse = p[15]; imp.friction_impulse = {p[16], p[17]};
            }
            now[s] = e;
            ++st.points;
        }
        for (; j < old.size(); ++j) { reg.destroy(old[j]); ++st.points_destroyed; }
        for (uint32_t s = 0; s < np; ++s) {
            auto &link = reg.get<contact_point_list>(now[s]);
            link.parent = me; link.next = s + 1 < np ? now[s + 1] : entt::entity{entt::null};
        }
        auto &state = reg.get<contact_manifold_state>(me);
        state.num_points = uint8_t(np);
        state.contact_entity = np ? now[0] : entt::entity{entt::null};
        for (auto e : fresh) reg.emplace<contact_started_tag>(e);
    }

public:
    void set_paused(bool paused) { m_paused = paused; m_accumulated_time = 0; }       // stepper_sequential.cpp:148-151
    bool is_paused() const { return m_paused; }
};

} // namespace edyn
