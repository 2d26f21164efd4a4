// TEST INFRASTRUCTURE.  Material entry points on top of oracle/ref_stepper.cpp (included before this header): bodies with
// a material id or without a material (a sensor), the registry's material_mix_table, and contact read-backs that do not
// assume every point has a contact_point_material / contact_point_impulse (a sensor's points have neither,
// collision_util.cpp:358-384).
#pragma once
#include <edyn/dynamics/material_mixing.hpp>

// refs_add_bodies, then per body: material[i] = 0xFFFFFFFF -> no material component (rigidbody_def::material left
// empty), else material::id = material[i].  make_rigidbody emplaces nothing else that depends on the material
// (util/rigidbody.cpp:95-96), and nothing reads it before the first step.
REFS_API int refm_add_bodies(void *h, uint32_t n, const float *pos, const float *orn, const float *lv, const float *av, const float *inv_mass,
                             const float *gravity, const uint32_t *kind, const uint32_t *shape_kind, const float *sp,
                             const float *friction, const float *restitution, const uint64_t *group, const uint64_t *mask,
                             int sleeping_disabled, const uint32_t *material) {
    auto *w = static_cast<World *>(h);
    const size_t first = w->bodies.size();
    if (int rc = refs_add_bodies(h, n, pos, orn, lv, av, inv_mass, gravity, kind, shape_kind, sp, friction, restitution, group, mask, sleeping_disabled)) return rc;
    for (uint32_t i = 0; i < n; ++i) {
        const auto e = w->bodies[first + i];
        if (material[i] == 0xFFFFFFFFu) w->registry.remove<edyn::material>(e);
        else w->registry.get<edyn::material>(e).id = edyn::material::id_type(material[i]);
    }
    return 0;
}
// material_mix_table insert / remove for n id pairs, straight into registry.ctx().get<material_mix_table>(): all that
// edyn::insert_material_mixing does in sequential mode (util/insert_material_mixing.cpp:9-22); its other branches
// reference the networking layer, which this build of the reference leaves out.
REFS_API void refm_set_material_mixing(void *h, uint32_t n, const uint32_t *id0, const uint32_t *id1, const float *friction,
                                       const float *restitution, int remove) {
    auto &table = static_cast<World *>(h)->registry.ctx().get<edyn::material_mix_table>();
    for (uint32_t i = 0; i < n; ++i) {
        const edyn::material_mix_table::pair_type pair{edyn::material::id_type(id0[i]), edyn::material::id_type(id1[i])};
        if (remove) { table.remove(pair); continue; }
        edyn::material_base m; m.friction = friction[i]; m.restitution = restitution[i];
        table.insert(pair, m);
    }
}
// refs_get_contacts' layout (pts14), plus per point mat4 = contact_point_material friction and restitution (0 without one),
// 1 if it carries a contact_constraint, 1 if it carries a contact_point_impulse
REFS_API uint32_t refm_get_contacts(void *h, uint32_t capacity, uint32_t *pairs, uint32_t *num, float *pts14, float *mat4) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    std::vector<uint32_t> index;
    for (size_t i = 0; i < w->bodies.size(); ++i) { const auto k = entt::to_entity(w->bodies[i]); if (k >= index.size()) index.resize(k + 1, 0xFFFFFFFFu); index[k] = uint32_t(i); }
    uint32_t n = 0;
    for (auto [entity, manifold, state] : r.view<edyn::contact_manifold, edyn::contact_manifold_state>().each()) {
        if (n >= capacity) break;
        pairs[2 * n] = index[entt::to_entity(manifold.body[0])]; pairs[2 * n + 1] = index[entt::to_entity(manifold.body[1])];
        num[n] = state.num_points;
        uint32_t k = 0;
        for (auto ce = state.contact_entity; ce != entt::null && k < 4; ++k) {
            const auto &cp = r.get<edyn::contact_point>(ce);
            const auto &geom = r.get<edyn::contact_point_geometry>(ce);
            const auto *imp = r.try_get<edyn::contact_point_impulse>(ce);
            const auto *mat = r.try_get<edyn::contact_point_material>(ce);
            float *o = pts14 + (size_t(n) * 4 + k) * 14, *q = mat4 + (size_t(n) * 4 + k) * 4;
            o[0] = cp.pivotA.x; o[1] = cp.pivotA.y; o[2] = cp.pivotA.z; o[3] = cp.pivotB.x; o[4] = cp.pivotB.y; o[5] = cp.pivotB.z;
            o[6] = cp.normal.x; o[7] = cp.normal.y; o[8] = cp.normal.z; o[9] = geom.distance;
            o[10] = imp ? imp->normal_impulse : 0; o[11] = imp ? imp->friction_impulse[0] : 0; o[12] = imp ? imp->friction_impulse[1] : 0;
            o[13] = float(cp.lifetime);
            q[0] = mat ? mat->friction : 0; q[1] = mat ? mat->restitution : 0;
            q[2] = r.all_of<edyn::contact_constraint>(ce) ? 1.0f : 0.0f; q[3] = imp ? 1.0f : 0.0f;
            ce = r.get<edyn::contact_point_list>(ce).next;
        }
        ++n;
    }
    return n;
}
