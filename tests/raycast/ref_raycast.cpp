// TEST INFRASTRUCTURE: the reference's own raycast behind a small C interface, for the raycast tests and
// tests/golden/make_raycast.py.  Compiled by tests/raycast_support.py against the reference's headers and linked with the
// reference's object files that oracle/Makefile (`make -C oracle stepper`) compiles in place into oracle/_ref/edyn_obj,
// with the same flags; only where those exist.  Nothing is copied from the reference.
#include <edyn/edyn.hpp>
#include <edyn/util/rigidbody.hpp>
#include <edyn/collision/raycast.hpp>
#include <edyn/networking/util/snap_to_pool_snapshot.hpp>
#include <edyn/networking/util/process_extrapolation_result.hpp>
#include <entt/entity/registry.hpp>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

// The asynchronous stepper's translation units mention two entry points of the networking layer, which is not linked;
// raycasts never reach them.
namespace edyn {
void snap_to_pool_snapshot(entt::registry &, const entity_map &, const std::vector<entt::entity> &, const std::vector<pool_snapshot> &, bool) {
    std::fputs("ref_raycast: networking code reached\n", stderr); std::abort();
}
void process_extrapolation_result(entt::registry &, entity_map &, const extrapolation_result &) {
    std::fputs("ref_raycast: networking code reached\n", stderr); std::abort();
}
}

#define RR_API extern "C" __attribute__((visibility("default")))

namespace {
struct World {
    entt::registry registry;
    std::vector<entt::entity> bodies;
};
edyn::vector3 v3(const float *p) { return {p[0], p[1], p[2]}; }
// out4 = fraction, normal; *feature = box face, capsule hemisphere index or 2 for the capsule side, 0xFFFFFFFF otherwise
// (include/b2d.h conventions).
void put(const edyn::shape_raycast_result &r, float *out4, uint32_t *feature) {
    out4[0] = r.fraction; out4[1] = r.normal.x; out4[2] = r.normal.y; out4[3] = r.normal.z;
    *feature = 0xFFFFFFFFu;
    if (auto *b = std::get_if<edyn::box_raycast_info>(&r.info_var)) *feature = uint32_t(b->face_index);
    if (auto *c = std::get_if<edyn::capsule_raycast_info>(&r.info_var))
        *feature = c->feature == edyn::capsule_feature::side ? 2u : uint32_t(c->hemisphere_index);
}
}

// edyn::shape_raycast of one shape (0 sphere{r}, 2 capsule{r, half_length, axis}, 3 box{half extents}, 6 plane{n, constant}),
// unfiltered.
RR_API void rr_shape_raycast(uint32_t kind, const float *p, const float *pos, const float *orn, const float *p0, const float *p1,
                             float *out4, uint32_t *feature) {
    edyn::raycast_context ctx{v3(pos), edyn::quaternion{orn[0], orn[1], orn[2], orn[3]}, v3(p0), v3(p1)};
    edyn::shape_raycast_result r;
    switch (kind) {
    case 0: r = edyn::shape_raycast(edyn::sphere_shape{p[0]}, ctx); break;
    case 2: r = edyn::shape_raycast(edyn::capsule_shape{p[0], p[1], static_cast<edyn::coordinate_axis>(int(p[2]))}, ctx); break;
    case 3: r = edyn::shape_raycast(edyn::box_shape{edyn::vector3{p[0], p[1], p[2]}}, ctx); break;
    case 6: r = edyn::shape_raycast(edyn::plane_shape{edyn::vector3{p[0], p[1], p[2]}, p[3]}, ctx); break;
    default: break;
    }
    put(r, out4, feature);
}

// A registry of n static bodies (edyn::attach, make_rigidbody, one edyn::update, as test/edyn/collision/test_raycast.cpp).
RR_API void *rr_create(uint32_t n, const float *pos, const float *orn, const uint32_t *shape_kind, const float *sp) {
    auto *w = new World();
    edyn::init_config cfg;
    cfg.execution_mode = edyn::execution_mode::sequential;
    edyn::attach(w->registry, cfg);
    for (uint32_t i = 0; i < n; ++i) {
        edyn::rigidbody_def def;
        def.kind = edyn::rigidbody_kind::rb_static;
        def.position = v3(pos + 3 * i);
        def.orientation = {orn[4 * i], orn[4 * i + 1], orn[4 * i + 2], orn[4 * i + 3]};
        const float *p = sp + 4 * i;
        switch (shape_kind[i]) {
        case 0: def.shape = edyn::sphere_shape{p[0]}; break;
        case 2: def.shape = edyn::capsule_shape{p[0], p[1], static_cast<edyn::coordinate_axis>(int(p[2]))}; break;
        case 3: def.shape = edyn::box_shape{edyn::vector3{p[0], p[1], p[2]}}; break;
        case 6: def.shape = edyn::plane_shape{edyn::vector3{p[0], p[1], p[2]}, p[3]}; break;
        default: break;
        }
        def.presentation = false;
        w->bodies.push_back(edyn::make_rigidbody(w->registry, def));
    }
    edyn::update(w->registry);
    return w;
}
RR_API void rr_destroy(void *h) {
    auto *w = static_cast<World *>(h);
    edyn::detach(w->registry);
    delete w;
}
// edyn::raycast(registry, p0, p1, ignore_entities); ignore and *body are body indices (*body = 0xFFFFFFFF for entt::null).
RR_API void rr_raycast(void *h, const float *p0, const float *p1, const uint32_t *ignore, uint32_t n, uint32_t *body, float *out4,
                       uint32_t *feature) {
    auto *w = static_cast<World *>(h);
    std::vector<entt::entity> ign;
    for (uint32_t i = 0; i < n; ++i) ign.push_back(w->bodies[ignore[i]]);
    const auto r = edyn::raycast(w->registry, v3(p0), v3(p1), ign);
    put(r, out4, feature);
    *body = 0xFFFFFFFFu;
    for (size_t i = 0; i < w->bodies.size(); ++i) if (w->bodies[i] == r.entity) *body = uint32_t(i);
}
