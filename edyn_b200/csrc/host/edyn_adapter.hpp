// C++17 host adapter over the C ABI (include/b2d.h): keeps the reference's public names for the sequential
// stepper so application code reads like Edyn code --
//     edyn::attach / detach            src/edyn/edyn.cpp:73-141, :148-197
//     edyn::make_rigidbody             src/edyn/util/rigidbody.cpp:47-185
//     edyn::make_hinge (make_constraint<hinge_constraint> + set_axes)   include/edyn/util/constraint_util.hpp:38-54
//     edyn::exclude_collision          src/edyn/util/exclude_collision.cpp
//     edyn::raycast                    src/edyn/collision/raycast.cpp:20-56
//     edyn::update / step_simulation   src/edyn/edyn.cpp:233-273, stepper_sequential.cpp:28-147
//     edyn::set_fixed_dt / set_solver_velocity_iterations / set_solver_position_iterations
// EnTT is not available in this image, so the "registry" here is a minimal component store with the same component
// layout (position, orientation, linvel, angvel, AABB ...); INTEGRATION.md shows the identical staging written against a
// real entt::registry.  Header-only; link with edyn_b200/libb2d.so.  There is no CPU fallback: attach() throws if the
// device world cannot be created.
#pragma once
#include "../../../include/b2d.h"
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <optional>
#include <stdexcept>
#include <string>
#include <variant>
#include <vector>

namespace edyn {

using scalar = float;
struct vector3 { scalar x{}, y{}, z{}; };
struct quaternion { scalar x{}, y{}, z{}, w{1}; };
using entity = std::uint32_t;                       // body id on the device == index in the registry below
inline constexpr entity null = 0xFFFFFFFFu;

struct sphere_shape { scalar radius; };
struct capsule_shape { scalar radius, half_length; int axis{0}; };
struct box_shape { vector3 half_extents; };
struct plane_shape { vector3 normal; scalar constant; };
using shapes_variant_t = std::variant<sphere_shape, capsule_shape, box_shape, plane_shape>;

struct material_base { scalar restitution{0}; scalar friction{0.5f}; };
// material::id keys the mixing table (insert_material_mixing); UnassignedID never matches an entry
struct material : material_base { using id_type = std::uint16_t; static constexpr id_type UnassignedID = 0xFFFF; id_type id{UnassignedID}; };
enum class rigidbody_kind : std::uint8_t { rb_dynamic, rb_kinematic, rb_static };

struct rigidbody_def {                               // include/edyn/util/rigidbody.hpp
    rigidbody_kind kind{rigidbody_kind::rb_dynamic};
    vector3 position{}; quaternion orientation{};
    scalar mass{1};
    std::optional<std::array<scalar, 9>> inertia;    // row-major; computed from the shape when absent
    vector3 linvel{}, angvel{};
    std::optional<vector3> gravity;                  // default: registry gravity
    std::optional<shapes_variant_t> shape;
    std::optional<edyn::material> material{edyn::material{}};
    std::uint64_t collision_group{~0ull}, collision_mask{~0ull};
    bool presentation{true};                         // present_position / present_orientation (dynamic bodies only)
};

struct init_config {                                 // include/edyn/edyn.hpp:39-60 (+ device capacities)
    scalar fixed_dt{scalar(1.0 / 60)};
    int device{0};
    std::uint32_t max_bodies{1u << 16}, max_manifolds{1u << 19}, max_hinges{0};
    unsigned num_solver_velocity_iterations{8}, num_solver_position_iterations{3};
    vector3 gravity{0, scalar(-9.8), 0};
    bool sleeping{false};                            // false = rigidbody_def::sleeping_disabled on every body (benchmark configurations)
};

struct AABB { vector3 min, max; };

// Component store + device world: what registry.ctx() holds after edyn::attach in the reference.
class registry {
public:
    // components, SoA (same fields the reference keeps per entity)
    std::vector<scalar> position, orientation, linvel, angvel, aabb;      // 3n, 4n, 3n, 3n, 6n
    // present_position / present_orientation, refreshed by every update(); bodies without them hold position / orientation
    std::vector<scalar> present_position, present_orientation;           // 3n, 4n
    std::size_t size() const { return position.size() / 3; }

    vector3 get_position(entity e) const { return {position[3 * e], position[3 * e + 1], position[3 * e + 2]}; }
    quaternion get_orientation(entity e) const { return {orientation[4 * e], orientation[4 * e + 1], orientation[4 * e + 2], orientation[4 * e + 3]}; }
    vector3 get_linvel(entity e) const { return {linvel[3 * e], linvel[3 * e + 1], linvel[3 * e + 2]}; }
    AABB get_aabb(entity e) const { return {{aabb[6 * e], aabb[6 * e + 1], aabb[6 * e + 2]}, {aabb[6 * e + 3], aabb[6 * e + 4], aabb[6 * e + 5]}}; }
    // writes go through these so the next update() re-stages them (the reference's patch/replace contract)
    void set_linvel(entity e, vector3 v) { linvel[3 * e] = v.x; linvel[3 * e + 1] = v.y; linvel[3 * e + 2] = v.z; dirty = true; }
    void set_position(entity e, vector3 v) { position[3 * e] = v.x; position[3 * e + 1] = v.y; position[3 * e + 2] = v.z; dirty = true; }

    b2d_world *world{nullptr};
    init_config config;
    double accumulated{0};
    unsigned max_steps_per_update{10};               // settings.max_steps_per_update
    bool dirty{false}, paused{false};
};

namespace detail {
inline void check(registry &r, int rc, const char *what) {
    if (rc != B2D_OK) throw std::runtime_error(std::string(what) + ": " + b2d_last_error(r.world));
}
// dynamics/moment_of_inertia.cpp:11-91 + matrix3x3.hpp:177-204 for the in-scope shapes (diagonal tensors)
inline std::array<scalar, 9> inverse_inertia(const shapes_variant_t &sh, scalar mass) {
    scalar ix = 0, iy = 0, iz = 0;
    if (auto *s = std::get_if<sphere_shape>(&sh)) { ix = iy = iz = scalar(0.4) * mass * s->radius * s->radius; }
    else if (auto *b = std::get_if<box_shape>(&sh)) {
        scalar ex = b->half_extents.x * 2, ey = b->half_extents.y * 2, ez = b->half_extents.z * 2;
        scalar k = scalar(1) / scalar(12) * mass;
        ix = k * (ey * ey + ez * ez); iy = k * (ez * ez + ex * ex); iz = k * (ex * ex + ey * ey);
    } else if (auto *c = std::get_if<capsule_shape>(&sh)) {
        const scalar pi = scalar(3.1415926535897932384626433832795029);
        scalar r = c->radius, len = c->half_length * 2;
        scalar cyl_vol = pi * r * r * len, sph_vol = pi * r * r * r * scalar(4) / scalar(3), total = cyl_vol + sph_vol;
        scalar cyl_mass = mass * cyl_vol / total, sph_mass = mass * sph_vol / total;
        scalar cxx = scalar(0.5) * cyl_mass * r * r, cyz = scalar(1) / scalar(12) * cyl_mass * (scalar(3) * r * r + len * len);
        scalar cyl[3] = {cyz, cyz, cyz}; cyl[c->axis] = cxx;       // axis-permuted first, read as .x/.y afterwards (:27-44, :76-77)
        scalar sph_i = scalar(0.4) * sph_mass * r * r;
        scalar xx = sph_i + cyl[0];
        scalar t = scalar(4) * len + scalar(3) * r;
        scalar yy = sph_i + sph_mass * (t * t) / scalar(64) + cyl[1];
        scalar d[3] = {yy, yy, yy}; d[c->axis] = xx; ix = d[0]; iy = d[1]; iz = d[2];
    } else throw std::runtime_error("dynamic bodies need a sphere, capsule or box shape");
    scalar det_inv = scalar(1) / (ix * (iy * iz));
    return {det_inv * (iy * iz), 0, 0, 0, det_inv * (ix * iz), 0, 0, 0, det_inv * (ix * iy)};
}
inline void pull(registry &r) {
    const std::size_t n = r.size();
    detail::check(r, b2d_download_state(r.world, r.position.data(), r.orientation.data(), r.linvel.data(), r.angvel.data(), r.aabb.data(), nullptr),
                  "b2d_download_state");
    (void)n;
}
inline void push(registry &r) {
    if (r.dirty) { detail::check(r, b2d_upload_state(r.world, r.position.data(), r.orientation.data(), r.linvel.data(), r.angvel.data()), "b2d_upload_state"); r.dirty = false; }
}
inline void pull_presentation(registry &r) {
    if (!r.size()) return;
    detail::check(r, b2d_download_presentation(r.world, r.present_position.data(), r.present_orientation.data()), "b2d_download_presentation");
}
}  // namespace detail

inline void attach(registry &r, const init_config &config = {}) {
    r.config = config;
    b2d_config c{};
    c.device = config.device; c.max_bodies = config.max_bodies; c.max_manifolds = config.max_manifolds; c.max_hinges = config.max_hinges;
    c.fixed_dt = config.fixed_dt; c.velocity_iterations = config.num_solver_velocity_iterations;
    c.position_iterations = config.num_solver_position_iterations;
    c.flags = config.sleeping ? B2D_FLAG_SLEEPING : 0u;
    r.world = b2d_create(&c);
    if (!r.world) throw std::runtime_error(std::string("edyn::attach: ") + b2d_last_error(nullptr));
}
inline void detach(registry &r) { b2d_destroy(r.world); r.world = nullptr; }

inline entity make_rigidbody(registry &r, const rigidbody_def &def) {
    const bool dyn = def.kind == rigidbody_kind::rb_dynamic;
    std::uint32_t kind = dyn ? B2D_DYNAMIC : (def.kind == rigidbody_kind::rb_kinematic ? B2D_KINEMATIC : B2D_STATIC);
    std::uint32_t sk = B2D_SHAPE_NONE; float sp[4] = {0, 0, 0, 0};
    if (def.shape) {
        if (auto *s = std::get_if<sphere_shape>(&*def.shape)) { sk = B2D_SHAPE_SPHERE; sp[0] = s->radius; }
        else if (auto *c = std::get_if<capsule_shape>(&*def.shape)) { sk = B2D_SHAPE_CAPSULE; sp[0] = c->radius; sp[1] = c->half_length; sp[2] = float(c->axis); }
        else if (auto *b = std::get_if<box_shape>(&*def.shape)) { sk = B2D_SHAPE_BOX; sp[0] = b->half_extents.x; sp[1] = b->half_extents.y; sp[2] = b->half_extents.z; }
        else if (auto *p = std::get_if<plane_shape>(&*def.shape)) { sk = B2D_SHAPE_PLANE; sp[0] = p->normal.x; sp[1] = p->normal.y; sp[2] = p->normal.z; sp[3] = p->constant; }
    }
    float pos[3] = {def.position.x, def.position.y, def.position.z};
    float orn[4] = {def.orientation.x, def.orientation.y, def.orientation.z, def.orientation.w};
    float lv[3] = {def.linvel.x, def.linvel.y, def.linvel.z}, av[3] = {def.angvel.x, def.angvel.y, def.angvel.z};
    float inv_mass = dyn ? scalar(1) / def.mass : 0;
    std::array<scalar, 9> inv_I{};
    if (dyn) {
        if (def.inertia) { auto &I = *def.inertia; scalar di = scalar(1) / (I[0] * (I[4] * I[8])); inv_I = {di * (I[4] * I[8]), 0, 0, 0, di * (I[0] * I[8]), 0, 0, 0, di * (I[0] * I[4])}; }
        else inv_I = detail::inverse_inertia(*def.shape, def.mass);
    }
    vector3 g = dyn ? def.gravity.value_or(r.config.gravity) : vector3{};
    float grav[3] = {g.x, g.y, g.z};
    float fr = def.material ? def.material->friction : 0, re = def.material ? def.material->restitution : 0;
    std::uint64_t grp = def.collision_group, msk = def.collision_mask;
    std::uint32_t mat = def.material ? std::uint32_t(def.material->id) : B2D_MATERIAL_NONE;      // no material: a sensor
    std::uint32_t pre = def.presentation && dyn ? 1u : 0u;          // util/rigidbody.cpp:99-102
    b2d_bodies b{1, pos, orn, lv, av, &inv_mass, inv_I.data(), grav, &kind, &sk, sp, &fr, &re, &grp, &msk, &mat, &pre};
    std::uint32_t id = 0;
    detail::check(r, b2d_add_bodies(r.world, &b, &id), "b2d_add_bodies");
    r.position.insert(r.position.end(), pos, pos + 3); r.orientation.insert(r.orientation.end(), orn, orn + 4);
    r.linvel.insert(r.linvel.end(), lv, lv + 3); r.angvel.insert(r.angvel.end(), av, av + 3);
    r.aabb.resize(r.aabb.size() + 6);
    r.present_position.insert(r.present_position.end(), pos, pos + 3); r.present_orientation.insert(r.present_orientation.end(), orn, orn + 4);
    return id;
}

inline void make_hinge(registry &r, entity a, entity b, vector3 pivot_a, vector3 pivot_b, vector3 axis_a, vector3 axis_b) {
    float pa[3] = {pivot_a.x, pivot_a.y, pivot_a.z}, pb[3] = {pivot_b.x, pivot_b.y, pivot_b.z};
    float xa[3] = {axis_a.x, axis_a.y, axis_a.z}, xb[3] = {axis_b.x, axis_b.y, axis_b.z};
    detail::check(r, b2d_add_hinges(r.world, 1, &a, &b, pa, pb, xa, xb), "b2d_add_hinges");
}
// edyn::insert_material_mixing (util/insert_material_mixing.cpp:9-22): contact points created from now on between bodies of
// material ids id0 and id1 (either order) take this friction and restitution instead of the mixed ones
inline void insert_material_mixing(registry &r, material::id_type id0, material::id_type id1, const material_base &m) {
    std::uint32_t a = id0, b = id1; float f = m.friction, e = m.restitution;
    detail::check(r, b2d_set_material_mixing(r.world, 1, &a, &b, &f, &e), "b2d_set_material_mixing");
}
inline void exclude_collision(registry &r, entity a, entity b) { detail::check(r, b2d_add_exclusions(r.world, 1, &a, &b), "b2d_add_exclusions"); }

// edyn::raycast_result (include/edyn/collision/raycast.hpp:103-136).  info: box face index, capsule hemisphere index or
// B2D_RAY_CAPSULE_SIDE, B2D_RAY_FEATURE_NONE for spheres, planes and misses; entity == null on a miss.
struct raycast_result {
    scalar fraction{3.402823466e+38f};                  // EDYN_SCALAR_MAX on a miss
    vector3 normal{};
    std::uint32_t info{B2D_RAY_FEATURE_NONE};
    edyn::entity entity{null};
};
// edyn::raycast(registry, p0, p1, ignore_entities) (src/edyn/collision/raycast.cpp:20-56); semantics in include/b2d.h.
inline raycast_result raycast(registry &r, vector3 p0, vector3 p1, const std::vector<entity> &ignore_entities = {}) {
    if (r.dirty) { detail::check(r, b2d_upload_state(r.world, r.position.data(), r.orientation.data(), r.linvel.data(), r.angvel.data()), "b2d_upload_state"); r.dirty = false; }
    const float a[3] = {p0.x, p0.y, p0.z}, b[3] = {p1.x, p1.y, p1.z};
    float n[3];
    raycast_result res;
    detail::check(r, b2d_raycast(r.world, 1, a, b, nullptr, ignore_entities.empty() ? nullptr : ignore_entities.data(),
                                 std::uint32_t(ignore_entities.size()), &res.entity, &res.fraction, n, &res.info), "b2d_raycast");
    res.normal = {n[0], n[1], n[2]};
    return res;
}

// registry.destroy(entity) of a rigid body: its manifolds and joints go with it (island_manager.cpp:47-66); ids are not reused.
inline void destroy_rigidbody(registry &r, entity e) { detail::check(r, b2d_remove_bodies(r.world, &e, 1), "b2d_remove_bodies"); }
// edyn::wake_up_entity (util/island_util.cpp)
inline void wake_up_entity(registry &r, entity e) { detail::check(r, b2d_wake_bodies(r.world, &e, 1), "b2d_wake_bodies"); }
// presence of sleeping_tag
inline bool is_sleeping(registry &r, entity e) {
    std::vector<std::uint32_t> asleep(r.position.size() / 3 + 1);
    detail::check(r, b2d_download_sleeping(r.world, asleep.data()), "b2d_download_sleeping");
    return asleep[e] != 0;
}

// edyn::set_paused (stepper_sequential.cpp:148-151): the accumulator restarts from zero
inline void set_paused(registry &r, bool paused) { r.paused = paused; r.accumulated = 0; }

// One fixed step (step_simulation semantics, stepper_sequential.cpp:121-147).
inline void step_simulation(registry &r) {
    detail::push(r);
    detail::check(r, b2d_step(r.world, 1), "b2d_step");
    detail::pull(r);
}

// edyn::update(registry, time): accumulate elapsed time, run floor(acc / fixed_dt) steps, capped (stepper_sequential.cpp:45-65),
// then update_presentation with interpolation_dt = min(float(acc - fixed_dt), fixed_dt), the elapsed-time form of
// stepper_sequential.cpp:104-105; while paused, snap_presentation (:37-43).  One presentation download per call.
inline unsigned update(registry &r, double elapsed) {
    detail::push(r);
    if (r.paused) {
        detail::check(r, b2d_snap_presentation(r.world), "b2d_snap_presentation");
        detail::pull_presentation(r);
        return 0;
    }
    r.accumulated += elapsed;
    unsigned n = unsigned(std::floor(r.accumulated / r.config.fixed_dt));
    r.accumulated -= double(n) * r.config.fixed_dt;
    if (n > r.max_steps_per_update) n = r.max_steps_per_update;
    if (n) {
        detail::check(r, b2d_step(r.world, n), "b2d_step");
        detail::pull(r);
    }
    const float dt = std::min(float(r.accumulated - double(r.config.fixed_dt)), float(r.config.fixed_dt));
    detail::check(r, b2d_update_presentation(r.world, dt), "b2d_update_presentation");
    detail::pull_presentation(r);
    return n;
}

}  // namespace edyn
