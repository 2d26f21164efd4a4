// TEST INFRASTRUCTURE.  tests/integration/stepper_b2d_capi.cpp (a real Edyn registry stepped by edyn::stepper_b2d, next to
// the reference's own stepper) extended for the presentation transforms: the reference's edyn::update / set_paused /
// step_simulation next to the binding's, on registries built the same way, and the reference's update_presentation /
// snap_presentation on given states.  One translation unit with the harness, so that it reaches the harness's worlds and
// steppers.  Linked once against b2d_mock_presentation.cpp (CPU suite) and once against edyn_b200/libb2d.so (-m gpu).
#include "../integration/stepper_b2d_capi.cpp"
#include <edyn/comp/present_orientation.hpp>
#include <edyn/comp/present_position.hpp>
#include <edyn/sys/update_presentation.hpp>
#include <limits>

// A body gets present_position / present_orientation as make_rigidbody emplaces them
// with rigidbody_def::presentation (util/rigidbody.cpp:99-102): at its current transform, before the next update.
namespace {
std::map<const entt::registry *, uint64_t> g_step_count;
void count_step(entt::registry &r) { ++g_step_count[&r]; }
}
REFS_API void eb2d_add_presentation(void *h, uint32_t body) {
    auto *w = static_cast<World *>(h);
    const auto e = w->bodies[body];
    w->registry.emplace<edyn::present_position>(e, w->registry.get<edyn::position>(e));
    w->registry.emplace<edyn::present_orientation>(e, w->registry.get<edyn::orientation>(e));
}
// steps run by whichever stepper drives the registry since the first call on it (settings.post_step_callback)
REFS_API uint64_t eb2d_count_steps(void *h) {
    auto &r = static_cast<World *>(h)->registry;
    auto &s = r.ctx().get<edyn::settings>();
    if (s.post_step_callback != &count_step) { s.post_step_callback = &count_step; g_step_count[&r] = 0; }   // first call: start counting
    return g_step_count[&r];
}
// out: present_position / present_orientation per scene body; has[i] = 0 where the body has none (or was destroyed)
REFS_API void eb2d_get_presentation(void *h, float *pos, float *orn, uint32_t *has) {
    auto *w = static_cast<World *>(h);
    auto &r = w->registry;
    for (size_t i = 0; i < w->bodies.size(); ++i) {
        const auto e = w->bodies[i];
        has[i] = r.valid(e) && r.all_of<edyn::present_position, edyn::present_orientation>(e) ? 1u : 0u;
        if (!has[i]) { for (int k = 0; k < 3; ++k) pos[3 * i + k] = 0; for (int k = 0; k < 4; ++k) orn[4 * i + k] = 0; continue; }
        const auto &p = r.get<edyn::present_position>(e); const auto &q = r.get<edyn::present_orientation>(e);
        pos[3 * i] = p.x; pos[3 * i + 1] = p.y; pos[3 * i + 2] = p.z;
        orn[4 * i] = q.x; orn[4 * i + 1] = q.y; orn[4 * i + 2] = q.z; orn[4 * i + 3] = q.w;
    }
}
REFS_API int eb2d_set_paused(void *h, int paused) { stepper(h).set_paused(paused != 0); return 0; }
REFS_API int eb2d_step_simulation(void *h, double time) {
    try { stepper(h).step_simulation(time); } catch (const std::exception &e) { std::fprintf(stderr, "eb2d_step_simulation: %s\n", e.what()); return -1; }
    return 0;
}
// the reference's side: stepper_sequential itself (refs_create leaves it paused; set_paused(false) starts the clock)
REFS_API void eb2d_ref_update(void *h, double time) { edyn::update(static_cast<World *>(h)->registry, time); }
REFS_API void eb2d_ref_set_paused(void *h, int paused) { edyn::set_paused(static_cast<World *>(h)->registry, paused != 0); }
REFS_API void eb2d_ref_step_simulation(void *h, double time) {
    static_cast<World *>(h)->registry.ctx().get<edyn::stepper_sequential>().step_simulation(time);
}
// edyn::update_presentation (snap = 0, interpolation_dt = dt) or edyn::snap_presentation (snap = 1) on n bodies with the
// given state, in a registry of their own.  kind: 0 dynamic (procedural_tag) or other; asleep: sleeping_tag; present: the
// two components.  out: the present transform of bodies with presentation, zeros for the others.
REFS_API void eb2d_ref_presentation(uint32_t n, int snap, float dt, const float *pos, const float *orn, const float *lv, const float *av,
                                    const uint32_t *kind, const uint32_t *asleep, const uint32_t *present, float *out_pos, float *out_orn) {
    entt::registry r;
    auto &s = r.ctx().emplace<edyn::settings>();
    s.fixed_dt = std::numeric_limits<edyn::scalar>::max();     // min(dt, fixed_dt) = dt
    std::vector<entt::entity> es(n);
    for (uint32_t i = 0; i < n; ++i) {
        const auto e = es[i] = r.create();
        r.emplace<edyn::position>(e, v3(pos + 3 * i));
        r.emplace<edyn::orientation>(e, edyn::quaternion{orn[4 * i], orn[4 * i + 1], orn[4 * i + 2], orn[4 * i + 3]});
        r.emplace<edyn::linvel>(e, v3(lv + 3 * i));
        r.emplace<edyn::angvel>(e, v3(av + 3 * i));
        if (kind[i] == 0) r.emplace<edyn::procedural_tag>(e);
        if (asleep[i]) r.emplace<edyn::sleeping_tag>(e);
        if (present[i]) { r.emplace<edyn::present_position>(e, edyn::vector3_zero); r.emplace<edyn::present_orientation>(e, edyn::quaternion_identity); }
    }
    if (snap) edyn::snap_presentation(r);
    else edyn::update_presentation(r, 0.0, double(dt), 0.0, 0.0);       // interpolation_dt = float(dt - 0 - 0)
    for (uint32_t i = 0; i < n; ++i) {
        for (int k = 0; k < 3; ++k) out_pos[3 * i + k] = 0;
        for (int k = 0; k < 4; ++k) out_orn[4 * i + k] = 0;
        if (!present[i]) continue;
        const auto &p = r.get<edyn::present_position>(es[i]); const auto &q = r.get<edyn::present_orientation>(es[i]);
        out_pos[3 * i] = p.x; out_pos[3 * i + 1] = p.y; out_pos[3 * i + 2] = p.z;
        out_orn[4 * i] = q.x; out_orn[4 * i + 1] = q.y; out_orn[4 * i + 2] = q.z; out_orn[4 * i + 3] = q.w;
    }
}
