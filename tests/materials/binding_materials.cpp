// TEST INFRASTRUCTURE.  The EnTT binding's harness (tests/integration/stepper_b2d_capi.cpp: a real Edyn registry stepped by
// edyn::stepper_b2d) with the material entry points of refm.hpp and two user actions the binding refuses.  Linked with
// edyn_b200/libb2d.so (tests/test_gpu_binding_materials.py) and with the C ABI mock (tests/test_stepper_b2d_materials.py).
#include "../integration/stepper_b2d_capi.cpp"
#include "refm.hpp"

// emplace (on != 0) or remove the material component of a body: a change between sensor and non-sensor
REFS_API void refm_toggle_material(void *h, uint32_t body, int on) {
    auto *w = static_cast<World *>(h);
    if (on) w->registry.emplace<edyn::material>(w->bodies[body]);
    else w->registry.remove<edyn::material>(w->bodies[body]);
}
// a material_mix_table entry with a contact extra (spin friction), which the device does not support
REFS_API void refm_insert_spin_mixing(void *h, uint32_t id0, uint32_t id1, float spin_friction) {
    edyn::material_base m; m.spin_friction = spin_friction;
    static_cast<World *>(h)->registry.ctx().get<edyn::material_mix_table>().insert({edyn::material::id_type(id0), edyn::material::id_type(id1)}, m);
}
