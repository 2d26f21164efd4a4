// TEST INFRASTRUCTURE.  tests/integration/b2d_mock.cpp (the oracle behind include/b2d.h) extended by the presentation
// entry points, for the CPU suite's run of the EnTT binding's update() (tests/test_stepper_b2d_presentation.py).  The mock
// is compiled here unchanged, with its b2d_add_bodies / b2d_remove_bodies / b2d_destroy renamed so that the wrappers below can record
// which bodies have presentation; the present transforms are kept here and computed by the restatement in
// ora_presentation.hpp from the oracle's state.
#define b2d_add_bodies b2d_mock_add_bodies
#define b2d_remove_bodies b2d_mock_remove_bodies
#define b2d_destroy b2d_mock_destroy
#include "../integration/b2d_mock.cpp"
#undef b2d_add_bodies
#undef b2d_remove_bodies
#undef b2d_destroy
#include "ora_presentation.hpp"
#include <map>

namespace {
struct Presentation { std::vector<uint32_t> kind, present; std::vector<float> ppos, porn; };
std::map<const b2d_world *, Presentation> g_pres;

// state, sleeping flags and present arrays of all bodies
void gather(b2d_world *w, std::vector<float> &pos, std::vector<float> &orn, std::vector<float> &lv, std::vector<float> &av,
            std::vector<uint32_t> &asleep) {
    const uint32_t n = ora_num_bodies(w->ora);
    pos.resize(3 * n); orn.resize(4 * n); lv.resize(3 * n); av.resize(3 * n); asleep.resize(n);
    ora_get_state(w->ora, pos.data(), orn.data(), lv.data(), av.data(), nullptr, nullptr);
    ora_get_sleeping(w->ora, asleep.data());
}
int run(b2d_world *w, int snap, float dt) {
    auto &p = g_pres[w];
    std::vector<float> pos, orn, lv, av; std::vector<uint32_t> asleep;
    gather(w, pos, orn, lv, av, asleep);
    ora::presentation(uint32_t(p.kind.size()), snap, dt, pos.data(), orn.data(), lv.data(), av.data(), p.kind.data(), asleep.data(),
                      p.present.data(), p.ppos.data(), p.porn.data());
    return B2D_OK;
}
}

extern "C" {
void b2d_destroy(b2d_world *w) { g_pres.erase(w); b2d_mock_destroy(w); }
int b2d_add_bodies(b2d_world *w, const b2d_bodies *b, uint32_t *first_id) {
    uint32_t first = 0;
    const int rc = b2d_mock_add_bodies(w, b, &first);
    if (rc != B2D_OK) return rc;
    auto &p = g_pres[w];
    for (uint32_t i = 0; i < b->count; ++i) {
        p.kind.push_back(b->kind[i]);
        p.present.push_back(b->presentation && b->presentation[i] ? 1u : 0u);
        p.ppos.insert(p.ppos.end(), b->pos + 3 * i, b->pos + 3 * i + 3);
        p.porn.insert(p.porn.end(), b->orn + 4 * i, b->orn + 4 * i + 4);
    }
    if (first_id) *first_id = first;
    return B2D_OK;
}
int b2d_remove_bodies(b2d_world *w, const uint32_t *ids, uint32_t n) {
    auto &p = g_pres[w];
    for (uint32_t k = 0; k < n; ++k) if (ids[k] < p.present.size()) { p.present[ids[k]] = 0; p.kind[ids[k]] = B2D_STATIC; }
    return b2d_mock_remove_bodies(w, ids, n);
}
int b2d_update_presentation(b2d_world *w, float dt) { return run(w, 0, dt); }
int b2d_snap_presentation(b2d_world *w) { return run(w, 1, 0.0f); }
// bodies without presentation report position / orientation, as include/b2d.h states
int b2d_download_presentation(b2d_world *w, float *pos, float *orn) {
    auto &p = g_pres[w];
    std::vector<float> sp, so, lv, av; std::vector<uint32_t> asleep;
    gather(w, sp, so, lv, av, asleep);
    for (size_t i = 0; i < p.present.size(); ++i) {
        for (int k = 0; k < 3; ++k) if (pos) pos[3 * i + k] = p.present[i] ? p.ppos[3 * i + k] : sp[3 * i + k];
        for (int k = 0; k < 4; ++k) if (orn) orn[4 * i + k] = p.present[i] ? p.porn[4 * i + k] : so[4 * i + k];
    }
    return B2D_OK;
}
}
