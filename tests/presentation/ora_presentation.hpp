// TEST INFRASTRUCTURE.  CPU restatement of the reference's update_presentation / snap_presentation
// (src/edyn/sys/update_presentation.cpp:56-93) over packed arrays, in the oracle's float arithmetic (oracle/ora_math.hpp:
// the same integrate as the step).  It is what k_presentation (edyn_b200/csrc/b2d_kernels.cuh) computes:
//   update (snap = 0): bodies with presentation that are dynamic (procedural_tag) and not asleep (the linear and angular
//                      views exclude sleeping_tag): pre = pos + linvel dt, pre_orn = integrate(orn, angvel, dt);
//   snap   (snap = 1): every body with presentation: pre = pos, pre_orn = orn.
// Other bodies' ppos / porn are left as they are.  Arrays are packed: 3n / 4n floats, n words.
#pragma once
#include "../../oracle/ora_math.hpp"

namespace ora {

inline void presentation(uint32_t n, int snap, float dt, const float *pos, const float *orn, const float *lv, const float *av,
                         const uint32_t *kind, const uint32_t *asleep, const uint32_t *present, float *ppos, float *porn) {
    for (uint32_t i = 0; i < n; ++i) {
        if (!present[i]) continue;
        const vec3 p{pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
        const quat q{orn[4 * i], orn[4 * i + 1], orn[4 * i + 2], orn[4 * i + 3]};
        vec3 pp; quat pq;
        if (snap) { pp = p; pq = q; }
        else if (kind[i] == 0 && !asleep[i]) {
            pp = p + vec3{lv[3 * i], lv[3 * i + 1], lv[3 * i + 2]} * dt;
            pq = integrate(q, vec3{av[3 * i], av[3 * i + 1], av[3 * i + 2]}, dt);
        } else continue;
        ppos[3 * i] = pp.x; ppos[3 * i + 1] = pp.y; ppos[3 * i + 2] = pp.z;
        porn[4 * i] = pq.x; porn[4 * i + 1] = pq.y; porn[4 * i + 2] = pq.z; porn[4 * i + 3] = pq.w;
    }
}

} // namespace ora
