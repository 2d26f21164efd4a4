// TEST INFRASTRUCTURE.  tests/presentation/_build/liborapres.so: the restatement of ora_presentation.hpp behind a C entry
// point, for tests/test_stepper_b2d_presentation.py (against the reference) and tests/emu/presentation.py (against the
// device kernel under the CPU emulation).  Needs nothing but a C++ compiler.
#include "ora_presentation.hpp"

extern "C" __attribute__((visibility("default")))
void orap_presentation(uint32_t n, int snap, float dt, const float *pos, const float *orn, const float *lv, const float *av,
                       const uint32_t *kind, const uint32_t *asleep, const uint32_t *present, float *ppos, float *porn) {
    ora::presentation(n, snap, dt, pos, orn, lv, av, kind, asleep, present, ppos, porn);
}
