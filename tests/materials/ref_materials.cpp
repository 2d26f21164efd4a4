// TEST INFRASTRUCTURE.  The reference's real stepper (oracle/ref_stepper.cpp) with the material entry points of refm.hpp:
// tests/materials/_build/libref_materials.so, for tests/test_ref_materials.py.
#include "../../oracle/ref_stepper.cpp"
#include "refm.hpp"
