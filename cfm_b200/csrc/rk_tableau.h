// Dormand-Prince 5(4) coefficients, one definition for both ODE drivers: rk.cu (device constants and compile-time
// stage rows) and ode_small.cu (device constants).  torchdyn's DormandPrince45 tableau (un-vendored dependency,
// SURVEY.md Appendix B), pinned against SciPy's RK45 in tests/test_oracle.py.
#pragma once

#define CFM_RK_C_INIT {0.f, 1.f / 5, 3.f / 10, 4.f / 5, 8.f / 9, 1.f, 1.f}
#define CFM_RK_A_INIT {                                                                     \
    {0, 0, 0, 0, 0, 0},                                                                     \
    {1.f / 5, 0, 0, 0, 0, 0},                                                               \
    {3.f / 40, 9.f / 40, 0, 0, 0, 0},                                                       \
    {44.f / 45, -56.f / 15, 32.f / 9, 0, 0, 0},                                             \
    {19372.f / 6561, -25360.f / 2187, 64448.f / 6561, -212.f / 729, 0, 0},                  \
    {9017.f / 3168, -355.f / 33, 46732.f / 5247, 49.f / 176, -5103.f / 18656, 0},           \
    {35.f / 384, 0.f, 500.f / 1113, 125.f / 192, -2187.f / 6784, 11.f / 84}}
/* b5 - b4 (embedded error weights), k1..k7 */
#define CFM_RK_E_INIT {(float)(35.0 / 384 - 1951.0 / 21600), 0.f,                           \
                       (float)(500.0 / 1113 - 22642.0 / 50085),                             \
                       (float)(125.0 / 192 - 451.0 / 720),                                  \
                       (float)(-2187.0 / 6784 + 12231.0 / 42400),                           \
                       (float)(11.0 / 84 - 649.0 / 6300), (float)(-1.0 / 60)}
