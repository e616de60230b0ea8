// The tanh-output instantiations of the policy kernels with tanh hidden layers, and their launchers (namespace
// promp::otanh_tu), compiled apart from the other units; see the note at the top of policy.cu.
#undef PROMP_EXP_CLOCKS
#define PROMP_POLICY_OTANH_TU
#include "policy.cu"
