// The tanh-output instantiations of the policy kernels with ReLU hidden layers, and their launchers (namespace
// promp::relu_otanh_tu), compiled apart from the other units; see the note at the top of policy.cu.
#undef PROMP_EXP_CLOCKS
#define PROMP_POLICY_RELU_TU
#define PROMP_POLICY_OTANH_TU
#include "policy.cu"
