// The ReLU instantiations of the policy kernels and their launchers (namespace promp::relu_tu), compiled apart from the tanh
// ones in policy.cu; see the note at the top of policy.cu.  The phase-clock experiment build instruments the tanh kernels only.
#undef PROMP_EXP_CLOCKS
#define PROMP_POLICY_RELU_TU
#include "policy.cu"
