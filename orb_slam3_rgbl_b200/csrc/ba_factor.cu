// The reduced-system factorisation of bundle adjustment (ba_factor.cuh): the kernels, ba_solve_reduced and, in the test-only library,
// rgbl_testing_reduced_solve.  Built with FMA contraction like api_ba.cu (csrc/Makefile).
#include "ba_factor.cuh"
