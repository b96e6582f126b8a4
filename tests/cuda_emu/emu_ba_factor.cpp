// The reduced-system factorisation of bundle adjustment (csrc/ba_factor.cuh) in the emulated library: its kernels, ba_solve_reduced (called
// by api_ba.cu's LM driver) and the test export rgbl_testing_reduced_solve, compiled from build.py's transformed copy of the header.
#include "ba_factor.cuh"
