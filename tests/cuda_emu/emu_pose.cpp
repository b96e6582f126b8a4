// TEST INFRASTRUCTURE: pose_optimize_kernel through its launcher on the CUDA-on-CPU shim, with the per-edge state the C ABI does not
// return: level[] (the edge levels the rounds ran with) and work[] (the errors the classification read).  A unit of the emulated
// library (tests/cuda_emu/build.py); tests/test_cuda_emu_pose_replica.py calls it.
#include <cstring>

#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

int emu_pose_optimize(const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2, const uint8_t* stereo,
                      float fx, float fy, float cx, float cy, float bf, float pose_out[7], uint8_t* outlier, uint8_t* level, double* work,
                      int* n_inliers) {
    PoseProblemDev p;
    p.n = n; p.n_dev = nullptr; p.pose_in_dev = nullptr;
    p.xw = xw; p.obs = obs; p.inv_sigma2 = inv_sigma2; p.stereo = stereo;
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = bf;
    std::memcpy(p.pose_in, pose_in, 7 * sizeof(float));
    launch_pose_optimize(nullptr, p, work, level, outlier, pose_out, n_inliers, nullptr, 1);
    return cudaStreamSynchronize(nullptr) == cudaSuccess ? 0 : -1;
}

}  // extern "C"
