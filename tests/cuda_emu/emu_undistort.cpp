// TEST INFRASTRUCTURE: Frame::UndistortKeyPoints / ComputeImageBounds of a distorted camera on the CUDA-on-CPU shim, through the
// library's real launcher and host helpers (tests/test_cuda_emu_undistort.py builds this file against depth_kernels.cu).
#include "cuda_runtime.h"

#include "depth_kernels.emu.cpp"

using namespace rgbl;

extern "C" {

// n_frames keypoint lists ([n_frames][cap], n_kp[f] valid) -> kps_un (same layout) with launch_undistort_keypoints
int emu_undistort_keypoints(float fx, float fy, float cx, float cy, const float* dist, int n_dist, const rgbl_keypoint* kps, const int* n_kp, int cap,
                            int n_frames, rgbl_keypoint* kps_un) {
    const UndistortDev m = make_undistort_dev(fx, fy, cx, cy, dist, n_dist);
    int max_n = 0;
    for (int f = 0; f < n_frames; ++f) max_n = n_kp[f] > max_n ? n_kp[f] : max_n;
    launch_undistort_keypoints(nullptr, m, kps, n_kp, cap, max_n, kps_un, n_frames);
    return 0;
}

// the bounds rgbl_set_camera_distortion computes on the host
int emu_image_bounds(float fx, float fy, float cx, float cy, const float* dist, int n_dist, int W, int H, float* bounds) {
    image_bounds(make_undistort_dev(fx, fy, cx, cy, dist, n_dist), dist[0], W, H, bounds);
    return 0;
}

}  // extern "C"
