// TEST INFRASTRUCTURE: the batched Frame::ComputeStereoMatches kernels on the CUDA-on-CPU shim, through the library's real launcher.
// A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu_stereo.py calls it.
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_internal.h"
#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

int emu_stereo_idx_cap(int cap, const float* scale, int n_levels, int n_rows) { return stereo_row_index_cap(cap, scale, n_levels, n_rows); }

// n_pairs pairs as one batch of 2 n_pairs frame slots (left images in [0, n), right ones in [n, 2n)).  levels: per slot, the level images
// packed one after the other (row stride = level width, lw / lh per level); n_kp / kps / desc: per slot [cap] keypoints and descriptors.
// -> depth / uright [2 n_pairs][cap] (the left slots are written), row_start [n_pairs][lh[0] + 1], row_idx [n_pairs][idx_cap].
int emu_stereo_matches(int n_pairs, int n_levels, const int* lw, const int* lh, const float* scale, const float* inv_scale, const uint8_t* levels,
                       const int* n_kp, const rgbl_keypoint* kps, const uint8_t* desc, int cap, float mb, float mbf, float* depth, float* uright,
                       int* row_start, int* row_idx) {
    std::vector<LevelGeom> lg(n_levels);
    size_t off = 0;
    for (int l = 0; l < n_levels; ++l) {
        lg[l] = LevelGeom{};
        lg[l].w = lw[l]; lg[l].h = lh[l]; lg[l].pitch = lw[l]; lg[l].off = (int)off;
        off += (size_t)lw[l] * lh[l];
    }
    StereoBatchDev s{};
    s.pyr = levels; s.frame_stride = off; s.levels = lg.data();
    s.kps = kps; s.desc = desc; s.n_sel = n_kp; s.cap = cap;
    s.l0 = 0; s.r0 = n_pairs; s.n_rows = lh[0];
    for (int l = 0; l < n_levels; ++l) { s.scale[l] = scale[l]; s.inv_scale[l] = inv_scale[l]; }
    s.mb = mb; s.mbf = mbf;
    s.depth = depth; s.uright = uright;
    std::vector<int> sad((size_t)n_pairs * cap);
    s.row_start = row_start; s.row_idx = row_idx; s.idx_cap = stereo_row_index_cap(cap, scale, n_levels, lh[0]); s.sad = sad.data();
    launch_stereo_matches(nullptr, s, n_pairs);
    return 0;
}

}  // extern "C"
