// TEST INFRASTRUCTURE: the RGB-D device code paths (16-bit depth PNG reconstruction, uint16 depth gather) on the CUDA-on-CPU shim,
// through the library's real launchers.  A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu_rgbd.py calls it.
#include <cstring>
#include <string>
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_internal.h"
#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

// one 16-bit depth PNG stream -> host inflate (png_inflate_batch, depth mode) -> launch_png_unfilter_depth16 into a pitched plane
// -> out (h x w, stride w).  Returns 0, the host decoder's negative code, or -100 for a bad filter byte.
int emu_png_depth16(const uint8_t* png, size_t n, int w, int h, uint16_t* out) {
    const size_t raw_stride = (((size_t)w * 4 + 1) * h + 255) & ~(size_t)255;
    std::vector<uint8_t> raw(raw_stride);
    int ch = 0;
    std::string err;
    const uint8_t* p[1] = {png};
    const size_t nb[1] = {n};
    const int rc = png_inflate_batch(1, p, nb, w, h, raw.data(), raw_stride, &ch, err, true);
    if (rc) return rc;
    const size_t pitch = ((size_t)w * 2 + 63) / 64 * 32;
    std::vector<uint16_t> plane(pitch * h, 0xdead);
    std::vector<uint32_t> band(w);
    int status = 0;
    launch_png_unfilter_depth16(nullptr, raw.data(), raw_stride, w, h, plane.data(), pitch * h, pitch, band.data(), &status, 1);
    if (status) return -100;
    for (int y = 0; y < h; ++y) std::memcpy(out + (size_t)y * w, plane.data() + (size_t)y * pitch, (size_t)w * 2);
    return 0;
}

// ComputeStereoFromRGBD on a uint16 plane (h x w, stride w, copied into a pitched plane): launch_depth_gather_u16 with mvKeysUn == mvKeys
int emu_gather_u16(const uint16_t* img, int w, int h, float scale, const rgbl_keypoint* kps, int n, float bf, float* depth, float* uright) {
    const size_t pitch = ((size_t)w * 2 + 63) / 64 * 32;
    std::vector<uint16_t> plane(pitch * h, 0);
    for (int y = 0; y < h; ++y) std::memcpy(plane.data() + (size_t)y * pitch, img + (size_t)y * w, (size_t)w * 2);
    launch_depth_gather_u16(nullptr, plane.data(), pitch * h, pitch, scale, kps, kps, &n, n, n, bf, depth, uright, 1);
    return 0;
}

}  // extern "C"
