// TEST INFRASTRUCTURE: the stereo rectification kernels (map conversion, batched remap) on the CUDA-on-CPU shim, through the library's
// real launchers.  A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu_rectify.py calls it.
#include "rgbl_device.cuh"
#include "rgbl_internal.h"
#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

// maps = [m1l | m2l | m1r | m2r] (H x W each) -> xy / a [2][H][pitch]
void emu_rectify_maps(const float* maps, int W, int H, uint32_t* xy, uint16_t* a, int pitch) { launch_rectify_maps(nullptr, maps, W, H, xy, a, pitch); }

// raw planes [2 n_pairs][H][src_pitch] -> dst planes [2 n_pairs] of dst_stride bytes, image at dst_off, rows of dst_pitch
void emu_rectify(const uint32_t* xy, const uint16_t* a, int pitch, int W, int H, const uint8_t* src, int src_pitch, uint8_t* dst, size_t dst_stride,
                 int dst_off, int dst_pitch, int n_pairs) {
    RectifyDev r{};
    r.xy = xy; r.a = a; r.map_pitch = pitch; r.W = W; r.H = H;
    r.src = src; r.src_stride = (size_t)src_pitch * H; r.src_pitch = src_pitch;
    r.dst = dst; r.dst_stride = dst_stride; r.dst_off = dst_off; r.dst_pitch = dst_pitch;
    launch_rectify(nullptr, r, n_pairs);
}

}  // extern "C"
