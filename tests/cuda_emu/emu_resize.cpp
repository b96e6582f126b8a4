// TEST INFRASTRUCTURE: the input-resize kernels (the 8-bit plane resize of orb_kernels.cu, both its staged-tile and its gather form, and the
// 16-bit depth resize of depth_kernels.cu) on the CUDA-on-CPU shim, through the library's real launchers (tests/test_cuda_emu_resize.py
// builds this file against the two kernel files and host_tables.cpp).
#include "cuda_runtime.h"

#include <vector>

#include "orb_kernels.emu.cpp"
#include "depth_kernels.emu.cpp"

using namespace rgbl;

extern "C" {

// n planes [n][sh][spitch] -> n destination planes of dst_stride bytes, image at dst_off with rows of dpitch bytes; the tables are the
// library's (linear_coefs), as rgbl_set_input_resize builds them
void emu_resize_planes(const uint8_t* src, int sw, int sh, int spitch, uint8_t* dst, size_t dst_stride, int dst_off, int dw, int dh, int dpitch, int n) {
    std::vector<LinCoef> t((size_t)dw + dh);
    linear_coefs(sw, dw, t.data());
    linear_coefs(sh, dh, t.data() + dw);
    LevelGeom s{}, d{};
    s.w = sw; s.h = sh; s.pitch = spitch;
    d.w = dw; d.h = dh; d.pitch = dpitch; d.off = dst_off;
    launch_resize_planes(nullptr, src, (size_t)spitch * sh, s, dst, dst_stride, d, t.data(), t.data() + dw, n);
}

// n depth planes [n][sh][spitch] (elements) -> [n][dh][dpitch] at integer factors kx, ky
void emu_resize_depth16(const uint16_t* src, int sh, int spitch, int kx, int ky, uint16_t* dst, int dw, int dh, int dpitch, int n) {
    launch_resize_depth16(nullptr, src, (size_t)spitch * sh, spitch, kx, ky, dst, (size_t)dpitch * dh, dpitch, dw, dh, n);
}

}  // extern "C"
