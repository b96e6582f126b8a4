// TEST INFRASTRUCTURE: the colour-input kernels on the CUDA-on-CPU shim, through the library's real launchers: the gray conversion of colour
// planes, the input resize and the stereo remap of colour planes (converted to gray in the same kernel) and the PNG reconstruction into
// colour planes.  A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu_colour.py calls it.
#include <string>
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_internal.h"
#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

// n colour planes [n][h][spitch] of ch bytes per pixel -> n gray destination planes of dst_stride bytes, image at dst_off, rows of dpitch
void emu_gray_planes(const uint8_t* src, int w, int h, int spitch, int ch, int w0, uint8_t* dst, size_t dst_stride, int dst_off, int dpitch, int n) {
    LevelGeom s{}, d{};
    s.w = w; s.h = h; s.pitch = spitch;
    d.w = w; d.h = h; d.pitch = dpitch; d.off = dst_off;
    launch_gray_planes(nullptr, src, (size_t)spitch * h, s, dst, dst_stride, d, ch, w0, n);
}

// n colour planes [n][sh][spitch] -> resized to dw x dh and converted to gray, laid out as for emu_gray_planes; the tables are the
// library's (linear_coefs), as rgbl_set_input_resize builds them
void emu_resize_colour(const uint8_t* src, int sw, int sh, int spitch, int ch, int w0, uint8_t* dst, size_t dst_stride, int dst_off, int dw, int dh,
                       int dpitch, int n) {
    std::vector<LinCoef> t((size_t)dw + dh);
    linear_coefs(sw, dw, t.data());
    linear_coefs(sh, dh, t.data() + dw);
    LevelGeom s{}, d{};
    s.w = sw; s.h = sh; s.pitch = spitch;
    d.w = dw; d.h = dh; d.pitch = dpitch; d.off = dst_off;
    launch_resize_planes(nullptr, src, (size_t)spitch * sh, s, dst, dst_stride, d, t.data(), t.data() + dw, n, ch, w0);
}

// maps = [m1l | m2l | m1r | m2r] (W x H floats each, the output size); colour raw planes [2 n_pairs][sh][spitch] of sw x sh pixels -> gray
// planes laid out as for emu_gray_planes
void emu_rectify_colour(const float* maps, int W, int H, const uint8_t* src, int sw, int sh, int spitch, int ch, int w0, uint8_t* dst,
                        size_t dst_stride, int dst_off, int dpitch, int n_pairs) {
    const int pitch = (W + 3) & ~3;
    std::vector<uint32_t> xy((size_t)2 * H * pitch);
    std::vector<uint16_t> a((size_t)2 * H * pitch);
    launch_rectify_maps(nullptr, maps, W, H, xy.data(), a.data(), pitch);
    RectifyDev r{};
    r.xy = xy.data(); r.a = a.data(); r.map_pitch = pitch; r.W = W; r.H = H; r.src_W = sw; r.src_H = sh;
    r.src = src; r.src_stride = (size_t)spitch * sh; r.src_pitch = spitch; r.ch = ch; r.w0 = w0;
    r.dst = dst; r.dst_stride = dst_stride; r.dst_off = dst_off; r.dst_pitch = dpitch;
    launch_rectify(nullptr, r, n_pairs);
}

// n colour PNG streams of w x h pixels -> their pixels' bytes in planes of dst_stride bytes, rows of `pitch` bytes; returns the channel count
// (or the inflate's negative status)
int emu_png_pixels(int n, const uint8_t* const* png, const size_t* png_bytes, int w, int h, uint8_t* dst, size_t dst_stride, int pitch) {
    const size_t raw_stride = ((size_t)(w * 4 + 1) * h + 255) & ~(size_t)255;
    std::vector<uint8_t> raw(raw_stride * n);
    std::vector<uint32_t> band((size_t)n * w);
    int ch = 0, status = 0;
    std::string err;
    const int rc = png_inflate_batch(n, png, png_bytes, w, h, raw.data(), raw_stride, &ch, err);
    if (rc) return rc;
    launch_png_unfilter_pixels(nullptr, raw.data(), raw_stride, w, h, ch, dst, dst_stride, pitch, band.data(), &status, n);
    return status ? -100 : ch;
}

}  // extern "C"
