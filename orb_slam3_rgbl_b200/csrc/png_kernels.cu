// The image input in front of the path: Examples/RGB-L/rgbl_kitti.cc:87 `cv::imread(file, IMREAD_UNCHANGED)` (OpenCV imgcodecs over
// libpng + zlib) and Tracking::GrabImageRGBL's cvtColor to gray (src/Tracking.cc:1567-1580).
//   host  (png_inflate_host): chunk walk (PNG spec 5.3), IHDR checks, CRC-32 of every chunk, the ONE zlib stream spread over the IDAT
//          chunks inflated (zlib) straight into a pinned staging buffer - entropy decoding is a serial bit stream and stays on the host,
//          one worker thread per frame;
//   device (png_unfilter_gray_kernel): scanline reconstruction (None / Sub / Up / Average / Paeth, spec 9.2-9.4) + the gray conversion,
//          written into level 0 of the frame's pyramid slot, so the decoded colour image never exists in memory.
// A reconstructed sample depends on its left neighbour (same row) and on the row above, so the parallel order is a wavefront: one CTA per
// frame, one thread per row of a band of up to 512 rows, thread r one pixel behind thread r-1; neighbours meet in a double-buffered
// shared-memory exchange (one barrier per step), the row above a band comes from a global one-row buffer written by the band before.
// The gray formula is cv::cvtColor's 8-bit one (15-bit fixed point: 9798, 19235, 3735, + 2^14, >> 15; pinned against cv2 on all 2^24
// colours); imread hands colour data over as B, G, R(, A), so with Camera.RGB = 1 (COLOR_RGB2GRAY) channel 0 = the file's BLUE is
// weighted as red - reproduced as is.
// The depth input of Tracking::GrabImageRGBD (src/Tracking.cc:1518) runs through the same kernel: a 16-bit gray PNG has two bytes per pixel,
// filtered byte-wise like any other, and the output stage writes the big-endian sample as uint16 into the frame's depth plane instead.
#include <zlib.h>

#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {
namespace {

constexpr int kPngRows = 512;

// DEPTH16: CH = 2 bytes of one big-endian 16-bit sample -> uint16 at (pyr + frame * frame_stride + off0) with row pitch pitch0 bytes
template <int CH, bool DEPTH16 = false>
__global__ void __launch_bounds__(kPngRows) png_unfilter_gray_kernel(const uint8_t* __restrict__ raw, size_t raw_stride, int w, int h, int camera_rgb,
                                                                     uint8_t* __restrict__ pyr, size_t frame_stride, int off0, int pitch0,
                                                                     uint32_t* __restrict__ band_rows, int* __restrict__ status) {
    __shared__ uint32_t ex[2][kPngRows];
    const int frame = blockIdx.x, tid = threadIdx.x;
    const uint8_t* R = raw + (size_t)frame * raw_stride;
    const size_t rb = (size_t)w * CH + 1;
    uint8_t* dst = pyr + (size_t)frame * frame_stride + off0;
    uint32_t* brow = band_rows + (size_t)frame * w;
    const int k0 = camera_rgb ? 3735 : 9798, k2 = camera_rgb ? 9798 : 3735;       // weights of the file's R and B samples (see header)
    auto load_px = [&](const uint8_t* src, int x) {
        uint32_t f = 0;
#pragma unroll
        for (int k = 0; k < CH; ++k) f |= (uint32_t)src[1 + (size_t)x * CH + k] << (8 * k);
        return f;
    };
    for (int y0 = 0; y0 < h; y0 += kPngRows) {
        const int rows = min(kPngRows, h - y0), y = y0 + tid;
        const bool live = tid < rows;
        const uint8_t* src = R + (size_t)(live ? y : 0) * rb;
        int ft = live ? src[0] : 0;
        if (ft > 4) { atomicExch(status, 1); ft = 0; }
        uint32_t a = 0, c = 0, gacc = 0;
        uint32_t f_next = (live && tid == 0) ? load_px(src, 0) : 0u;
        const int nsteps = w + rows - 1;
        for (int s = 0; s < nsteps; ++s) {
            const int x = s - tid;
            const bool act = live && x >= 0 && x < w;
            if (act) {
                const uint32_t f = f_next;
                const uint32_t b = tid ? ex[(s + 1) & 1][tid - 1] : (y0 ? brow[x] : 0u);
                uint32_t px = 0;
#pragma unroll
                for (int k = 0; k < CH; ++k) {
                    const int fa = (a >> (8 * k)) & 255, fb = (b >> (8 * k)) & 255, fc = (c >> (8 * k)) & 255;
                    const int p = fa + fb - fc, pa = abs(p - fa), pb = abs(p - fb), pc = abs(p - fc);
                    const int paeth = (pa <= pb && pa <= pc) ? fa : (pb <= pc ? fb : fc);
                    const int pred = ft == 1 ? fa : ft == 2 ? fb : ft == 3 ? ((fa + fb) >> 1) : ft == 4 ? paeth : 0;
                    px |= (uint32_t)((((f >> (8 * k)) & 255) + pred) & 255) << (8 * k);
                }
                a = px; c = b;
                ex[s & 1][tid] = px;
                if (tid == rows - 1 && y0 + kPngRows < h) brow[x] = px;             // the row above the next band
                if constexpr (DEPTH16) {
                    gacc |= (((px & 255u) << 8) | ((px >> 8) & 255u)) << (16 * (x & 1));
                    if ((x & 1) == 1 || x == w - 1) {                              // depth rows are 64-byte aligned and padded too
                        *reinterpret_cast<uint32_t*>(dst + (size_t)y * pitch0 + (size_t)(x & ~1) * 2) = gacc;
                        gacc = 0;
                    }
                } else {
                    uint32_t g = px;
                    if (CH >= 3) g = ((px & 255) * k0 + ((px >> 8) & 255) * 19235u + ((px >> 16) & 255) * k2 + (1u << 14)) >> 15;
                    gacc |= (g & 255u) << (8 * (x & 3));
                    if ((x & 3) == 3 || x == w - 1) {                              // rows are 64-byte aligned and padded: whole words
                        *reinterpret_cast<uint32_t*>(dst + (size_t)y * pitch0 + (x & ~3)) = gacc;
                        gacc = 0;
                    }
                }
            }
            if (live && x + 1 >= 0 && x + 1 < w) f_next = load_px(src, x + 1);      // in flight across the barrier
            __syncthreads();
        }
    }
}

inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

}  // namespace

// One PNG stream -> its filtered scanlines ((w * ch + 1) * h bytes) in `out`.  Returns 0 or a negative code with `err` set.
// depth16: the caller expects a depth image (16-bit gray only, ch = 2 bytes per pixel); else an image (8-bit gray / RGB / RGBA).
int png_inflate_host(const uint8_t* png, size_t n, int want_w, int want_h, uint8_t* out, size_t cap, int* ch_out, std::string& err, bool depth16) {
    static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
    if (!png || n < 8 + 25 || std::memcmp(png, sig, 8)) { err = "not a PNG stream"; return -1; }
    size_t pos = 8;
    int ch = 0;
    bool end = false, inflating = false;
    size_t need = 0;
    z_stream z;
    std::memset(&z, 0, sizeof z);
    auto fail = [&](const char* m, int code) { if (inflating) inflateEnd(&z); err = m; return code; };
    while (!end) {
        if (pos + 12 > n) return fail("truncated PNG stream", -1);
        const uint32_t len = be32(png + pos);
        const uint8_t* type = png + pos + 4;
        if (pos + 12 + (size_t)len > n) return fail("truncated PNG chunk", -1);
        const uint8_t* data = png + pos + 8;
        if ((uint32_t)crc32(crc32(0L, Z_NULL, 0), type, len + 4) != be32(data + len)) return fail("PNG chunk CRC mismatch", -3);
        if (!std::memcmp(type, "IHDR", 4)) {
            if (len != 13 || ch) return fail("bad IHDR", -3);
            const int w = (int)be32(data), h = (int)be32(data + 4), ctype = data[9];
            if (depth16) {
                if (data[8] != 16 || ctype != 0 || data[12] != 0 || data[10] != 0 || data[11] != 0)
                    return fail("a depth PNG must be 16-bit single-channel gray, non-interlaced (what imread returns as CV_16U)", -2);
                ch = 2;
            } else {
                if (data[8] != 8 || data[12] != 0 || data[10] != 0 || data[11] != 0) return fail("only 8-bit non-interlaced PNG is supported (what imread returns as CV_8U unchanged)", -2);
                ch = ctype == 0 ? 1 : ctype == 2 ? 3 : ctype == 6 ? 4 : 0;
                if (!ch) return fail("PNG colour type not supported (gray, RGB, RGBA only)", -2);
            }
            if (w != want_w || h != want_h) return fail("PNG size does not match the context", -4);
            need = ((size_t)w * ch + 1) * h;
            if (need > cap) return fail("PNG staging buffer too small", -4);
            if (inflateInit(&z) != Z_OK) return fail("zlib inflateInit failed", -3);
            inflating = true;
            z.next_out = out; z.avail_out = (uInt)need;
        } else if (!std::memcmp(type, "IDAT", 4)) {
            if (!inflating) return fail("IDAT before IHDR", -3);
            z.next_in = const_cast<Bytef*>(data); z.avail_in = len;
            const int r = inflate(&z, Z_NO_FLUSH);
            if (r != Z_OK && r != Z_STREAM_END) return fail("corrupt zlib stream in IDAT", -3);
            if (z.avail_in && r != Z_STREAM_END) return fail("PNG holds more image data than IHDR announces", -3);
        } else if (!std::memcmp(type, "IEND", 4)) {
            end = true;
        }
        pos += 12 + (size_t)len;
    }
    if (!inflating) { err = "PNG without IHDR"; return -1; }
    const bool complete = z.total_out == need;
    inflateEnd(&z);
    if (!complete) { err = "PNG image data shorter than IHDR announces"; return -3; }
    *ch_out = ch;
    return 0;
}

// n PNG streams -> staged filtered scanlines (pinned h_raw, one slot of raw_stride bytes per frame), in parallel over the frames.
int png_inflate_batch(int n_frames, const uint8_t* const* png, const size_t* png_bytes, int w, int h, uint8_t* h_raw, size_t raw_stride, int* ch_out,
                      std::string& err, bool depth16) {
    std::vector<int> rc(n_frames, 0), ch(n_frames, 0);
    std::vector<std::string> errs(n_frames);
    const int hw = (int)std::thread::hardware_concurrency();
    const int n_workers = std::max(1, std::min(n_frames, hw > 0 ? hw : 4));
    auto work = [&](int t) {
        for (int f = t; f < n_frames; f += n_workers)
            rc[f] = png_inflate_host(png[f], png_bytes[f], w, h, h_raw + (size_t)f * raw_stride, raw_stride, &ch[f], errs[f], depth16);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_workers; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& t : th) t.join();
    for (int f = 0; f < n_frames; ++f) {
        if (rc[f]) { err = "frame " + std::to_string(f) + ": " + errs[f]; return rc[f]; }
        if (ch[f] != ch[0]) { err = "the PNG streams of one batch must have the same channel count"; return -2; }
    }
    *ch_out = ch[0];
    return 0;
}

void launch_png_unfilter_gray(cudaStream_t st, const uint8_t* d_raw, size_t raw_stride, int w, int h, int channels, int camera_rgb, uint8_t* pyr,
                              size_t frame_stride, const LevelGeom& l0, uint32_t* band_rows, int* status, int n_frames) {
    if (channels == 1) png_unfilter_gray_kernel<1><<<n_frames, kPngRows, 0, st>>>(d_raw, raw_stride, w, h, camera_rgb, pyr, frame_stride, l0.off, l0.pitch, band_rows, status);
    else if (channels == 3) png_unfilter_gray_kernel<3><<<n_frames, kPngRows, 0, st>>>(d_raw, raw_stride, w, h, camera_rgb, pyr, frame_stride, l0.off, l0.pitch, band_rows, status);
    else png_unfilter_gray_kernel<4><<<n_frames, kPngRows, 0, st>>>(d_raw, raw_stride, w, h, camera_rgb, pyr, frame_stride, l0.off, l0.pitch, band_rows, status);
}

void launch_png_unfilter_depth16(cudaStream_t st, const uint8_t* d_raw, size_t raw_stride, int w, int h, uint16_t* depth, size_t frame_elems,
                                 size_t pitch_elems, uint32_t* band_rows, int* status, int n_frames) {
    png_unfilter_gray_kernel<2, true><<<n_frames, kPngRows, 0, st>>>(d_raw, raw_stride, w, h, 0, reinterpret_cast<uint8_t*>(depth), frame_elems * 2, 0,
                                                                      (int)(pitch_elems * 2), band_rows, status);
}

}  // namespace rgbl
