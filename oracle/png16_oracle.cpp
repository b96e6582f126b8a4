// TEST INFRASTRUCTURE (CPU oracle; never linked or called by the product).
// The depth input of System::TrackRGBD: Examples/RGB-D/rgbd_kitti.cc's `cv::imread(depth_file, cv::IMREAD_UNCHANGED)` of a 16-bit
// single-channel PNG, which returns a CV_16U image in host byte order.  Restated from the PNG specification (ISO/IEC 15948: chunk
// layout 5.3, IHDR 11.2.2, one zlib stream over all IDAT chunks 10, scanline filters 9.2-9.4 applied byte-wise with bpp = 2 bytes
// for 16-bit gray, samples stored big-endian 7.1) like png_oracle.cpp does for 8-bit images.  Pinned by tests/test_oracle_rgbd.py
// against python-cv2's imdecode(IMREAD_UNCHANGED) live when cv2 is importable, and by tests/golden/png16_golden.npz otherwise.
// Scope: bit depth 16, colour type 0, no interlace; everything else is reported as unsupported (-2).
#include <zlib.h>

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {
inline uint32_t be32_16(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
inline int paeth16(int a, int b, int c) {
    const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}
}  // namespace

extern "C" {

// -> 0, or < 0: -1 not a PNG / truncated, -2 unsupported format, -3 corrupt stream, -4 output too small.
// out (nullable): h x w uint16 (stride w); a call with out == NULL only reports the size.
int orc_png_decode_depth16(const uint8_t* png, size_t n, int* w_out, int* h_out, uint16_t* out, size_t out_cap) {
    static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
    if (n < 8 + 25 || std::memcmp(png, sig, 8)) return -1;
    size_t pos = 8;
    int w = 0, h = 0;
    std::vector<uint8_t> idat;
    bool have_ihdr = false, end = false;
    while (!end) {
        if (pos + 12 > n) return -1;
        const uint32_t len = be32_16(png + pos);
        const uint8_t* type = png + pos + 4;
        if (pos + 12 + (size_t)len > n) return -1;
        const uint8_t* data = png + pos + 8;
        if ((uint32_t)crc32(crc32(0L, Z_NULL, 0), type, len + 4) != be32_16(data + len)) return -3;
        if (!std::memcmp(type, "IHDR", 4)) {
            if (len != 13) return -3;
            w = (int)be32_16(data); h = (int)be32_16(data + 4);
            if (data[8] != 16 || data[9] != 0 || data[10] != 0 || data[11] != 0 || data[12] != 0) return -2;
            if (w <= 0 || h <= 0) return -2;
            have_ihdr = true;
        } else if (!std::memcmp(type, "IDAT", 4)) {
            if (!have_ihdr) return -3;
            idat.insert(idat.end(), data, data + len);
        } else if (!std::memcmp(type, "IEND", 4)) {
            end = true;
        }
        pos += 12 + (size_t)len;
    }
    if (!have_ihdr) return -1;
    *w_out = w; *h_out = h;
    if (!out) return 0;
    if (out_cap < (size_t)w * h) return -4;
    const size_t row = (size_t)w * 2, raw_bytes = (row + 1) * h;
    std::vector<uint8_t> raw(raw_bytes);
    uLongf got = (uLongf)raw_bytes;
    if (uncompress(raw.data(), &got, idat.data(), (uLong)idat.size()) != Z_OK || got != raw_bytes) return -3;
    std::vector<uint8_t> img(row * h);
    for (int y = 0; y < h; ++y) {
        const uint8_t ft = raw[(row + 1) * y];
        const uint8_t* f = &raw[(row + 1) * y + 1];
        uint8_t* cur = &img[row * y];
        const uint8_t* up = y ? &img[row * (y - 1)] : nullptr;
        if (ft > 4) return -3;
        for (size_t i = 0; i < row; ++i) {
            const int a = i >= 2 ? cur[i - 2] : 0, b = up ? up[i] : 0, c = (up && i >= 2) ? up[i - 2] : 0;
            int pred = 0;
            switch (ft) { case 1: pred = a; break; case 2: pred = b; break; case 3: pred = (a + b) >> 1; break; case 4: pred = paeth16(a, b, c); break; default: break; }
            cur[i] = (uint8_t)(f[i] + pred);
        }
    }
    for (size_t p = 0; p < (size_t)w * h; ++p) out[p] = (uint16_t)((img[2 * p] << 8) | img[2 * p + 1]);
    return 0;
}

}  // extern "C"
