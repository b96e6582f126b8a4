// ORACLE (test infrastructure): cv::remap(src, dst, mapx, mapy, INTER_LINEAR, BORDER_CONSTANT, 0) for an 8UC1 source and two CV_32FC1
// maps, the call System::TrackStereo makes on both images of a pair before GrabImageStereo (src/System.cc:251 ff.), and the
// cv::convertMaps(mapx, mapy, CV_16SC2) form of the maps.  Restated from OpenCV's fixed-point bilinear remap (imgproc remapBilinear,
// INTER_BITS = 5): X = cvRound(mapx * 32), Y = cvRound(mapy * 32) (round half to even, saturated to int), (sx, sy) = (sat16(X >> 5),
// sat16(Y >> 5)), (ax, ay) = (X & 31, Y & 31); weights (32 - ay)(32 - ax) 32, (32 - ay) ax 32, ay (32 - ax) 32, ay ax 32 (sum 2^15);
// dst = sat_u8((sum + 2^14) >> 15), taps outside the source contribute 0.  Compiled with -ffp-contract=off; pinned against python-cv2 in
// tests/test_oracle_rectify.py.
#include <climits>
#include <cmath>
#include <cstdint>

namespace {

int round_fixed5(float v) {
    const float r = std::nearbyint(v * 32.f);
    if (r >= 2147483648.f) return INT_MAX;
    if (r < -2147483648.f) return INT_MIN;
    return (int)r;
}

int sat16(int v) { return v < SHRT_MIN ? SHRT_MIN : (v > SHRT_MAX ? SHRT_MAX : v); }

}  // namespace

extern "C" {

// maps (row stride mstride floats) of dw x dh -> xy [dh][dw][2] int16 (sx, sy), a [dh][dw] = ay * 32 + ax
void orc_convert_maps(const float* mapx, const float* mapy, int mstride, int dw, int dh, int16_t* xy, uint16_t* a) {
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
            const int X = round_fixed5(mapx[(size_t)y * mstride + x]), Y = round_fixed5(mapy[(size_t)y * mstride + x]);
            const size_t o = (size_t)y * dw + x;
            xy[2 * o] = (int16_t)sat16(X >> 5);
            xy[2 * o + 1] = (int16_t)sat16(Y >> 5);
            a[o] = (uint16_t)((Y & 31) * 32 + (X & 31));
        }
}

// src sw x sh (row stride sstride bytes) -> dst dw x dh (row stride dstride) through the maps
void orc_remap_u8(const uint8_t* src, int sw, int sh, int sstride, const float* mapx, const float* mapy, int mstride, int dw, int dh, uint8_t* dst,
                  int dstride) {
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) {
            const int X = round_fixed5(mapx[(size_t)y * mstride + x]), Y = round_fixed5(mapy[(size_t)y * mstride + x]);
            const int sx = sat16(X >> 5), sy = sat16(Y >> 5), ax = X & 31, ay = Y & 31;
            const int w[4] = {(32 - ay) * (32 - ax) * 32, (32 - ay) * ax * 32, ay * (32 - ax) * 32, ay * ax * 32};
            int s = 1 << 14;
            for (int t = 0; t < 4; ++t) {
                const int tx = sx + (t & 1), ty = sy + (t >> 1);
                if (tx >= 0 && tx < sw && ty >= 0 && ty < sh) s += (int)src[(size_t)ty * sstride + tx] * w[t];
            }
            s >>= 15;
            dst[(size_t)y * dstride + x] = (uint8_t)(s > 255 ? 255 : s);
        }
}

}  // extern "C"
