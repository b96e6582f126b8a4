// Warp-per-keypoint orientation + steered BRIEF with the two pixel neighbourhoods staged in shared memory
// (IC_Angle src/ORBextractor.cc:76-103, computeOrbDescriptor :107-146).
//
// Why: a warp that maps lane <-> ROW of the radius-15 disc and gathers the 512 BRIEF samples straight from global memory
// touches ~32 different cache lines with almost every one of its ~47 load instructions (≈ 1.5 k L1 wavefronts per keypoint,
// the bound of that formulation).  Here the 31 x 31 patch of the level and the 37 x 37 window of the
// blurred level (|rotated pattern coordinate| <= round(13 * sqrt 2) = 18) are copied with aligned 32-bit loads of
// consecutive words (≈ 22 load instructions, 1-2 lines each); the centroid sums then run lane <-> COLUMN (a row of the
// patch is one shared-memory wavefront) and the BRIEF samples are shared-memory byte reads.  All sums are integer, the
// sample coordinates use the same float operations: the results are bit-identical.
//
// The per-lane pieces are plain functions of (lane, staged data) shared by the kernel and by a host twin that loops over the
// 32 lanes (tests/test_host_abi.py compares the twin with the oracle's angles and descriptors).
#ifndef RGBL_DESCRIBE_WARP_CUH
#define RGBL_DESCRIBE_WARP_CUH

#include <stdint.h>

#include "rgbl_device.cuh"

namespace rgbl {
namespace dw {

constexpr int kPatchWords = 9;      // 31 px + <= 3 alignment bytes
constexpr int kPatchRows = 31;
constexpr int kWinR = 18;           // radius of the blurred window
constexpr int kWinRows = 2 * kWinR + 1;
constexpr int kWinWords = 10;       // 37 px + <= 3 alignment bytes
constexpr int kWarpWords = kPatchRows * kPatchWords + kWinRows * kWinWords;     // 649 words of shared memory per warp

// Copy `rows` rows of `words` aligned 32-bit words starting at byte column x_first (rounded down to a multiple of 4) of row
// y_first into dst (row-major).  Lane `lane` of `n_lanes` takes every n_lanes-th word.  Words that would end beyond the row
// pitch are skipped (their bytes are never used).  Returns nothing; the alignment offset is x_first & 3.
RGBL_HD void stage_words(int lane, int n_lanes, const uint8_t* img, int pitch, int x_first, int y_first, int rows, int words,
                         uint32_t* dst) {
    const int base = x_first & ~3;
    for (int it = lane; it < rows * words; it += n_lanes) {
        const int r = it / words, w = it - r * words;
        const int col = base + 4 * w;
        uint32_t v = 0;
        if (col + 4 <= pitch) {
            const uint8_t* p = img + (size_t)(y_first + r) * pitch + col;
#if defined(__CUDA_ARCH__)
            v = __ldg(reinterpret_cast<const uint32_t*>(p));
#else
            v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
#endif
        }
        dst[it] = v;
    }
}

// The same copy for one warp with compile-time sizes: ALL loads of the lane are issued before the first store (a lane owns
// ceil(ROWS * WORDS / 32) words), so a warp keeps ~20 independent global loads in flight instead of one or two - the kernel is bound
// by the latency of these gathers, not by their bytes (ncu: long-scoreboard stalls, ~1 TB/s with every SM full of warps).
template <int ROWS, int WORDS>
struct StagedWords { uint32_t v[(ROWS * WORDS + 31) / 32]; };
template <int ROWS, int WORDS>
RGBL_HD void stage_load(int lane, const uint8_t* img, int pitch, int x_first, int y_first, StagedWords<ROWS, WORDS>& out) {
    const int base = x_first & ~3;
#pragma unroll
    for (int t = 0; t < (ROWS * WORDS + 31) / 32; ++t) {
        const int it = lane + 32 * t;
        const int r = it / WORDS, w = it - r * WORDS;
        const int col = base + 4 * w;
        uint32_t v = 0;
        if (it < ROWS * WORDS && col + 4 <= pitch) {
            const uint8_t* p = img + (size_t)(y_first + r) * pitch + col;
#if defined(__CUDA_ARCH__)
            v = __ldg(reinterpret_cast<const uint32_t*>(p));
#else
            v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
#endif
        }
        out.v[t] = v;
    }
}
template <int ROWS, int WORDS>
RGBL_HD void stage_store(int lane, const StagedWords<ROWS, WORDS>& in, uint32_t* dst) {
#pragma unroll
    for (int t = 0; t < (ROWS * WORDS + 31) / 32; ++t) {
        const int it = lane + 32 * t;
        if (it < ROWS * WORDS) dst[it] = in.v[t];
    }
}

// lane <-> column u = lane - 15 of the disc: partial m10 = u * sum_v I(u, v), partial m01 = sum_v v * I(u, v) over the rows
// whose half width umax[|v|] covers the column (the reference walks the same pixels row pair by row pair, :86-100)
RGBL_HD void centroid_partial(int lane, const uint32_t* patch, int align, const int* umax, int* m10, int* m01) {
    *m10 = 0; *m01 = 0;
    if (lane >= kPatchRows) return;
    const int u = lane - kHalfPatch, au = u < 0 ? -u : u;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(patch);
    int s = 0, t = 0;
    for (int r = 0; r < kPatchRows; ++r) {
        const int v = r - kHalfPatch;
        if (au <= umax[v < 0 ? -v : v]) {
            const int val = bytes[r * (kPatchWords * 4) + align + lane];
            s += val;
            t += v * val;
        }
    }
    *m10 = u * s;
    *m01 = t;
}

// lane <-> descriptor byte: 8 comparisons of rotated pattern pairs on the blurred window (:112-144)
RGBL_HD int brief_byte(int lane, const uint32_t* win, int align, float a /*cos*/, float b /*sin*/, const int8_t* pattern) {
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(win);
#if defined(__CUDA_ARCH__)
    // the lane's 32 pattern bytes as two 16-byte loads (the kernel is bound by its load / shared-memory instruction queue: 2 instead of 32 LDG.U8)
    const uint4 p0 = __ldg(reinterpret_cast<const uint4*>(pattern + lane * 32)), p1 = __ldg(reinterpret_cast<const uint4*>(pattern + lane * 32) + 1);
    const uint32_t pw[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#else
    const int8_t* pat = pattern + lane * 32;
#endif
    int val = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int t[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
#if defined(__CUDA_ARCH__)
            const uint32_t w = pw[j] >> (16 * e);                       // bytes 4 j + 2 e, + 1 of the lane's pattern row
            const float px = (float)(int)(int8_t)(w & 0xffu), py = (float)(int)(int8_t)((w >> 8) & 0xffu);
#else
            const float px = (float)pat[4 * j + 2 * e], py = (float)pat[4 * j + 2 * e + 1];
#endif
#if defined(__CUDA_ARCH__)
            const int rr = __float2int_rn(RGBL_FADD(RGBL_FMUL(px, b), RGBL_FMUL(py, a)));
            const int cc = __float2int_rn(RGBL_FSUB(RGBL_FMUL(px, a), RGBL_FMUL(py, b)));
#else
            const int rr = (int)lrintf(RGBL_FADD(RGBL_FMUL(px, b), RGBL_FMUL(py, a)));      // cvRound
            const int cc = (int)lrintf(RGBL_FSUB(RGBL_FMUL(px, a), RGBL_FMUL(py, b)));
#endif
            t[e] = bytes[(rr + kWinR) * (kWinWords * 4) + align + cc + kWinR];
        }
        val |= (t[0] < t[1]) << j;
    }
    return val;
}

}  // namespace dw
}  // namespace rgbl
#endif
