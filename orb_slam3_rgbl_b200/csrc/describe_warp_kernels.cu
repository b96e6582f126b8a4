// Describe kernel (staged formulation, describe_warp.cuh): kernel, launcher, host twin and its test hook.  Host twin checked against
// the oracle on the CPU (tests/test_host_abi.py), device path on the CUDA-on-CPU shim and on the GPU.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "describe_warp.cuh"
#include "rgbl_kernels.h"
#ifdef RGBL_TESTING_EXPORTS
#include "rgbl_testing.h"
#endif

namespace rgbl {

static const int8_t h_pattern31[1024] = {
#include "orb_pattern_31.inc"
};
__device__ __align__(16) const int8_t d_pattern31[1024] = {
#include "orb_pattern_31.inc"
};

struct UmaxTab { int v[16]; };

__global__ void __launch_bounds__(256) describe_staged_kernel(const uint8_t* __restrict__ pyr, const uint8_t* __restrict__ blur,
                                                              size_t frame_stride, const LevelGeom* __restrict__ levels,
                                                              const SelKp* __restrict__ sel, const int* __restrict__ n_sel, int cap,
                                                              UmaxTab umax, rgbl_keypoint* __restrict__ kps, uint8_t* __restrict__ desc) {
    __shared__ uint32_t sm[8][dw::kWarpWords];
    const int frame = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k = blockIdx.x * 8 + warp;
    if (k >= n_sel[frame]) return;                       // warp-uniform
    const SelKp kp = sel[(size_t)frame * cap + k];
    const LevelGeom lg = levels[kp.level];
    const size_t lvl = (size_t)frame * frame_stride + lg.off;
    uint32_t* patch = sm[warp];
    uint32_t* win = patch + dw::kPatchRows * dw::kPatchWords;
    {
        dw::StagedWords<dw::kPatchRows, dw::kPatchWords> rp;
        dw::StagedWords<dw::kWinRows, dw::kWinWords> rw;
        dw::stage_load(lane, pyr + lvl, lg.pitch, kp.x - kHalfPatch, kp.y - kHalfPatch, rp);
        dw::stage_load(lane, blur + lvl, lg.pitch, kp.x - dw::kWinR, kp.y - dw::kWinR, rw);
        dw::stage_store(lane, rp, patch);
        dw::stage_store(lane, rw, win);
    }
    __syncwarp();
    int m10, m01;
    dw::centroid_partial(lane, patch, (kp.x - kHalfPatch) & 3, umax.v, &m10, &m01);
    m10 = __reduce_add_sync(0xffffffffu, m10);
    m01 = __reduce_add_sync(0xffffffffu, m01);
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    const float factor_pi = (float)(3.14159265358979323846 / 180.0);
    float a, b;
    glibc_sincosf(RGBL_FMUL(angle, factor_pi), &b, &a);      // a = cos, b = sin
    desc[((size_t)frame * cap + k) * 32 + lane] = (uint8_t)dw::brief_byte(lane, win, (kp.x - dw::kWinR) & 3, a, b, d_pattern31);
    if (lane == 0) {
        rgbl_keypoint o;
        const float fx = (float)kp.x, fy = (float)kp.y;
        o.x = (kp.level != 0) ? RGBL_FMUL(fx, lg.scale) : fx;
        o.y = (kp.level != 0) ? RGBL_FMUL(fy, lg.scale) : fy;
        o.size = (float)lg.scaled_patch;
        o.angle = angle;
        o.response = (float)kp.score;
        o.octave = kp.level;
        o.class_id = -1;
        kps[(size_t)frame * cap + k] = o;
    }
}

void launch_describe_staged(cudaStream_t st, const uint8_t* pyr, const uint8_t* blur, size_t frame_stride, const LevelGeom* d_levels,
                            const SelKp* sel, const int* n_sel, int cap, int max_n, const int umax[16], rgbl_keypoint* kps, uint8_t* desc,
                            int n_frames) {
    if (max_n <= 0) return;
    UmaxTab t;
    for (int i = 0; i < 16; ++i) t.v[i] = umax[i];
    describe_staged_kernel<<<dim3((max_n + 7) / 8, n_frames), 256, 0, st>>>(pyr, blur, frame_stride, d_levels, sel, n_sel, cap, t, kps, desc);
}

// Host twin: the same per-lane functions, the 32 lanes one after the other.
void describe_staged_host(const uint8_t* img, const uint8_t* blur, int pitch, int x, int y, const int umax[16], float* angle_out,
                          uint8_t desc32[32]) {
    uint32_t patch[dw::kPatchRows * dw::kPatchWords], win[dw::kWinRows * dw::kWinWords];
    for (int lane = 0; lane < 32; ++lane) {
        dw::stage_words(lane, 32, img, pitch, x - kHalfPatch, y - kHalfPatch, dw::kPatchRows, dw::kPatchWords, patch);
        dw::stage_words(lane, 32, blur, pitch, x - dw::kWinR, y - dw::kWinR, dw::kWinRows, dw::kWinWords, win);
    }
    int m10 = 0, m01 = 0;
    for (int lane = 0; lane < 32; ++lane) {
        int p10, p01;
        dw::centroid_partial(lane, patch, (x - kHalfPatch) & 3, umax, &p10, &p01);
        m10 += p10; m01 += p01;
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);
    const float factor_pi = (float)(3.14159265358979323846 / 180.0);
    float a, b;
    glibc_sincosf(RGBL_FMUL(angle, factor_pi), &b, &a);
    for (int lane = 0; lane < 32; ++lane) desc32[lane] = (uint8_t)dw::brief_byte(lane, win, (x - dw::kWinR) & 3, a, b, h_pattern31);
    *angle_out = angle;
}

}  // namespace rgbl

#ifdef RGBL_TESTING_EXPORTS        // test hooks: only in librgbl_b200_testing.so (csrc/rgbl_testing.h)
extern "C" {

// test hook: orientation (degrees) and 32-byte descriptor of n keypoints (x, y in level coordinates, >= 19 px from the border)
// of one pyramid level and its 7x7-blurred copy (both w x h, row stride `stride`), computed by the host twin of the staged
// describe kernel.  orb: only the tables derived from it (umax) are used.
int rgbl_describe_staged_emulation(const rgbl_orb_params* orb, const uint8_t* level_img, const uint8_t* blurred_img, int w, int h,
                                   int stride, int n, const int32_t* xy, float* angle_out, uint8_t* desc_out) {
    using namespace rgbl;
    if (!orb || !level_img || !blurred_img || n < 0 || (n > 0 && (!xy || !angle_out || !desc_out))) return RGBL_E_INVALID;
    OrbTables tab;
    const int rc = compute_orb_tables(*orb, tab);
    if (rc) return rc;
    const int pitch = (w + 63) & ~63;                  // the device layout: rows padded to 64 bytes
    std::vector<uint8_t> a((size_t)pitch * h + 64, 0), b((size_t)pitch * h + 64, 0);
    for (int y = 0; y < h; ++y) { std::memcpy(&a[(size_t)y * pitch], level_img + (size_t)y * stride, w); std::memcpy(&b[(size_t)y * pitch], blurred_img + (size_t)y * stride, w); }
    for (int i = 0; i < n; ++i) {
        const int x = xy[2 * i], y = xy[2 * i + 1];
        if (x < kEdgeThreshold || y < kEdgeThreshold || x >= w - kEdgeThreshold || y >= h - kEdgeThreshold) return RGBL_E_INVALID;
        describe_staged_host(a.data(), b.data(), pitch, x, y, tab.umax, angle_out + i, desc_out + 32 * (size_t)i);
    }
    return RGBL_OK;
}

}  // extern "C"
#endif  // RGBL_TESTING_EXPORTS
