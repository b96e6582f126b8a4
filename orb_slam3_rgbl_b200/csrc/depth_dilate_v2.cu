// DepthModule::Upsample_InverseDilation (src/DepthModule.cc:230-274); validated on the CUDA-on-CPU shim and on the GPU against the oracle.
// Per 32 x 32 tile: recompute the winning point's depth of every pixel of the tile and its halo (same arithmetic as depth_project_kernel),
// build the inverted map t = M - d (zeroed above M-1), take the max over the structuring element, invert back: the exact float pipeline
// of the reference.  Max is exact and order-free, so the following shortcuts do not change a bit:
//   * a tile whose staged window holds no LiDAR return skips the structuring-element loop: every in-image value of the inverted
//     map is 0 there, so the output is 0 whatever the element is (most of the upper half of a KITTI frame);
//   * the (dy, dx) taps are turned once per CTA into shared-memory offsets, so a tap costs two shared loads and one FMNMX
//     instead of two constant-bank loads, the address arithmetic, one shared load and one FMNMX;
//   * the 5x5 diamond (the element of the KITTI RGB-L settings, Examples/RGB-L/KITTI00-02.yaml) has its 13 taps compiled in: 13 loads
//     with immediate offsets and a tree of maxima (2-input FMNMX on sm_90a) instead of a 13-trip loop with an offset load per tap.
#include <cfloat>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

namespace {
constexpr int kStampShift2 = 22;                      // same packing as depth_kernels.cu: stamp << 22 | (point index + 1)
constexpr uint32_t kIdxMask2 = (1u << kStampShift2) - 1u;

__device__ __forceinline__ float project_row2(const float* P, float x, float y, float z, float o) {
    double acc = __dmul_rn((double)P[0], (double)x);
    acc = __dadd_rn(acc, __dmul_rn((double)P[1], (double)y));
    acc = __dadd_rn(acc, __dmul_rn((double)P[2], (double)z));
    acc = __dadd_rn(acc, __dmul_rn((double)P[3], (double)o));
    return (float)acc;
}
struct DilateTaps2 { int n; int8_t dx[81], dy[81]; };
}  // namespace

template <int SHAPE /* 0: any element <= 9x9, 1: 5x5 diamond */>
__global__ void __launch_bounds__(256) depth_resolve_dilate_v2_kernel(const float* __restrict__ pts, int pts_stride, const int* __restrict__ n_pts,
                                                                      DepthDev prm, DilateTaps2 taps, int W, int H,
                                                                      const uint32_t* __restrict__ idx_map, uint32_t stamp,
                                                                      float* __restrict__ raw, float* __restrict__ processed) {
    constexpr int TW = 32, TH = 32, HALO = 4, SW = TW + 2 * HALO, SH = TH + 2 * HALO, SP = SW + 1;
    __shared__ float t[SH * SP];
    __shared__ int s_off[81];
    const int frame = blockIdx.z, tid = threadIdx.x;
    const int lx = tid & 31, ly = tid >> 5;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const int n = n_pts[frame];
    const float* X = pts + (size_t)frame * pts_stride;
    const uint32_t* im = idx_map + (size_t)frame * W * H;
    const float M = prm.inv_scale_m, thr = __fsub_rn(M, 1.0f);

    if (tid < taps.n) s_off[tid] = taps.dy[tid] * SP + taps.dx[tid];
    int any_valid = 0;
    for (int r = ly; r < SH; r += 8) {
        const int gy = y0 + r - HALO;
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
            const int c = lx + 32 * cc;
            if (c >= SW) break;
            const int gx = x0 + c - HALO;
            float tv = -FLT_MAX;                      // out-of-image taps are ignored by cv::dilate
            if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
                const uint32_t e = __ldg(im + (size_t)gy * W + gx);
                float d = 0.f;
                if ((e >> kStampShift2) == stamp) {
                    const int p = (int)(e & kIdxMask2) - 1;
                    d = project_row2(prm.P + 8, __ldg(X + p), __ldg(X + n + p), __ldg(X + 2 * (size_t)n + p), __ldg(X + 3 * (size_t)n + p));
                    any_valid = 1;
                }
                const bool interior = (r >= HALO && r < HALO + TH && c >= HALO && c < HALO + TW);
                if (interior && raw) raw[(size_t)frame * W * H + (size_t)gy * W + gx] = d;
                const float inv = __fsub_rn(M, d);
                tv = (inv > thr) ? 0.f : inv;         // THRESH_TOZERO_INV at M-1
            }
            t[r * SP + c] = tv;
        }
    }
    const int tile_has_points = __syncthreads_or(any_valid);
    const int gx = x0 + lx;
    if (gx >= W) return;
    if (!tile_has_points) {
        // t is 0 at every in-image position: max over any tap set containing an in-image tap is 0 -> M - 0 = M > M - 1 -> 0; a
        // tap set that only reaches outside the image gives M + FLT_MAX > M - 1 -> 0 as well
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int gy = y0 + ly + 8 * k;
            if (gy < H) processed[(size_t)frame * W * H + (size_t)gy * W + gx] = 0.f;
        }
        return;
    }
    const int nt = taps.n;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = ly + 8 * k, gy = y0 + r;
        if (gy >= H) break;
        const float* tp = &t[(r + HALO) * SP + lx + HALO];
        float best;
        if (SHAPE == 1) {
            const float a0 = fmaxf(fmaxf(tp[-2 * SP], tp[-SP - 1]), tp[-SP]), a1 = fmaxf(fmaxf(tp[-SP + 1], tp[-2]), tp[-1]);
            const float a2 = fmaxf(fmaxf(tp[0], tp[1]), tp[2]), a3 = fmaxf(fmaxf(tp[SP - 1], tp[SP]), tp[SP + 1]);
            best = fmaxf(fmaxf(fmaxf(a0, a1), fmaxf(a2, a3)), tp[2 * SP]);
        } else {
            best = -FLT_MAX;
            for (int q = 0; q < nt; ++q) best = fmaxf(best, tp[s_off[q]]);
        }
        const float o = __fsub_rn(M, best);
        processed[(size_t)frame * W * H + (size_t)gy * W + gx] = (o > thr) ? 0.f : o;
    }
}

void launch_depth_resolve_dilate_v2(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts, const DepthDev& prm, int W, int H,
                                    const uint32_t* idx_map, uint32_t stamp, float* raw, float* processed, int n_frames) {
    DilateTaps2 taps;
    taps.n = 0;
    const int ax = prm.ku / 2, ay = prm.kv / 2;
    for (int j = 0; j < prm.kv; ++j)
        for (int i = 0; i < prm.ku; ++i)
            if (prm.mask[j * prm.ku + i]) { taps.dx[taps.n] = (int8_t)(i - ax); taps.dy[taps.n] = (int8_t)(j - ay); ++taps.n; }
    static const int8_t kDiamond5[13][2] = {{0, -2}, {-1, -1}, {0, -1}, {1, -1}, {-2, 0}, {-1, 0}, {0, 0}, {1, 0}, {2, 0}, {-1, 1}, {0, 1}, {1, 1}, {0, 2}};      // (dx, dy) in mask order
    bool diamond5 = prm.ku == 5 && prm.kv == 5 && taps.n == 13;
    for (int q = 0; diamond5 && q < 13; ++q) diamond5 = taps.dx[q] == kDiamond5[q][0] && taps.dy[q] == kDiamond5[q][1];
    const dim3 grid((W + 31) / 32, (H + 31) / 32, n_frames);
    if (diamond5) depth_resolve_dilate_v2_kernel<1><<<grid, 256, 0, st>>>(pts, pts_stride, n_pts, prm, taps, W, H, idx_map, stamp, raw, processed);
    else depth_resolve_dilate_v2_kernel<0><<<grid, 256, 0, st>>>(pts, pts_stride, n_pts, prm, taps, W, H, idx_map, stamp, raw, processed);
}

}  // namespace rgbl
