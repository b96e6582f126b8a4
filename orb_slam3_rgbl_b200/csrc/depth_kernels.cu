// DepthModule kernels for sm_90a (reference: src/DepthModule.cc:50-139,230-274).
//
//   project  : one LiDAR point per thread; Q = P*X with each dot product accumulated in double and
//              rounded once (what cv::gemm does for CV_32F), u = Qx*(1/Qz), v = Qy*(1/Qz) with the
//              reciprocal rounded separately (Mat::mul(1/row)), strict bounds, C truncation.
//              The reference scatters sequentially, so the LAST point in file order owns a pixel:
//              atomicMax on (stamp << 22 | point_index+1).  The per-call stamp makes stale entries of
//              earlier frames lose automatically, so the index map is never cleared on the hot path.
//   resolve+dilate : per tile, recompute the winning point's depth (same arithmetic), build the
//              inverted map t = M - d (zeroed above M-1), take the max over the structuring element,
//              invert back: the exact float pipeline of Upsample_InverseDilation.
//   gather   : GetFeatureDepthFromDepthMap (:82-104), and Frame::ComputeStereoFromRGBD (src/Frame.cc:1074-1095) on a uint16 RGB-D plane.
//   undistort: Frame::UndistortKeyPoints (src/Frame.cc:837-869), mvKeys -> mvKeysUn of a distorted camera, before the gather.
#include <cfloat>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

constexpr int kStampShift = 22;
constexpr uint32_t kIdxMask = (1u << kStampShift) - 1u;

__device__ __forceinline__ float project_row(const float* P, float x, float y, float z, float o) {
    double acc = __dmul_rn((double)P[0], (double)x);
    acc = __dadd_rn(acc, __dmul_rn((double)P[1], (double)y));
    acc = __dadd_rn(acc, __dmul_rn((double)P[2], (double)z));
    acc = __dadd_rn(acc, __dmul_rn((double)P[3], (double)o));
    return (float)acc;
}

__global__ void __launch_bounds__(256) depth_project_kernel(const float* __restrict__ pts, int pts_stride,
                                                            const int* __restrict__ n_pts, DepthDev prm, int W, int H,
                                                            uint32_t* __restrict__ idx_map, uint32_t stamp) {
    const int frame = blockIdx.y;
    const int n = n_pts[frame];
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float* X = pts + (size_t)frame * pts_stride;
    const float x = __ldg(X + i), y = __ldg(X + n + i), z = __ldg(X + 2 * (size_t)n + i), o = __ldg(X + 3 * (size_t)n + i);
    const float q0 = project_row(prm.P, x, y, z, o);
    const float q1 = project_row(prm.P + 4, x, y, z, o);
    const float d = project_row(prm.P + 8, x, y, z, o);
    const float inv = __fdiv_rn(1.0f, d);
    const float u = __fmul_rn(q0, inv), v = __fmul_rn(q1, inv);
    if (u > 0.f && v > 0.f && u < (float)W && v < (float)H && d > prm.min_dist && d < prm.max_dist) {
        uint32_t* m = idx_map + (size_t)frame * W * H + (size_t)(int)v * W + (int)u;
        atomicMax(m, (stamp << kStampShift) | (uint32_t)(i + 1));
    }
}

// The reference's loader (Examples/RGB-L/rgbl_kitti.cc:151-185) re-lays the .bin records out element by element on the host
// (x, y, z rows and a row of ones); here the records are uploaded as they are and transposed on the device.
__global__ void __launch_bounds__(256) deinterleave_xyzr_kernel(const float* __restrict__ raw, float* __restrict__ pts, int pts_stride,
                                                                const int* __restrict__ n_pts) {
    const int frame = blockIdx.y, n = n_pts[frame], i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float4 r = __ldg(reinterpret_cast<const float4*>(raw + (size_t)frame * pts_stride) + i);
    float* X = pts + (size_t)frame * pts_stride;
    X[i] = r.x; X[n + i] = r.y; X[2 * (size_t)n + i] = r.z; X[3 * (size_t)n + i] = 1.0f;
}

struct DilateTaps { int n; int8_t dx[81], dy[81]; };

__global__ void __launch_bounds__(256) depth_resolve_dilate_kernel(const float* __restrict__ pts, int pts_stride,
                                                                   const int* __restrict__ n_pts, DepthDev prm,
                                                                   DilateTaps taps, int W, int H,
                                                                   const uint32_t* __restrict__ idx_map,
                                                                   uint32_t stamp, float* __restrict__ raw,
                                                                   float* __restrict__ processed) {
    constexpr int TW = 32, TH = 32, HALO = 4, SW = TW + 2 * HALO, SH = TH + 2 * HALO;
    __shared__ float t[SH][SW + 1];
    const int frame = blockIdx.z, tid = threadIdx.x;
    const int lx = tid & 31, ly = tid >> 5;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const int n = n_pts[frame];
    const float* X = pts + (size_t)frame * pts_stride;
    const uint32_t* im = idx_map + (size_t)frame * W * H;
    const float M = prm.inv_scale_m, thr = __fsub_rn(M, 1.0f);

    // rows: warp `ly` handles rows ly, ly+8, ...; lanes cover the 40 columns in two passes
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
                if ((e >> kStampShift) == stamp) {
                    const int p = (int)(e & kIdxMask) - 1;
                    d = project_row(prm.P + 8, __ldg(X + p), __ldg(X + n + p), __ldg(X + 2 * (size_t)n + p),
                                    __ldg(X + 3 * (size_t)n + p));
                }
                const bool interior = (r >= HALO && r < HALO + TH && c >= HALO && c < HALO + TW);
                if (interior && raw) raw[(size_t)frame * W * H + (size_t)gy * W + gx] = d;
                const float inv = __fsub_rn(M, d);
                tv = (inv > thr) ? 0.f : inv;         // THRESH_TOZERO_INV at M-1
            }
            t[r][c] = tv;
        }
    }
    __syncthreads();
    const int gx = x0 + lx;
    if (gx >= W) return;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = ly + 8 * k, gy = y0 + r;
        if (gy >= H) break;
        float best = -FLT_MAX;
        for (int q = 0; q < taps.n; ++q) best = fmaxf(best, t[r + HALO + taps.dy[q]][lx + HALO + taps.dx[q]]);
        const float o = __fsub_rn(M, best);
        processed[(size_t)frame * W * H + (size_t)gy * W + gx] = (o > thr) ? 0.f : o;
    }
}

// The plane holds metric depth (float: the processed LiDAR depth map, or a scaled RGB-D map) or the raw 16-bit RGB-D samples, scaled here
// as Tracking::GrabImageRGBD's imDepth.convertTo(CV_32F, mDepthMapFactor) does per pixel (src/Tracking.cc:1538-1539): (float)u * scale,
// rounded once - so the bits equal convert-then-gather.
__device__ __forceinline__ float depth_sample(float d, float) { return d; }
__device__ __forceinline__ float depth_sample(uint16_t u, float scale) { return __fmul_rn((float)u, scale); }

template <class T>
__global__ void __launch_bounds__(256) depth_gather_kernel(const T* __restrict__ plane, size_t frame_elems, size_t pitch_elems, float scale,
                                                           const rgbl_keypoint* __restrict__ kps,
                                                           const rgbl_keypoint* __restrict__ kps_un,
                                                           const int* __restrict__ n_kp, int cap, float bf,
                                                           float* __restrict__ depth, float* __restrict__ uright) {
    const int frame = blockIdx.y;
    const int k = blockIdx.x * 256 + threadIdx.x;
    if (k >= n_kp[frame]) return;
    const size_t o = (size_t)frame * cap + k;
    const float u = kps[o].x, v = kps[o].y;
    const float d = depth_sample(__ldg(plane + (size_t)frame * frame_elems + (size_t)(int)v * pitch_elems + (int)u), scale);
    float dd = -1.f, ur = -1.f;
    if (d > 0.f && bf >= 0.f) {          // bf < 0: LiDAR.Method None -> no depth association
        dd = d;
        ur = __fsub_rn(kps_un[o].x, __fdiv_rn(bf, d));
    }
    depth[o] = dd;
    uright[o] = ur;
}

// Frame::UndistortKeyPoints (src/Frame.cc:837-869): one keypoint per thread, blockIdx.y = frame.  The output keypoint is the input one with
// only pt replaced, as the reference copies mvKeys[i] and sets pt.x / pt.y.
__global__ void __launch_bounds__(256) undistort_keypoints_kernel(UndistortDev cam, const rgbl_keypoint* __restrict__ kps,
                                                                  const int* __restrict__ n_kp, int cap, rgbl_keypoint* __restrict__ kps_un) {
    const int frame = blockIdx.y;
    const int k = blockIdx.x * 256 + threadIdx.x;
    if (k >= n_kp[frame]) return;
    const size_t o = (size_t)frame * cap + k;
    rgbl_keypoint kp = kps[o];
    undistort_point(cam, kp.x, kp.y, &kp.x, &kp.y);
    kps_un[o] = kp;
}

// ---- DepthModule::Upsample_AverageFiltering (src/DepthModule.cc:200-228) ------------------------------------------
// Filtered = filter2D(Raw, ones(k,k)/k^2, BORDER_REFLECT_101) with OpenCV's accumulation acc = fma(tap, src, acc) in
// row-major tap order; Count = box sum of (Raw > 0); Processed = Filtered * (k^2 / Count)  (0 * inf = NaN where empty).
__device__ __forceinline__ int reflect101d(int p, int n) {
    if (p < 0) p = -p;
    if (p >= n) p = 2 * (n - 1) - p;
    return min(max(p, 0), n - 1);
}

__global__ void __launch_bounds__(256) depth_average_filter_kernel(const float* __restrict__ raw, int W, int H, int k,
                                                                   float* __restrict__ processed) {
    constexpr int TW = 32, TH = 32, HALO = 4, SW = TW + 2 * HALO, SH = TH + 2 * HALO;
    __shared__ float t[SH][SW + 1];
    const int frame = blockIdx.z, tid = threadIdx.x, lx = tid & 31, ly = tid >> 5;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const float* src = raw + (size_t)frame * W * H;
    for (int r = ly; r < SH; r += 8) {
        const int gy = reflect101d(y0 + r - HALO, H);
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
            const int c = lx + 32 * cc;
            if (c >= SW) break;
            t[r][c] = __ldg(src + (size_t)gy * W + reflect101d(x0 + c - HALO, W));
        }
    }
    __syncthreads();
    const int gx = x0 + lx;
    if (gx >= W) return;
    const int a = k / 2;
    const float kv = __fdiv_rn(1.0f, (float)(k * k)), k2 = (float)(k * k);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int r = ly + 8 * q, gy = y0 + r;
        if (gy >= H) break;
        float s = 0.f, c = 0.f;
        for (int j = 0; j < k; ++j)
            for (int i = 0; i < k; ++i) {
                const float v = t[r + HALO + j - a][lx + HALO + i - a];
                s = __fmaf_rn(kv, v, s);
                c = __fadd_rn(c, (v > 0.f) ? 1.f : 0.f);
            }
        processed[(size_t)frame * W * H + (size_t)gy * W + gx] = __fmul_rn(s, __fdiv_rn(k2, c));
    }
}

// ---- DepthModule::Upsample_NearestNeighbor_Pixel (src/DepthModule.cc:145-198): one warp per keypoint -----------------
// cv::distanceTransform(DIST_L2, DIST_MASK_5) runs a 5x5 chamfer in 16.16 fixed point (65536 / 91750 / 143976), so its value
// at a pixel is the closed-form chamfer cost to the nearest pixel with a (rounded) non-zero depth; only values below
// SearchRadius matter, so a (2R+3)^2 window is exact.  Then max of Raw over the 2sr x 2sr box at offsets [-sr, sr-1].
__device__ __forceinline__ unsigned chamfer5_fixed(int dx, int dy) {
    dx = abs(dx); dy = abs(dy);
    if (dx < dy) { const int tmp = dx; dx = dy; dy = tmp; }
    if (dx >= 2 * dy) return (unsigned)(dx - 2 * dy) * 65536u + (unsigned)dy * 143976u;
    return (unsigned)(2 * dy - dx) * 91750u + (unsigned)(dx - dy) * 143976u;
}

__global__ void __launch_bounds__(256) depth_nn_pixel_kernel(const float* __restrict__ raw, int W, int H,
                                                             const rgbl_keypoint* __restrict__ kps,
                                                             const rgbl_keypoint* __restrict__ kps_un,
                                                             const int* __restrict__ n_kp, int cap, float bf, float Rf,
                                                             float* __restrict__ depth, float* __restrict__ uright) {
    const int frame = blockIdx.y;
    const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= n_kp[frame]) return;
    const size_t o = (size_t)frame * cap + k;
    const float* src = raw + (size_t)frame * W * H;
    const float kx = kps[o].x, ky = kps[o].y;
    const int u = (int)kx, v = (int)ky, R = (int)Rf, win = R + 1, side = 2 * win + 1;
    unsigned best = 0xffffffffu;
    for (int i = lane; i < side * side; i += 32) {
        const int dy = i / side - win, dx = i - (dy + win) * side - win;
        const int xx = u + dx, yy = v + dy;
        if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
        const float d = __ldg(src + (size_t)yy * W + xx);
        if (__float2int_rn(d) > 0 || d >= 255.5f) best = min(best, chamfer5_fixed(dx, dy));
    }
    best = __reduce_min_sync(0xffffffffu, best);
    float dd = -1.f, ur = -1.f;
    if (best != 0xffffffffu) {
        const float dist = (float)((double)best * (1.0 / 65536.0));
        int sr = (int)dist;
        if (sr >= 0 && (float)sr < Rf) {
            ++sr;
            const int bx = (int)__fsub_rn(__fadd_rn(kx, Rf), (float)sr) - R, by = (int)__fsub_rn(__fadd_rn(ky, Rf), (float)sr) - R;
            unsigned mx = 0;                       // depths are >= 0: float order == unsigned order of the bit patterns
            for (int i = lane; i < 4 * sr * sr; i += 32) {
                const int yy = by + i / (2 * sr), xx = bx + i % (2 * sr);
                if (xx >= 0 && xx < W && yy >= 0 && yy < H) mx = max(mx, __float_as_uint(__ldg(src + (size_t)yy * W + xx)));
            }
            mx = __reduce_max_sync(0xffffffffu, mx);
            const float d = __uint_as_float(mx);
            if (d > 0.f) { dd = d; ur = __fsub_rn(kps_un[o].x, __fdiv_rn(bf, d)); }
        }
    }
    if (lane == 0) { depth[o] = dd; uright[o] = ur; }
}

void launch_depth_average_filter(cudaStream_t st, const float* raw, int W, int H, int k, float* processed, int n_frames) {
    depth_average_filter_kernel<<<dim3((W + 31) / 32, (H + 31) / 32, n_frames), 256, 0, st>>>(raw, W, H, k, processed);
}

void launch_depth_nn_pixel(cudaStream_t st, const float* raw, int W, int H, const rgbl_keypoint* kps, const rgbl_keypoint* kps_un,
                           const int* n_kp, int cap, int max_n, float bf, float R, float* depth, float* uright, int n_frames) {
    if (max_n <= 0) return;
    depth_nn_pixel_kernel<<<dim3((max_n + 7) / 8, n_frames), 256, 0, st>>>(raw, W, H, kps, kps_un, n_kp, cap, bf, R, depth, uright);
}

void launch_depth_project(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts, int max_n_pts,
                          const DepthDev& prm, int W, int H, uint32_t* idx_map, uint32_t stamp, int n_frames) {
    if (max_n_pts <= 0) return;
    depth_project_kernel<<<dim3((max_n_pts + 255) / 256, n_frames), 256, 0, st>>>(pts, pts_stride, n_pts, prm, W, H,
                                                                                 idx_map, stamp);
}

void launch_deinterleave_xyzr(cudaStream_t st, const float* raw, float* pts, int pts_stride, const int* n_pts, int max_n_pts, int n_frames) {
    if (max_n_pts <= 0) return;
    deinterleave_xyzr_kernel<<<dim3((max_n_pts + 255) / 256, n_frames), 256, 0, st>>>(raw, pts, pts_stride, n_pts);
}

void launch_depth_resolve_dilate(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts,
                                 const DepthDev& prm, int W, int H, const uint32_t* idx_map, uint32_t stamp,
                                 float* raw, float* processed, int n_frames) {
    DilateTaps taps;
    taps.n = 0;
    const int ax = prm.ku / 2, ay = prm.kv / 2;
    for (int j = 0; j < prm.kv; ++j)
        for (int i = 0; i < prm.ku; ++i)
            if (prm.mask[j * prm.ku + i]) { taps.dx[taps.n] = (int8_t)(i - ax); taps.dy[taps.n] = (int8_t)(j - ay); ++taps.n; }
    depth_resolve_dilate_kernel<<<dim3((W + 31) / 32, (H + 31) / 32, n_frames), 256, 0, st>>>(
        pts, pts_stride, n_pts, prm, taps, W, H, idx_map, stamp, raw, processed);
}

void launch_depth_gather(cudaStream_t st, const float* processed, int W, int H, const rgbl_keypoint* kps,
                         const rgbl_keypoint* kps_un, const int* n_kp, int cap, int max_n, float bf, float* depth,
                         float* uright, int n_frames) {
    if (max_n <= 0) return;
    depth_gather_kernel<float><<<dim3((max_n + 255) / 256, n_frames), 256, 0, st>>>(processed, (size_t)W * H, (size_t)W, 1.f, kps, kps_un, n_kp, cap, bf,
                                                                                   depth, uright);
}

void launch_undistort_keypoints(cudaStream_t st, const UndistortDev& cam, const rgbl_keypoint* kps, const int* n_kp, int cap, int max_n,
                                rgbl_keypoint* kps_un, int n_frames) {
    if (max_n <= 0) return;
    undistort_keypoints_kernel<<<dim3((max_n + 255) / 256, n_frames), 256, 0, st>>>(cam, kps, n_kp, cap, kps_un);
}

void launch_depth_gather_u16(cudaStream_t st, const uint16_t* plane, size_t frame_elems, size_t pitch_elems, float scale, const rgbl_keypoint* kps,
                             const rgbl_keypoint* kps_un, const int* n_kp, int cap, int max_n, float bf, float* depth, float* uright, int n_frames) {
    if (max_n <= 0) return;
    depth_gather_kernel<uint16_t><<<dim3((max_n + 255) / 256, n_frames), 256, 0, st>>>(plane, frame_elems, pitch_elems, scale, kps, kps_un, n_kp, cap, bf,
                                                                                      depth, uright);
}

}  // namespace rgbl
