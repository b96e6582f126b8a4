// Frame::ComputeStereoMatches (src/Frame.cc:901-1071) for n_pairs (left, right) pairs of frame slots of one batched extraction, one
// launch per kernel, keypoint counts read on the device:
//   row index   vRowIndices (:918-940) as CSR per pair: count (one warp per row), exclusive scan (one CTA per pair), fill.  A row lists
//               its right keypoints in ascending index order, so the match kernel sees the candidates in the reference's order;
//   match       one warp per left keypoint over its row's list: octave +-1, disparity range, Hamming best (first strictly smaller in
//               right-keypoint order), then the 11x11 SAD over 11 shifts on the resident pyramid level and the parabola fit;
//   median      the median-based rejection (:1057-1070), one CTA per pair.
#include <algorithm>
#include <climits>
#include <cmath>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

// rows of vRowIndices a right keypoint is listed in (:929-937): floor(y - r) .. ceil(y + r), r = 2 * mvScaleFactors[octave]
__device__ __forceinline__ bool stereo_lists_row(const StereoBatchDev& s, const rgbl_keypoint& kr, int row) {
    const float r = __fmul_rn(2.0f, s.scale[kr.octave]);
    const int maxr = (int)ceilf(__fadd_rn(kr.y, r)), minr = (int)floorf(__fsub_rn(kr.y, r));
    return row >= minr && row <= maxr;
}

// one warp per (pair, row): walks the pair's right keypoints in index order.  kFill == false: row_start[row] = the row's length;
// kFill == true (row_start scanned): the row's list, in ascending right-keypoint order
template <bool kFill>
__global__ void __launch_bounds__(256) stereo_rows_kernel(StereoBatchDev s) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, p = blockIdx.y;
    if (row >= s.n_rows) return;
    const int n_r = s.n_sel[s.r0 + p];
    const rgbl_keypoint* R = s.kps + (size_t)(s.r0 + p) * s.cap;
    int* start = s.row_start + (size_t)p * (s.n_rows + 1);
    int* out = s.row_idx + (size_t)p * s.idx_cap;
    int pos = kFill ? start[row] : 0;
    for (int base = 0; base < n_r; base += 32) {
        const int ir = base + lane;
        const bool in = ir < n_r && stereo_lists_row(s, R[ir], row);
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (kFill && in) out[pos + __popc(m & ((1u << lane) - 1u))] = ir;
        pos += __popc(m);
    }
    if (!kFill && lane == 0) start[row] = pos;
}

// one CTA per pair: row lengths -> exclusive prefix sums in place, row_start[n_rows] = the pair's total
__global__ void __launch_bounds__(1024) stereo_row_scan_kernel(StereoBatchDev s) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    int* start = s.row_start + (size_t)blockIdx.x * (s.n_rows + 1);
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < s.n_rows; base += 1024) {
        const int i = base + tid;
        const int v = i < s.n_rows ? start[i] : 0;
        int x = v;
        for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
        if (lane == 31) s_warp[w] = x;
        __syncthreads();
        if (w == 0) {
            int t = s_warp[lane];
            for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, t, d); if (lane >= d) t += y; }
            s_warp[lane] = t;
        }
        __syncthreads();
        const int excl = s_carry + (w ? s_warp[w - 1] : 0) + x - v;
        if (i < s.n_rows) start[i] = excl;
        __syncthreads();
        if (tid == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) start[s.n_rows] = s_carry;
}

// one warp per (pair, left keypoint)
__global__ void __launch_bounds__(256) stereo_match_kernel(StereoBatchDev s) {
    const int il = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, p = blockIdx.y;
    const int sl = s.l0 + p, sr = s.r0 + p;
    if (il >= s.n_sel[sl]) return;
    const rgbl_keypoint* Rk = s.kps + (size_t)sr * s.cap;
    const uint8_t* Ld = s.desc + (size_t)sl * s.cap * 32;
    const uint8_t* Rd = s.desc + (size_t)sr * s.cap * 32;
    const int* start = s.row_start + (size_t)p * (s.n_rows + 1);
    const int* idx = s.row_idx + (size_t)p * s.idx_cap;
    const rgbl_keypoint kp = s.kps[(size_t)sl * s.cap + il];
    const int lvl = kp.octave;
    const float vL = kp.y, uL = kp.x;
    const int row = (int)vL;
    const float maxD = __fdiv_rn(s.mbf, s.mb), minU = __fsub_rn(uL, maxD), maxU = uL;     // minD = 0
    float out_d = -1.f, out_u = -1.f; int out_sad = -1;
    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(Ld + (size_t)il * 32)), d1 = __ldg(reinterpret_cast<const uint4*>(Ld + (size_t)il * 32) + 1);
    unsigned best = 0xffffffffu;                    // dist << 16 | iR  (first strictly smaller in iR order = min of this key)
    if (!(maxU < 0) && row >= 0 && row < s.n_rows) {
        const int end = start[row + 1];
        for (int k = start[row] + lane; k < end; k += 32) {
            const int ir = idx[k];
            const rgbl_keypoint kr = Rk[ir];
            if (kr.octave < lvl - 1 || kr.octave > lvl + 1) continue;
            if (!(kr.x >= minU && kr.x <= maxU)) continue;
            const uint8_t* b = Rd + (size_t)ir * 32;
            const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(b)), b1 = __ldg(reinterpret_cast<const uint4*>(b) + 1);
            const int d = __popc(d0.x ^ b0.x) + __popc(d0.y ^ b0.y) + __popc(d0.z ^ b0.z) + __popc(d0.w ^ b0.w) +
                          __popc(d1.x ^ b1.x) + __popc(d1.y ^ b1.y) + __popc(d1.z ^ b1.z) + __popc(d1.w ^ b1.w);
            if (d < 100) best = min(best, ((unsigned)d << 16) | (unsigned)ir);      // bestDist starts at TH_HIGH, strict <
        }
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (best != 0xffffffffu && (int)(best >> 16) < 75) {                            // thOrbDist = (TH_HIGH + TH_LOW) / 2
        const int ir = (int)(best & 0xffffu);
        const float uR0 = Rk[ir].x;
        const float sf = s.inv_scale[lvl];
        const float su = roundf(__fmul_rn(kp.x, sf)), sv = roundf(__fmul_rn(kp.y, sf)), sur0 = roundf(__fmul_rn(uR0, sf));
        const LevelGeom lg = s.levels[lvl];
        const float iniu = sur0, endu = __fadd_rn(sur0, 11.0f);                       // scaleduR0 + L - w, scaleduR0 + L + w + 1
        if (!(iniu < 0 || endu >= (float)lg.w)) {
            const uint8_t* IL = s.pyr + (size_t)sl * s.frame_stride + lg.off;
            const uint8_t* IR = s.pyr + (size_t)sr * s.frame_stride + lg.off;
            const int cu = (int)su, cv = (int)sv, cr = (int)sur0;
            int sad = INT_MAX;
            if (lane < 11) {
                const int inc = lane - 5;
                sad = 0;
                for (int dy = -5; dy <= 5; ++dy) {
                    const uint8_t* a = IL + (size_t)(cv + dy) * lg.pitch + cu - 5;
                    const uint8_t* b = IR + (size_t)(cv + dy) * lg.pitch + cr + inc - 5;
#pragma unroll
                    for (int dx = 0; dx < 11; ++dx) sad += abs((int)__ldg(a + dx) - (int)__ldg(b + dx));
                }
            }
            // best shift: first strictly smaller in inc order = min of (sad << 8 | lane)
            unsigned long long key = (lane < 11) ? (((unsigned long long)(unsigned)sad << 8) | (unsigned)lane) : ~0ull;
            unsigned lo = (unsigned)(key & 0xffffffffu), hi = (unsigned)(key >> 32);
            // 40-bit key min via two-step reduce (hi then lo among the hi-minimal lanes)
            const unsigned hmin = __reduce_min_sync(0xffffffffu, hi);
            const unsigned lmin = __reduce_min_sync(0xffffffffu, (hi == hmin) ? lo : 0xffffffffu);
            const int best_lane = (int)(lmin & 0xffu);
            const int best_inc = best_lane - 5;
            const int best_sad = (int)((((unsigned long long)hmin << 32) | lmin) >> 8);
            if (best_inc != -5 && best_inc != 5) {
                const float dist1 = (float)__shfl_sync(0xffffffffu, sad, best_lane - 1);
                const float dist2 = (float)__shfl_sync(0xffffffffu, sad, best_lane);
                const float dist3 = (float)__shfl_sync(0xffffffffu, sad, best_lane + 1);
                const float den = __fmul_rn(2.0f, __fsub_rn(__fadd_rn(dist1, dist3), __fmul_rn(2.0f, dist2)));
                const float deltaR = __fdiv_rn(__fsub_rn(dist1, dist3), den);
                if (!(deltaR < -1.f || deltaR > 1.f)) {
                    float best_ur = __fmul_rn(s.scale[lvl], __fadd_rn(__fadd_rn(sur0, (float)best_inc), deltaR));
                    float disparity = __fsub_rn(uL, best_ur);
                    if (disparity >= 0.f && disparity < maxD) {
                        if (disparity <= 0.f) { disparity = (float)0.01; best_ur = (float)((double)uL - 0.01); }
                        out_d = __fdiv_rn(s.mbf, disparity); out_u = best_ur; out_sad = best_sad;
                    }
                }
            } else {
                // keep the shuffles convergent for the whole warp
                (void)__shfl_sync(0xffffffffu, sad, 0); (void)__shfl_sync(0xffffffffu, sad, 0); (void)__shfl_sync(0xffffffffu, sad, 0);
            }
        }
    }
    if (lane == 0) {
        const size_t o = (size_t)sl * s.cap + il;
        s.depth[o] = out_d; s.uright[o] = out_u; s.sad[(size_t)p * s.cap + il] = out_sad;
    }
}

// median-based rejection (src/Frame.cc:1057-1070), one CTA per pair.  The threshold needs the SAD at index size/2 of the sorted list
// of matched SADs.  SADs are integers in [0, 11 * 11 * 255] < 2^15, so an exact selection takes two histogram passes: the bin of the
// high 8 bits (sad >> 7) that holds the rank, then the low 7 bits among the SADs of that bin.
__global__ void __launch_bounds__(1024) stereo_median_kernel(StereoBatchDev s) {
    __shared__ int hist[256];
    __shared__ int s_hi, s_rank, s_median;
    const int p = blockIdx.x, sl = s.l0 + p, tid = threadIdx.x;
    const int n = s.n_sel[sl];
    const int* sad = s.sad + (size_t)p * s.cap;
    float* depth = s.depth + (size_t)sl * s.cap;
    float* uright = s.uright + (size_t)sl * s.cap;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += 1024) { const int v = sad[i]; if (v >= 0) atomicAdd(&hist[v >> 7], 1); }
    __syncthreads();
    if (tid == 0) {
        int m = 0;
        for (int b = 0; b < 256; ++b) m += hist[b];
        s_hi = -1;
        if (m) {
            const int target = m / 2;
            int cum = 0, b = 0;
            while (cum + hist[b] <= target) cum += hist[b++];
            s_hi = b; s_rank = target - cum;
        }
    }
    __syncthreads();
    const int hb = s_hi;
    if (hb < 0) return;                              // no match in this pair
    if (tid < 128) hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += 1024) { const int v = sad[i]; if (v >= 0 && (v >> 7) == hb) atomicAdd(&hist[v & 127], 1); }
    __syncthreads();
    if (tid == 0) {
        int cum = 0, b = 0;
        while (cum + hist[b] <= s_rank) cum += hist[b++];
        s_median = (hb << 7) | b;
    }
    __syncthreads();
    const float th = __fmul_rn(__fmul_rn(1.5f, 1.4f), (float)s_median);
    for (int i = tid; i < n; i += 1024)
        if (sad[i] >= 0 && !((float)sad[i] < th)) { depth[i] = -1.f; uright[i] = -1.f; }
}

int stereo_row_index_cap(int cap, const float* scale, int n_levels, int n_rows) {
    float smax = 0.f;
    for (int l = 0; l < n_levels; ++l) smax = std::max(smax, scale[l]);
    return cap * std::min(n_rows, (int)std::ceil(4.f * smax) + 4);
}

void launch_stereo_matches(cudaStream_t st, const StereoBatchDev& s, int n_pairs) {
    const dim3 rows((s.n_rows + 7) / 8, n_pairs), keys((s.cap + 7) / 8, n_pairs);
    stereo_rows_kernel<false><<<rows, 256, 0, st>>>(s);
    stereo_row_scan_kernel<<<n_pairs, 1024, 0, st>>>(s);
    stereo_rows_kernel<true><<<rows, 256, 0, st>>>(s);
    stereo_match_kernel<<<keys, 256, 0, st>>>(s);
    stereo_median_kernel<<<n_pairs, 1024, 0, st>>>(s);
}

// ---- Rectification of stereo pairs: the cv::remap(im, imRect, M1, M2, INTER_LINEAR) that System::TrackStereo runs on both images before
// GrabImageStereo when Settings::needToRectify() (src/System.cc:251 ff.), for 8UC1 images, two CV_32FC1 maps, BORDER_CONSTANT 0.
//
// OpenCV's bilinear remap works in fixed point (imgproc remapBilinear with INTER_BITS = 5): X = cvRound(mapx * 32), Y = cvRound(mapy * 32)
// (round half to even, saturated to int), source pixel (sx, sy) = (sat16(X >> 5), sat16(Y >> 5)), fraction (ax, ay) = (X & 31, Y & 31),
// tap weights (32 - ay)(32 - ax) 32, (32 - ay) ax 32, ay (32 - ax) 32, ay ax 32 (their sum is 2^15, so OpenCV's table correction never
// changes them) and dst = sat_u8((sum of tap * weight + 2^14) >> 15), a tap outside the source contributing 0.  cv::remap with the float
// maps gives what it gives with convertMaps(..., CV_16SC2) maps, so the maps are converted to that form once, when they are set
// (launch_rectify_maps); the remap of a batch reads the converted form (launch_rectify).

namespace {

__device__ __forceinline__ int round_fixed5(float v) {        // cvRound(v * 32), saturated
    const float r = rintf(v * 32.f);
    if (r >= 2147483648.f) return INT_MAX;
    if (r < -2147483648.f) return INT_MIN;
    return (int)r;
}

__device__ __forceinline__ int sat16(int v) { return v < SHRT_MIN ? SHRT_MIN : (v > SHRT_MAX ? SHRT_MAX : v); }

// one thread per map entry: maps = [m1l | m2l | m1r | m2r], each H x W floats; camera = blockIdx.z (0 left, 1 right)
__global__ void __launch_bounds__(256) rectify_maps_kernel(const float* maps, int W, int H, uint32_t* xy, uint16_t* a, int pitch) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, cam = blockIdx.z;
    if (x >= pitch) return;
    const size_t o = ((size_t)cam * H + y) * pitch + x;
    if (x >= W) { xy[o] = 0u; a[o] = 0; return; }           // row padding: read by the last group of a row, never used
    const size_t i = ((size_t)2 * cam * H + y) * W + x;
    const int X = round_fixed5(maps[i]), Y = round_fixed5(maps[i + (size_t)H * W]);
    xy[o] = (uint32_t)(uint16_t)sat16(X >> 5) | ((uint32_t)(uint16_t)sat16(Y >> 5) << 16);
    a[o] = (uint16_t)((Y & 31) * 32 + (X & 31));
}

constexpr int kGroup = 4;                  // output pixels per thread: one 32-bit store per row group

// One thread per group of 4 output pixels of row blockIdx.y of camera blockIdx.z: the group's map entries are read once, then the
// camera's n frames are remapped with them.  Taps outside the source get weight 0 and offset 0, so the frame loop has no branch.
__global__ void __launch_bounds__(128) rectify_kernel(RectifyDev r, int n) {
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * kGroup, y = blockIdx.y, cam = blockIdx.z;
    if (x0 >= r.W) return;
    const size_t o = ((size_t)cam * r.H + y) * r.map_pitch + x0;
    const uint4 m = *reinterpret_cast<const uint4*>(r.xy + o);
    const unsigned long long fr = *reinterpret_cast<const unsigned long long*>(r.a + o);
    const uint32_t mxy[kGroup] = {m.x, m.y, m.z, m.w};
    int off[kGroup][4], w[kGroup][4];
#pragma unroll
    for (int p = 0; p < kGroup; ++p) {
        const int sx = (int)(int16_t)(mxy[p] & 0xffffu), sy = (int)(int16_t)(mxy[p] >> 16);
        const int f = (int)((fr >> (16 * p)) & 0xffffu), ax = f & 31, ay = f >> 5;
        const int wt[4] = {(32 - ay) * (32 - ax) * 32, (32 - ay) * ax * 32, ay * (32 - ax) * 32, ay * ax * 32};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int tx = sx + (t & 1), ty = sy + (t >> 1);
            const bool in = tx >= 0 && tx < r.W && ty >= 0 && ty < r.H;
            off[p][t] = in ? ty * r.src_pitch + tx : 0;
            w[p][t] = in ? wt[t] : 0;
        }
    }
    const int n_out = min(kGroup, r.W - x0);
    for (int f = 0; f < n; ++f) {
        const int slot = cam * n + f;
        const uint8_t* src = r.src + (size_t)slot * r.src_stride;
        uint32_t packed = 0;
#pragma unroll
        for (int p = 0; p < kGroup; ++p) {
            int s = 1 << 14;
#pragma unroll
            for (int t = 0; t < 4; ++t) s += (int)__ldg(src + off[p][t]) * w[p][t];
            packed |= (uint32_t)min(s >> 15, 255) << (8 * p);
        }
        uint8_t* dst = r.dst + (size_t)slot * r.dst_stride + r.dst_off + (size_t)y * r.dst_pitch + x0;
        if (n_out == kGroup) *reinterpret_cast<uint32_t*>(dst) = packed;
        else for (int p = 0; p < n_out; ++p) dst[p] = (uint8_t)(packed >> (8 * p));     // the row's padding is not written
    }
}

}  // namespace

void launch_rectify_maps(cudaStream_t st, const float* maps, int W, int H, uint32_t* xy, uint16_t* a, int pitch) {
    rectify_maps_kernel<<<dim3((pitch + 255) / 256, H, 2), 256, 0, st>>>(maps, W, H, xy, a, pitch);
}

void launch_rectify(cudaStream_t st, const RectifyDev& r, int n_pairs) {
    if (n_pairs < 1) return;
    const int groups = (r.W + kGroup - 1) / kGroup;
    rectify_kernel<<<dim3((groups + 127) / 128, r.H, 2), 128, 0, st>>>(r, n_pairs);
}

}  // namespace rgbl
