// LocalMapping-thread kernels (SURVEY 8(f) row 3): MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:329-403) for a batch
// of map points and ORBmatcher::SearchForTriangulation (src/ORBmatcher.cc:907-1146) between two key frames.  Both are
// embarrassingly parallel in this version of the reference (vbMatched2 is never set, so the key-frame-1 features are
// independent): one warp per map point / per feature, __popc Hamming, warp reductions.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "rgbl_ctx.h"
#include "rgbl_device.cuh"

namespace rgbl {
namespace {

__device__ __forceinline__ int hamming32(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b) {
    const uint4 a0 = __ldg(reinterpret_cast<const uint4*>(a)), a1 = __ldg(reinterpret_cast<const uint4*>(a) + 1);
    const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(b)), b1 = __ldg(reinterpret_cast<const uint4*>(b) + 1);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// One warp per map point.  For every observation i the sorted row of distances is only needed at rank k = (N - 1) / 2:
// the lanes histogram the row (257 bins, distances are 0..256) and a warp scan finds the bin that holds rank k - the value
// std::sort + vDists[0.5 * (N - 1)] returns.  The first row with the smallest median wins (strict '<' in the reference).
__global__ void __launch_bounds__(128) distinctive_kernel(int n_points, const int* __restrict__ obs_start, const uint8_t* __restrict__ desc,
                                                          int* __restrict__ best) {
    __shared__ int hist_all[4][288];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, p = blockIdx.x * 4 + warp;
    if (p >= n_points) return;
    int* hist = hist_all[warp];
    const int b = obs_start[p], N = obs_start[p + 1] - b;
    if (N <= 0) { if (lane == 0) best[p] = -1; return; }
    const int k = (N - 1) >> 1;
    int best_median = 0x7fffffff, best_idx = 0;
    for (int i = 0; i < N; ++i) {
        for (int t = lane; t < 288; t += 32) hist[t] = 0;
        __syncwarp();
        for (int j = lane; j < N; j += 32) atomicAdd(&hist[(i == j) ? 0 : hamming32(desc + 32 * (size_t)(b + i), desc + 32 * (size_t)(b + j))], 1);
        __syncwarp();
        int c[9], s = 0;
#pragma unroll
        for (int t = 0; t < 9; ++t) { c[t] = hist[9 * lane + t]; s += c[t]; }
        int incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        const unsigned m = __ballot_sync(0xffffffffu, incl > k);
        const int src = __ffs(m) - 1;                       // first lane whose bins reach past rank k
        int median = 0;
        if (lane == src) {
            int acc = incl - s;
#pragma unroll
            for (int t = 0; t < 9; ++t) { acc += c[t]; if (acc > k) { median = 9 * lane + t; break; } }
        }
        median = __shfl_sync(0xffffffffu, median, src);
        if (median < best_median) { best_median = median; best_idx = i; }
        __syncwarp();
    }
    if (lane == 0) best[p] = best_idx;
}

struct TriFrame { const uint8_t* desc; const rgbl_keypoint* keys; const uint8_t* has_mp; const float* uright; };
struct TriPair { float F12[9]; float ep[2]; };                 // the constants of one key-frame pair
struct TriParams { TriPair pair; float scale2[RGBL_MAX_LEVELS]; float sigma2[RGBL_MAX_LEVELS]; int only_stereo, coarse; };

// One key-frame-1 feature that shares a vocabulary node with key frame 2, one warp.  The reference's scan keeps a candidate when
// dist <= TH_LOW and dist <= bestDist and the geometric tests pass, so it ends with the LAST candidate of minimum distance among
// those passing the tests: min over (dist << 20 | 0xfffff - position).  Lane 0 writes the match (-1: none) and its rotation bin.
__device__ __forceinline__ void triangulation_search_one(int idx1, int cb, int ce, int lane, const int* __restrict__ node_feat2, const TriFrame& A,
                                                         const TriFrame& B, const TriPair& pr, const TriParams& prm, int* m_out, uint8_t* bin_out) {
    const rgbl_keypoint kp1 = A.keys[idx1];
    const bool stereo1 = A.uright[idx1] >= 0.f;
    // epipolar line of kp1 in image 2 (Pinhole::epipolarConstrain, src/CameraModels/Pinhole.cpp:114-117)
    const float la = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, pr.F12[0]), __fmul_rn(kp1.y, pr.F12[3])), pr.F12[6]);
    const float lb = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, pr.F12[1]), __fmul_rn(kp1.y, pr.F12[4])), pr.F12[7]);
    const float lc = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, pr.F12[2]), __fmul_rn(kp1.y, pr.F12[5])), pr.F12[8]);
    const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
    unsigned best = 0xffffffffu;
    for (int c0 = cb; c0 < ce; c0 += 32) {
        const int c = c0 + lane;
        if (c >= ce) continue;
        const int idx2 = node_feat2[c];
        if (B.has_mp[idx2]) continue;
        const bool stereo2 = B.uright[idx2] >= 0.f;
        if (prm.only_stereo && !stereo2) continue;
        const int dist = hamming32(A.desc + 32 * (size_t)idx1, B.desc + 32 * (size_t)idx2);
        if (dist > 50) continue;                               // TH_LOW
        const rgbl_keypoint kp2 = B.keys[idx2];
        if (!stereo1 && !stereo2) {
            const float ex = __fsub_rn(pr.ep[0], kp2.x), ey = __fsub_rn(pr.ep[1], kp2.y);
            if (__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)) < __fmul_rn(100.f, prm.scale2[kp2.octave])) continue;
        }
        bool ok = prm.coarse != 0;
        if (!ok && den != 0.f) {
            const float num = __fadd_rn(__fadd_rn(__fmul_rn(la, kp2.x), __fmul_rn(lb, kp2.y)), lc);
            const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
            ok = (double)dsqr < 3.84 * (double)prm.sigma2[kp2.octave];
        }
        if (ok) best = min(best, ((unsigned)dist << 20) | (0xfffffu - (unsigned)(c - cb)));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) {
        int m = -1; uint8_t bin = 255;
        if (best != 0xffffffffu) {
            m = node_feat2[cb + (int)(0xfffffu - (best & 0xfffffu))];
            float rot = __fsub_rn(kp1.angle, B.keys[m].angle);
            if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
            int bb = (int)roundf(__fmul_rn(rot, 1.0f / 30));
            if (bb == 30) bb = 0;
            bin = (uint8_t)bb;
        }
        *m_out = m; *bin_out = bin;
    }
}

__global__ void __launch_bounds__(256) triangulation_search_kernel(int n_q, const int* __restrict__ q_feat, const int* __restrict__ q_cbeg,
                                                                   const int* __restrict__ q_cend, const int* __restrict__ node_feat2, TriFrame A,
                                                                   TriFrame B, TriParams prm, int* __restrict__ match12, uint8_t* __restrict__ bins) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= n_q) return;
    const int idx1 = q_feat[q];
    triangulation_search_one(idx1, q_cbeg[q], q_cend[q], lane, node_feat2, A, B, prm.pair, prm, match12 + idx1, bins + idx1);
}

// ComputeThreeMaxima (src/ORBmatcher.cc:2012-2053) over hist[0..29], warp 0 of the CTA: keep[0..2] = the kept bins (-1: none)
__device__ __forceinline__ void three_maxima_keep(const int* hist, int* keep) {
    const int tid = threadIdx.x;
    const int cnt = tid < 30 ? hist[tid] : 0;
    int key = cnt > 0 ? ((cnt << 8) | (255 - tid)) : 0, top_i[3], top_c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        int m = key;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        top_c[r] = m >> 8; top_i[r] = m > 0 ? 255 - (m & 0xff) : -1;
        if (key == m) key = 0;
    }
    int i2 = top_i[1], i3 = top_i[2];
    if ((float)top_c[1] < __fmul_rn(0.1f, (float)top_c[0])) { i2 = -1; i3 = -1; }
    else if ((float)top_c[2] < __fmul_rn(0.1f, (float)top_c[0])) i3 = -1;
    if (tid == 0) { keep[0] = top_i[0]; keep[1] = i2; keep[2] = i3; }
}

// rotation-consistency filter (ComputeThreeMaxima, src/ORBmatcher.cc:2012-2053) + count; one CTA
__global__ void __launch_bounds__(1024) triangulation_finish_kernel(int n1, int check_orientation, int* __restrict__ match12, const uint8_t* __restrict__ bins,
                                                                    int* __restrict__ n_matches) {
    __shared__ int hist[32], keep[3], s_nm;
    const int tid = threadIdx.x;
    if (tid < 32) hist[tid] = 0;
    if (tid == 0) s_nm = 0;
    __syncthreads();
    if (check_orientation) {
        for (int i = tid; i < n1; i += 1024) if (match12[i] >= 0) atomicAdd(&hist[bins[i]], 1);
        __syncthreads();
        if (tid < 32) three_maxima_keep(hist, keep);
        __syncthreads();
    }
    int local = 0;
    for (int i = tid; i < n1; i += 1024) {
        if (match12[i] < 0) continue;
        if (check_orientation) { const int b = bins[i]; if (b != keep[0] && b != keep[1] && b != keep[2]) { match12[i] = -1; continue; } }
        ++local;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    if ((tid & 31) == 0 && local) atomicAdd(&s_nm, local);
    __syncthreads();
    if (tid == 0) *n_matches = s_nm;
}

// ---- LocalMapping::CreateNewMapPoints (src/LocalMapping.cc, Nleft == -1, no IMU) over all neighbours of a key frame -----------
// Search (cnmp_search_kernel: the body above, one query per (neighbour, key-frame-1 feature)), triangulation and checks of every
// candidate match (cnmp_triangulate_kernel: depends on the two key frames only), then one CTA that walks the neighbours in order
// (cnmp_order_kernel): a key-frame-1 feature claimed by an earlier neighbour is dropped, which is exactly the reference's
// `if (pMP1) continue;` since every other query of the search is independent of it.

__global__ void __launch_bounds__(256) cnmp_search_kernel(int n_q, const int* __restrict__ q_feat, const int* __restrict__ q_cbeg, const int* __restrict__ q_cend,
                                                          const int* __restrict__ q_pair, const int* __restrict__ node_feat2, TriFrame A, TriFrame B,
                                                          const TriPair* __restrict__ pairs, TriParams prm, int n1, int* __restrict__ match,
                                                          uint8_t* __restrict__ bins) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= n_q) return;
    const int idx1 = q_feat[q], j = q_pair[q];
    const TriPair pr = pairs[j];
    const size_t slot = (size_t)j * n1 + idx1;
    triangulation_search_one(idx1, q_cbeg[q], q_cend[q], lane, node_feat2, A, B, pr, prm, match + slot, bins + slot);
}

struct CnmpFrame { const rgbl_keypoint* keys; const rgbl_keypoint* keys_un; const float* uright; const float* depth; };
struct CnmpCam {
    float fx, fy, cx, cy, bf, mb, invfx, invfy, th_far, ratio_factor;
    float scale[RGBL_MAX_LEVELS]; float sigma2[RGBL_MAX_LEVELS];
};

__device__ __forceinline__ float dot3(const float* a, const float* b) { return eig_sum3(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1]), __fmul_rn(a[2], b[2])); }

// Eigen 3.4 JacobiSVD<Matrix4f>(A, ComputeFullV) (SVD/JacobiSVD.h: square, so no QR preconditioner; Jacobi/RealSvd2x2.h, Jacobi/Jacobi.h),
// float32 in the library's order of operations; returns the right singular vector of the smallest singular value (column 3 of V after the
// descending sort).  false for a non-finite A, or when 64 sweeps did not converge (Eigen has no limit; a finite A converges in a few).
__device__ __forceinline__ bool jacobi_svd4_null(const float A[4][4], float v3[4]) {
    float scale = 0.f;
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float a = fabsf(A[i][k]); finite = finite && isfinite(a); scale = a > scale ? a : scale; }
    if (!finite) return false;
    if (scale == 0.f) scale = 1.f;
    float W[4][4], V[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) { W[i][k] = __fdiv_rn(A[i][k], scale); V[i][k] = i == k ? 1.f : 0.f; }
    const float precision = __fmul_rn(2.f, 1.1920928955078125e-07f), tiny = 1.17549435e-38f;   // 2 epsilon, FLT_MIN
    float max_diag = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) max_diag = fmaxf(max_diag, fabsf(W[i][i]));
    bool finished = false;
    for (int sweep = 0; sweep < 64 && !finished; ++sweep) {
        finished = true;
#pragma unroll
        for (int p = 1; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < p; ++q) {
                const float pm = __fmul_rn(precision, max_diag), threshold = tiny < pm ? pm : tiny;
                if (!(fabsf(W[p][q]) > threshold || fabsf(W[q][p]) > threshold)) continue;
                finished = false;
                // real_2x2_jacobi_svd
                const float m00 = W[p][p], m01 = W[p][q], m10 = W[q][p], m11 = W[q][q];
                const float t = __fadd_rn(m00, m11), d = __fsub_rn(m10, m01);
                float c1 = 1.f, s1 = 0.f;
                if (!(fabsf(d) < tiny)) {
                    const float u = __fdiv_rn(t, d), tmp = __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(u, u)));
                    s1 = __fdiv_rn(1.f, tmp); c1 = __fdiv_rn(u, tmp);
                }
                float n00 = m00, n01 = m01, n11 = m11;
                if (!(c1 == 1.f && s1 == 0.f)) {            // m.applyOnTheLeft(0, 1, rot1)
                    n00 = __fadd_rn(__fmul_rn(c1, m00), __fmul_rn(s1, m10)); n01 = __fadd_rn(__fmul_rn(c1, m01), __fmul_rn(s1, m11));
                    n11 = __fadd_rn(__fmul_rn(-s1, m01), __fmul_rn(c1, m11));
                }
                float cr = 1.f, sr = 0.f;                   // j_right.makeJacobi(m, 0, 1)
                const float deno = __fmul_rn(2.f, fabsf(n01));
                if (!(deno < tiny)) {
                    const float tau = __fdiv_rn(__fsub_rn(n00, n11), deno), w = __fsqrt_rn(__fadd_rn(__fmul_rn(tau, tau), 1.f));
                    const float tt = tau > 0.f ? __fdiv_rn(1.f, __fadd_rn(tau, w)) : __fdiv_rn(1.f, __fsub_rn(tau, w));
                    const float sign_t = tt > 0.f ? 1.f : -1.f, n = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fmul_rn(tt, tt), 1.f)));
                    sr = __fmul_rn(__fmul_rn(__fmul_rn(-sign_t, __fdiv_rn(n01, fabsf(n01))), fabsf(tt)), n);
                    cr = n;
                }
                // j_left = rot1 * j_right.transpose()
                const float cl = __fsub_rn(__fmul_rn(c1, cr), __fmul_rn(s1, -sr)), sl = __fadd_rn(__fmul_rn(c1, -sr), __fmul_rn(s1, cr));
                if (!(cl == 1.f && sl == 0.f)) {            // W.applyOnTheLeft(p, q, j_left): rows p, q
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float x = W[p][k], y = W[q][k];
                        W[p][k] = __fadd_rn(__fmul_rn(cl, x), __fmul_rn(sl, y)); W[q][k] = __fadd_rn(__fmul_rn(-sl, x), __fmul_rn(cl, y));
                    }
                }
                if (!(cr == 1.f && sr == 0.f)) {            // W and V .applyOnTheRight(p, q, j_right): columns p, q with (cr, -sr)
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float x = W[k][p], y = W[k][q];
                        W[k][p] = __fadd_rn(__fmul_rn(cr, x), __fmul_rn(-sr, y)); W[k][q] = __fadd_rn(__fmul_rn(sr, x), __fmul_rn(cr, y));
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float x = V[k][p], y = V[k][q];
                        V[k][p] = __fadd_rn(__fmul_rn(cr, x), __fmul_rn(-sr, y)); V[k][q] = __fadd_rn(__fmul_rn(sr, x), __fmul_rn(cr, y));
                    }
                }
                max_diag = fmaxf(max_diag, fmaxf(fabsf(W[p][p]), fabsf(W[q][q])));
            }
    }
    if (!finished) return false;
    float sv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) sv[i] = __fmul_rn(fabsf(W[i][i]), scale);
    // descending sort, first maximum, stopping at a zero maximum; columns of V follow
    bool stop = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float mx = sv[i]; int pos = i;
#pragma unroll
        for (int k = i + 1; k < 4; ++k) if (sv[k] > mx) { mx = sv[k]; pos = k; }
        if (stop || mx == 0.f) { stop = true; continue; }
#pragma unroll
        for (int k = i + 1; k < 4; ++k)
            if (pos == k) {
                const float t = sv[i]; sv[i] = sv[k]; sv[k] = t;
#pragma unroll
                for (int r = 0; r < 4; ++r) { const float v = V[r][i]; V[r][i] = V[r][k]; V[r][k] = v; }
            }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) v3[r] = V[r][3];
    return true;
}

// reprojection test of one key frame (mono: Pinhole::project, 5.991 sigma^2; stereo: invz = 1.0 / z in double, 7.8 sigma^2)
__device__ __forceinline__ bool reprojection_ok(const CnmpCam& cam, const float Rcw[9], const float* tcw, const float x3D[3], float z,
                                                const rgbl_keypoint& kp, bool stereo, float ur) {
    const float sigma2 = cam.sigma2[kp.octave];
    const float x = __fadd_rn(dot3(Rcw, x3D), tcw[0]), y = __fadd_rn(dot3(Rcw + 3, x3D), tcw[1]);
    const float invz = (float)(1.0 / (double)z);
    if (!stereo) {
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(cam.fx, x), z), cam.cx), v = __fadd_rn(__fdiv_rn(__fmul_rn(cam.fy, y), z), cam.cy);
        const float ex = __fsub_rn(u, kp.x), ey = __fsub_rn(v, kp.y);
        return !((double)__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)) > 5.991 * (double)sigma2);
    }
    const float u = __fadd_rn(__fmul_rn(__fmul_rn(cam.fx, x), invz), cam.cx);
    const float u_r = __fsub_rn(u, __fmul_rn(cam.bf, invz));
    const float v = __fadd_rn(__fmul_rn(__fmul_rn(cam.fy, y), invz), cam.cy);
    const float ex = __fsub_rn(u, kp.x), ey = __fsub_rn(v, kp.y), er = __fsub_rn(u_r, ur);
    return !((double)__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er)) > 7.8 * (double)sigma2);
}

// KeyFrame::UnprojectStereo (src/KeyFrame.cc): the distorted keypoint, x3D = mRwc * x3Dc + mTwc.translation()
__device__ __forceinline__ bool unproject_stereo(const CnmpCam& cam, const float* pose, const CnmpFrame& f, int i, float x3D[3]) {
    const float z = f.depth[i];
    if (!(z > 0.f)) return false;
    const rgbl_keypoint kp = f.keys[i];
    float Rwc[9], Ow[3];
    chain_pose_matrices(pose, Rwc, Ow);
    const float pc[3] = {__fmul_rn(__fmul_rn(__fsub_rn(kp.x, cam.cx), z), cam.invfx), __fmul_rn(__fmul_rn(__fsub_rn(kp.y, cam.cy), z), cam.invfy), z};
#pragma unroll
    for (int r = 0; r < 3; ++r) x3D[r] = __fadd_rn(dot3(Rwc + 3 * r, pc), Ow[r]);
    return true;
}

// One thread per (neighbour, key-frame-1 feature) slot with a candidate match: steps 1-6 of CreateNewMapPoints' loop body.
__global__ void __launch_bounds__(128) cnmp_triangulate_kernel(int n_slots, int n1, const int* __restrict__ match, const float* __restrict__ pose1,
                                                               const float* __restrict__ poses2, CnmpFrame F1, CnmpFrame F2, CnmpCam cam,
                                                               uint8_t* __restrict__ ok_out, float* __restrict__ x_out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const int g2 = match[s];
    ok_out[s] = 0;
    if (g2 < 0) return;
    const int j = s / n1, idx1 = s - j * n1;
    const float* pose2 = poses2 + 7 * j;
    float Rcw1[9], Rcw2[9];
    quatf_to_matrix(pose1, Rcw1); quatf_to_matrix(pose2, Rcw2);
    const float* tcw1 = pose1 + 4; const float* tcw2 = pose2 + 4;
    const rgbl_keypoint kp1 = F1.keys_un[idx1], kp2 = F2.keys_un[g2];
    const float ur1 = F1.uright[idx1], ur2 = F2.uright[g2];
    const bool st1 = ur1 >= 0.f, st2 = ur2 >= 0.f;
    // Pinhole::unprojectEig; rays in the world frame with Rwc = Rcw^T
    const float xn1[3] = {__fdiv_rn(__fsub_rn(kp1.x, cam.cx), cam.fx), __fdiv_rn(__fsub_rn(kp1.y, cam.cy), cam.fy), 1.f};
    const float xn2[3] = {__fdiv_rn(__fsub_rn(kp2.x, cam.cx), cam.fx), __fdiv_rn(__fsub_rn(kp2.y, cam.cy), cam.fy), 1.f};
    float ray1[3], ray2[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        ray1[r] = eig_sum3(__fmul_rn(Rcw1[r], xn1[0]), __fmul_rn(Rcw1[3 + r], xn1[1]), __fmul_rn(Rcw1[6 + r], xn1[2]));
        ray2[r] = eig_sum3(__fmul_rn(Rcw2[r], xn2[0]), __fmul_rn(Rcw2[3 + r], xn2[1]), __fmul_rn(Rcw2[6 + r], xn2[2]));
    }
    const float cos_rays = __fdiv_rn(dot3(ray1, ray2), __fmul_rn(__fsqrt_rn(dot3(ray1, ray1)), __fsqrt_rn(dot3(ray2, ray2))));
    float cos_st1 = __fadd_rn(cos_rays, 1.f), cos_st2 = cos_st1;
    // cos(2 atan2(mb / 2, depth)): double libm calls, as the reference's unqualified cos / atan2 resolve to them
    if (st1) cos_st1 = (float)cos(2.0 * atan2((double)__fdiv_rn(cam.mb, 2.f), (double)F1.depth[idx1]));
    else if (st2) cos_st2 = (float)cos(2.0 * atan2((double)__fdiv_rn(cam.mb, 2.f), (double)F2.depth[g2]));
    const float cos_st = cos_st2 < cos_st1 ? cos_st2 : cos_st1;
    float x3D[3];
    if (cos_rays < cos_st && cos_rays > 0.f && (st1 || st2 || (double)cos_rays < 0.9998)) {
        // GeometricTools::Triangulate: A = [x1 P1.row(2) - P1.row(0); y1 P1.row(2) - P1.row(1); same for 2], V.col(3) dehomogenised
        float A[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float p10 = k < 3 ? Rcw1[k] : tcw1[0], p11 = k < 3 ? Rcw1[3 + k] : tcw1[1], p12 = k < 3 ? Rcw1[6 + k] : tcw1[2];
            const float p20 = k < 3 ? Rcw2[k] : tcw2[0], p21 = k < 3 ? Rcw2[3 + k] : tcw2[1], p22 = k < 3 ? Rcw2[6 + k] : tcw2[2];
            A[0][k] = __fsub_rn(__fmul_rn(xn1[0], p12), p10); A[1][k] = __fsub_rn(__fmul_rn(xn1[1], p12), p11);
            A[2][k] = __fsub_rn(__fmul_rn(xn2[0], p22), p20); A[3][k] = __fsub_rn(__fmul_rn(xn2[1], p22), p21);
        }
        float v[4];
        if (!jacobi_svd4_null(A, v) || v[3] == 0.f) return;
        x3D[0] = __fdiv_rn(v[0], v[3]); x3D[1] = __fdiv_rn(v[1], v[3]); x3D[2] = __fdiv_rn(v[2], v[3]);
    } else if (st1 && cos_st1 < cos_st2) {
        if (!unproject_stereo(cam, pose1, F1, idx1, x3D)) return;
    } else if (st2 && cos_st2 < cos_st1) {
        if (!unproject_stereo(cam, pose2, F2, g2, x3D)) return;
    } else {
        return;                                              // no stereo and very low parallax
    }
    const float z1 = __fadd_rn(dot3(Rcw1 + 6, x3D), tcw1[2]);
    if (z1 <= 0.f) return;
    const float z2 = __fadd_rn(dot3(Rcw2 + 6, x3D), tcw2[2]);
    if (z2 <= 0.f) return;
    if (!reprojection_ok(cam, Rcw1, tcw1, x3D, z1, kp1, st1, ur1)) return;
    if (!reprojection_ok(cam, Rcw2, tcw2, x3D, z2, kp2, st2, ur2)) return;
    // scale consistency
    float q[4], Ow1[3], Ow2[3];
    se3f_inverse(pose1, q, Ow1); se3f_inverse(pose2, q, Ow2);
    const float n1v[3] = {__fsub_rn(x3D[0], Ow1[0]), __fsub_rn(x3D[1], Ow1[1]), __fsub_rn(x3D[2], Ow1[2])};
    const float n2v[3] = {__fsub_rn(x3D[0], Ow2[0]), __fsub_rn(x3D[1], Ow2[1]), __fsub_rn(x3D[2], Ow2[2])};
    const float dist1 = __fsqrt_rn(dot3(n1v, n1v)), dist2 = __fsqrt_rn(dot3(n2v, n2v));
    if (dist1 == 0.f || dist2 == 0.f) return;
    if (cam.th_far > 0.f && (dist1 >= cam.th_far || dist2 >= cam.th_far)) return;
    const float ratio_dist = __fdiv_rn(dist2, dist1), ratio_octave = __fdiv_rn(cam.scale[kp1.octave], cam.scale[kp2.octave]);
    if (__fmul_rn(ratio_dist, cam.ratio_factor) < ratio_octave || ratio_dist > __fmul_rn(ratio_octave, cam.ratio_factor)) return;
    ok_out[s] = 1;
    x_out[3 * (size_t)s] = x3D[0]; x_out[3 * (size_t)s + 1] = x3D[1]; x_out[3 * (size_t)s + 2] = x3D[2];
}

// One CTA walks the neighbours in order.  Per neighbour: the matches of features not yet claimed, the rotation histogram over them,
// their count (n_matches[j]), then the accepted points in ascending idx1 (an ordered block scan per 1024 features), which claim
// their features.  out = [created_start: n_pairs + 1][n_matches: n_pairs][idx1: M][idx2: M], xo = [x3D: 3 M]; points past M
// are counted, not written.
__global__ void __launch_bounds__(1024) cnmp_order_kernel(int n_pairs, int n1, int check_orientation, const int* __restrict__ base2,
                                                          const int* __restrict__ match, const uint8_t* __restrict__ bins, const uint8_t* __restrict__ tri_ok,
                                                          const float* __restrict__ tri_x, uint8_t* __restrict__ claimed, int M, int* __restrict__ out,
                                                          float* __restrict__ xo) {
    __shared__ int hist[32], keep[3], warp_sum[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int* created_start = out; int* n_matches = out + n_pairs + 1; int* o_idx1 = n_matches + n_pairs; int* o_idx2 = o_idx1 + M;
    int total = 0;
    if (tid == 0) created_start[0] = 0;
    for (int j = 0; j < n_pairs; ++j) {
        const int* mj = match + (size_t)j * n1; const uint8_t* bj = bins + (size_t)j * n1;
        if (check_orientation) {
            if (tid < 32) hist[tid] = 0;
            __syncthreads();
            for (int i = tid; i < n1; i += 1024) if (mj[i] >= 0 && !claimed[i]) atomicAdd(&hist[bj[i]], 1);
            __syncthreads();
            if (tid < 32) three_maxima_keep(hist, keep);
            __syncthreads();
        }
        int nm = 0;
        for (int base = 0; base < n1; base += 1024) {
            const int i = base + tid;
            bool live = i < n1 && mj[i] >= 0 && !claimed[i];
            if (live && check_orientation) { const int b = bj[i]; live = b == keep[0] || b == keep[1] || b == keep[2]; }
            const bool acc = live && tri_ok[(size_t)j * n1 + i];
            const unsigned bal = __ballot_sync(0xffffffffu, acc);
            if (lane == 0) warp_sum[warp] = __popc(bal);
            nm += __syncthreads_count(live);                 // also orders warp_sum
            int before = 0, chunk = 0;
            for (int w = 0; w < 32; ++w) { const int v = warp_sum[w]; before += w < warp ? v : 0; chunk += v; }
            if (acc) {
                const int pos = total + before + __popc(bal & ((1u << lane) - 1u));
                if (pos < M) {
                    o_idx1[pos] = i; o_idx2[pos] = mj[i] - base2[j];
                    const float* x = tri_x + 3 * ((size_t)j * n1 + i);
                    xo[3 * pos] = x[0]; xo[3 * pos + 1] = x[1]; xo[3 * pos + 2] = x[2];
                }
                claimed[i] = 1;
            }
            total += chunk;
            __syncthreads();                                 // warp_sum is rewritten by the next chunk; claimed[] is read by the next neighbour
        }
        if (tid == 0) { created_start[j + 1] = total; n_matches[j] = nm; }
    }
}

}  // namespace
}  // namespace rgbl

using namespace rgbl;

extern "C" {

int rgbl_distinctive_descriptors(rgbl_ctx* ctx, int n_points, const int32_t* obs_start, const uint8_t* desc, int32_t* best) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (n_points < 0 || (n_points > 0 && (!obs_start || !best))) { c->err = "bad argument"; return RGBL_E_INVALID; }
    if (n_points == 0) return RGBL_OK;
    const int total = obs_start[n_points];
    if (obs_start[0] != 0 || total < 0 || (total > 0 && !desc)) { c->err = "bad observation table"; return RGBL_E_INVALID; }
    for (int p = 0; p < n_points; ++p) if (obs_start[p + 1] < obs_start[p]) { c->err = "obs_start is not monotone"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    ArenaCarve a(c, (size_t)(n_points + 1) * 4 + (size_t)total * 32 + (size_t)n_points * 4 + 4096);
    if (!a.base) { c->err = "device allocation failed (distinctive descriptors)"; return RGBL_E_CUDA; }
    int* d_start = a.take<int>(n_points + 1); uint8_t* d_desc = a.take<uint8_t>((size_t)std::max(total, 1) * 32); int* d_best = a.take<int>(n_points);
    CU(cudaMemcpyAsync(d_start, obs_start, (size_t)(n_points + 1) * 4, cudaMemcpyHostToDevice, c->st));
    if (total) CU(cudaMemcpyAsync(d_desc, desc, (size_t)total * 32, cudaMemcpyHostToDevice, c->st));
    stage_begin(c, ST_MATCH, c->st);
    distinctive_kernel<<<(n_points + 3) / 4, 128, 0, c->st>>>(n_points, d_start, d_desc, d_best);
    stage_end(c, ST_MATCH, c->st, 1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(best, d_best, (size_t)n_points * 4, cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_search_for_triangulation(rgbl_ctx* ctx, int n1, const uint8_t* desc1, const rgbl_keypoint* keys1, const uint8_t* has_mp1, const float* uright1,
                                  int nn1, const uint32_t* node_ids1, const int32_t* node_start1, const int32_t* node_feat1,
                                  int n2, const uint8_t* desc2, const rgbl_keypoint* keys2, const uint8_t* has_mp2, const float* uright2,
                                  int nn2, const uint32_t* node_ids2, const int32_t* node_start2, const int32_t* node_feat2,
                                  const float F12[9], const float ep[2], int n_levels, const float* scale_factors2, const float* level_sigma2_2,
                                  int only_stereo, int coarse, int check_orientation, int32_t* match12, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (n1 < 0 || n2 < 0 || nn1 < 0 || nn2 < 0 || !match12 || !F12 || !ep || n_levels < 1 || n_levels > RGBL_MAX_LEVELS || !scale_factors2 || !level_sigma2_2 ||
        (n1 > 0 && (!desc1 || !keys1 || !has_mp1 || !uright1)) || (n2 > 0 && (!desc2 || !keys2 || !has_mp2 || !uright2)) ||
        (nn1 > 0 && (!node_ids1 || !node_start1 || !node_feat1)) || (nn2 > 0 && (!node_ids2 || !node_start2 || !node_feat2))) {
        c->err = "bad argument"; return RGBL_E_INVALID;
    }
    for (int i = 0; i < n1; ++i) match12[i] = -1;
    if (n_matches) *n_matches = 0;
    // merge-join of the two feature vectors (src/ORBmatcher.cc:958-1110); key-frame-1 features with a map point are skipped here
    std::vector<int> q_feat, q_cbeg, q_cend;
    int a = 0, b = 0;
    while (a < nn1 && b < nn2) {
        if (node_ids1[a] == node_ids2[b]) {
            for (int i1 = node_start1[a]; i1 < node_start1[a + 1]; ++i1) {
                const int idx1 = node_feat1[i1];
                if (idx1 < 0 || idx1 >= n1) { c->err = "feature index out of range (key frame 1)"; return RGBL_E_INVALID; }
                if (has_mp1[idx1]) continue;
                if (only_stereo && !(uright1[idx1] >= 0.f)) continue;
                q_feat.push_back(idx1); q_cbeg.push_back(node_start2[b]); q_cend.push_back(node_start2[b + 1]);
            }
            ++a; ++b;
        } else if (node_ids1[a] < node_ids2[b]) ++a;
        else ++b;
    }
    const int n_q = (int)q_feat.size();
    const int n_csr2 = nn2 > 0 ? node_start2[nn2] : 0;
    for (int k = 0; k < n_csr2; ++k) if (node_feat2[k] < 0 || node_feat2[k] >= n2) { c->err = "feature index out of range (key frame 2)"; return RGBL_E_INVALID; }
    for (int i = 0; i < n2; ++i) if (keys2[i].octave < 0 || keys2[i].octave >= n_levels) { c->err = "keypoint octave out of range"; return RGBL_E_INVALID; }
    if (n_q == 0 || n2 == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    ArenaCarve ar(c, (size_t)(n1 + n2) * (32 + sizeof(rgbl_keypoint) + 1 + 4 + 8) + (size_t)n_q * 12 + (size_t)n_csr2 * 4 + 16384);
    if (!ar.base) { c->err = "device allocation failed (SearchForTriangulation)"; return RGBL_E_CUDA; }
    uint8_t* d_desc1 = ar.take<uint8_t>((size_t)n1 * 32); uint8_t* d_desc2 = ar.take<uint8_t>((size_t)n2 * 32);
    rgbl_keypoint* d_k1 = ar.take<rgbl_keypoint>(n1); rgbl_keypoint* d_k2 = ar.take<rgbl_keypoint>(n2);
    uint8_t* d_mp1 = ar.take<uint8_t>(n1); uint8_t* d_mp2 = ar.take<uint8_t>(n2); float* d_ur1 = ar.take<float>(n1); float* d_ur2 = ar.take<float>(n2);
    int* d_q = ar.take<int>((size_t)3 * n_q); int* d_nf2 = ar.take<int>(std::max(n_csr2, 1)); int* d_match = ar.take<int>(n1); uint8_t* d_bins = ar.take<uint8_t>(n1);
    int* d_nm = ar.take<int>(4);
    auto up = [&](void* d, const void* h, size_t bytes) { return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->st); };
    CU(up(d_desc1, desc1, (size_t)n1 * 32)); CU(up(d_desc2, desc2, (size_t)n2 * 32)); CU(up(d_k1, keys1, (size_t)n1 * sizeof(rgbl_keypoint)));
    CU(up(d_k2, keys2, (size_t)n2 * sizeof(rgbl_keypoint))); CU(up(d_mp1, has_mp1, n1)); CU(up(d_mp2, has_mp2, n2)); CU(up(d_ur1, uright1, (size_t)n1 * 4));
    CU(up(d_ur2, uright2, (size_t)n2 * 4)); CU(up(d_q, q_feat.data(), (size_t)n_q * 4)); CU(up(d_q + n_q, q_cbeg.data(), (size_t)n_q * 4));
    CU(up(d_q + 2 * n_q, q_cend.data(), (size_t)n_q * 4)); CU(up(d_nf2, node_feat2, (size_t)n_csr2 * 4));
    CU(cudaMemsetAsync(d_match, 0xff, (size_t)n1 * 4, c->st));
    CU(cudaMemsetAsync(d_bins, 0xff, n1, c->st));
    TriParams prm{};
    for (int i = 0; i < 9; ++i) prm.pair.F12[i] = F12[i];
    prm.pair.ep[0] = ep[0]; prm.pair.ep[1] = ep[1];
    for (int l = 0; l < n_levels; ++l) { prm.scale2[l] = scale_factors2[l]; prm.sigma2[l] = level_sigma2_2[l]; }
    prm.only_stereo = only_stereo; prm.coarse = coarse;
    stage_begin(c, ST_MATCH, c->st);
    triangulation_search_kernel<<<(n_q + 7) / 8, 256, 0, c->st>>>(n_q, d_q, d_q + n_q, d_q + 2 * n_q, d_nf2, TriFrame{d_desc1, d_k1, d_mp1, d_ur1},
                                                                TriFrame{d_desc2, d_k2, d_mp2, d_ur2}, prm, d_match, d_bins);
    triangulation_finish_kernel<<<1, 1024, 0, c->st>>>(n1, check_orientation, d_match, d_bins, d_nm);
    stage_end(c, ST_MATCH, c->st, 2);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(match12, d_match, (size_t)n1 * 4, cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_scalars, d_nm, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    if (n_matches) *n_matches = c->h_scalars[0];
    return RGBL_OK;
}


// A key frame view is valid when its arrays exist for its sizes, its feature vector is a CSR over features 0..n-1 and its
// keypoint octaves and pose are usable.
static const char* keyframe_view_error(const rgbl_keyframe_view* v, int n_levels) {
    if (!v || v->n < 0 || v->n_nodes < 0) return "bad key frame view";
    if (v->n > 0 && (!v->desc || !v->keys || !v->keys_un || !v->uright || !v->depth || !v->has_mp)) return "missing key frame array";
    if (v->n_nodes > 0 && (!v->node_ids || !v->node_start || !v->node_feat)) return "missing feature vector array";
    for (int i = 0; i < 7; ++i) if (!std::isfinite(v->Tcw[i])) return "pose is not finite";
    if (v->n_nodes > 0) {
        if (v->node_start[0] != 0) return "feature vector does not start at 0";
        for (int a = 0; a < v->n_nodes; ++a) if (v->node_start[a + 1] < v->node_start[a]) return "node_start is not monotone";
        for (int k = 0; k < v->node_start[v->n_nodes]; ++k) if (v->node_feat[k] < 0 || v->node_feat[k] >= v->n) return "feature index out of range";
    }
    for (int i = 0; i < v->n; ++i) if (v->keys_un[i].octave < 0 || v->keys_un[i].octave >= n_levels) return "keypoint octave out of range";
    return nullptr;
}

int rgbl_create_new_map_points(rgbl_ctx* ctx, const rgbl_keyframe_view* kf1, int n_neighbours, const rgbl_keyframe_view* kf2, const float* F12,
                               const float* ep, float fx, float fy, float cx, float cy, float bf, int n_levels, const float* scale_factors,
                               const float* level_sigma2, float th_far, int check_orientation, int coarse, int32_t* created_start, int32_t* idx1,
                               int32_t* idx2, float* x3d, int cap, int32_t* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (n_neighbours < 0 || (n_neighbours > 0 && (!kf2 || !F12 || !ep)) || !created_start || cap < 0 || (cap > 0 && (!idx1 || !idx2 || !x3d)) ||
        n_levels < 2 || n_levels > RGBL_MAX_LEVELS || !scale_factors || !level_sigma2 || !std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) ||
        !std::isfinite(cy) || !std::isfinite(bf) || fx == 0.f || fy == 0.f) {
        c->err = "bad argument"; return RGBL_E_INVALID;
    }
    if (const char* e = keyframe_view_error(kf1, n_levels)) { c->err = std::string(e) + " (key frame 1)"; return RGBL_E_INVALID; }
    for (int j = 0; j < n_neighbours; ++j)
        if (const char* e = keyframe_view_error(&kf2[j], n_levels)) { c->err = std::string(e) + " (neighbour " + std::to_string(j) + ")"; return RGBL_E_INVALID; }
    const int n1 = kf1->n, np = n_neighbours;
    // queries: the merge-join of every pair's feature vectors (src/ORBmatcher.cc:958-1110) over the caller's has_mp1 only
    std::vector<int> q_feat, q_cbeg, q_cend, q_pair, base2(std::max(np, 1)), csr2(np + 1, 0);
    int n2_total = 0;
    for (int j = 0; j < np; ++j) {
        const rgbl_keyframe_view& v2 = kf2[j];
        base2[j] = n2_total; n2_total += v2.n;
        csr2[j + 1] = csr2[j] + (v2.n_nodes > 0 ? v2.node_start[v2.n_nodes] : 0);
        int a = 0, b = 0;
        while (a < kf1->n_nodes && b < v2.n_nodes) {
            if (kf1->node_ids[a] == v2.node_ids[b]) {
                for (int i1 = kf1->node_start[a]; i1 < kf1->node_start[a + 1]; ++i1) {
                    const int f = kf1->node_feat[i1];
                    if (kf1->has_mp[f]) continue;
                    q_feat.push_back(f); q_cbeg.push_back(csr2[j] + v2.node_start[b]); q_cend.push_back(csr2[j] + v2.node_start[b + 1]); q_pair.push_back(j);
                }
                ++a; ++b;
            } else if (kf1->node_ids[a] < v2.node_ids[b]) ++a;
            else ++b;
        }
    }
    const int n_q = (int)q_feat.size();
    if (n_q == 0) {
        for (int j = 0; j <= np; ++j) created_start[j] = 0;
        if (n_matches) for (int j = 0; j < np; ++j) n_matches[j] = 0;
        return RGBL_OK;
    }
    CU(cudaSetDevice(c->cfg.device));
    const int M = std::min(cap, n1), n_csr2 = csr2[np];
    const size_t n_slots = (size_t)np * n1;
    const size_t bytes = (size_t)(n1 + n2_total) * (32 + 2 * sizeof(rgbl_keypoint) + 1 + 8) + (size_t)n_q * 16 + (size_t)n_csr2 * 4 +
                         (size_t)np * (sizeof(TriPair) + 32) + 28 + n_slots * 18 + ((size_t)2 * np + 1 + 5 * (size_t)M) * 4 + 24 * 256;
    ArenaCarve ar(c, bytes);
    if (!ar.base) { c->err = "device allocation failed (CreateNewMapPoints)"; return RGBL_E_CUDA; }
    // everything the host provides is carved first and packed into one staging buffer of the same layout: one upload
    uint8_t* d_desc1 = ar.take<uint8_t>((size_t)n1 * 32); rgbl_keypoint* d_kun1 = ar.take<rgbl_keypoint>(n1); rgbl_keypoint* d_k1 = ar.take<rgbl_keypoint>(n1);
    float* d_ur1 = ar.take<float>(n1); float* d_dep1 = ar.take<float>(n1); uint8_t* d_mp1 = ar.take<uint8_t>(n1);
    uint8_t* d_desc2 = ar.take<uint8_t>((size_t)n2_total * 32); rgbl_keypoint* d_kun2 = ar.take<rgbl_keypoint>(n2_total);
    rgbl_keypoint* d_k2 = ar.take<rgbl_keypoint>(n2_total); float* d_ur2 = ar.take<float>(n2_total); float* d_dep2 = ar.take<float>(n2_total);
    uint8_t* d_mp2 = ar.take<uint8_t>(n2_total); int* d_nf2 = ar.take<int>(std::max(n_csr2, 1)); int* d_q = ar.take<int>((size_t)4 * n_q);
    TriPair* d_pairs = ar.take<TriPair>(np); float* d_pose1 = ar.take<float>(7); float* d_poses2 = ar.take<float>((size_t)7 * np); int* d_base2 = ar.take<int>(np);
    const size_t up_bytes = ar.used;
    int* d_match = ar.take<int>(n_slots); uint8_t* d_bins = ar.take<uint8_t>(n_slots); uint8_t* d_ok = ar.take<uint8_t>(n_slots);
    float* d_x = ar.take<float>(3 * n_slots);
    const size_t out_ints = (size_t)2 * np + 1 + 2 * (size_t)M;
    int* d_out = ar.take<int>(out_ints + 3 * (size_t)M);
    float* d_xo = reinterpret_cast<float*>(d_out + out_ints);
    if (ar.used > ar.cap) { c->err = "internal: CreateNewMapPoints carve exceeds its arena"; return RGBL_E_CUDA; }
    std::vector<char> stage(up_bytes);
    auto put = [&](void* d, const void* h, size_t n) { if (n) std::memcpy(stage.data() + (static_cast<char*>(d) - ar.base), h, n); };
    auto at = [&](void* d) { return stage.data() + (static_cast<char*>(d) - ar.base); };
    put(d_desc1, kf1->desc, (size_t)n1 * 32); put(d_kun1, kf1->keys_un, (size_t)n1 * sizeof(rgbl_keypoint)); put(d_k1, kf1->keys, (size_t)n1 * sizeof(rgbl_keypoint));
    put(d_ur1, kf1->uright, (size_t)n1 * 4); put(d_dep1, kf1->depth, (size_t)n1 * 4); put(d_mp1, kf1->has_mp, n1);
    put(d_pose1, kf1->Tcw, 28);
    for (int j = 0; j < np; ++j) {
        const rgbl_keyframe_view& v2 = kf2[j];
        const size_t o = base2[j];
        put(d_desc2 + 32 * o, v2.desc, (size_t)v2.n * 32); put(d_kun2 + o, v2.keys_un, (size_t)v2.n * sizeof(rgbl_keypoint));
        put(d_k2 + o, v2.keys, (size_t)v2.n * sizeof(rgbl_keypoint)); put(d_ur2 + o, v2.uright, (size_t)v2.n * 4); put(d_dep2 + o, v2.depth, (size_t)v2.n * 4);
        put(d_mp2 + o, v2.has_mp, v2.n);
        int* nf = reinterpret_cast<int*>(at(d_nf2)) + csr2[j];
        for (int k = 0; k < csr2[j + 1] - csr2[j]; ++k) nf[k] = v2.node_feat[k] + base2[j];      // global key-frame-2 indices
        TriPair pr;
        for (int i = 0; i < 9; ++i) pr.F12[i] = F12[9 * j + i];
        pr.ep[0] = ep[2 * j]; pr.ep[1] = ep[2 * j + 1];
        put(d_pairs + j, &pr, sizeof pr); put(d_poses2 + 7 * j, v2.Tcw, 28); put(d_base2 + j, &base2[j], 4);
    }
    put(d_q, q_feat.data(), (size_t)n_q * 4); put(d_q + n_q, q_cbeg.data(), (size_t)n_q * 4); put(d_q + 2 * n_q, q_cend.data(), (size_t)n_q * 4);
    put(d_q + 3 * n_q, q_pair.data(), (size_t)n_q * 4);
    CU(cudaMemcpyAsync(ar.base, stage.data(), up_bytes, cudaMemcpyHostToDevice, c->st));
    CU(cudaMemsetAsync(d_match, 0xff, n_slots * 4, c->st));
    TriParams prm{};
    for (int l = 0; l < n_levels; ++l) { prm.scale2[l] = scale_factors[l]; prm.sigma2[l] = level_sigma2[l]; }
    prm.only_stereo = 0; prm.coarse = coarse;
    CnmpCam cam{};
    cam.fx = fx; cam.fy = fy; cam.cx = cx; cam.cy = cy; cam.bf = bf; cam.mb = bf / fx; cam.invfx = 1.0f / fx; cam.invfy = 1.0f / fy;
    cam.th_far = th_far; cam.ratio_factor = 1.5f * scale_factors[1];
    for (int l = 0; l < n_levels; ++l) { cam.scale[l] = scale_factors[l]; cam.sigma2[l] = level_sigma2[l]; }
    stage_begin(c, ST_MATCH, c->st);
    cnmp_search_kernel<<<(n_q + 7) / 8, 256, 0, c->st>>>(n_q, d_q, d_q + n_q, d_q + 2 * n_q, d_q + 3 * n_q, d_nf2, TriFrame{d_desc1, d_kun1, d_mp1, d_ur1},
                                                        TriFrame{d_desc2, d_kun2, d_mp2, d_ur2}, d_pairs, prm, n1, d_match, d_bins);
    cnmp_triangulate_kernel<<<(unsigned)((n_slots + 127) / 128), 128, 0, c->st>>>((int)n_slots, n1, d_match, d_pose1, d_poses2,
                                                                                  CnmpFrame{d_k1, d_kun1, d_ur1, d_dep1}, CnmpFrame{d_k2, d_kun2, d_ur2, d_dep2},
                                                                                  cam, d_ok, d_x);
    cnmp_order_kernel<<<1, 1024, 0, c->st>>>(np, n1, check_orientation, d_base2, d_match, d_bins, d_ok, d_x, d_mp1, M, d_out, d_xo);
    stage_end(c, ST_MATCH, c->st, 3);
    CU(cudaGetLastError());
    std::vector<int> h_out(out_ints + 3 * (size_t)M);
    CU(cudaMemcpyAsync(h_out.data(), d_out, h_out.size() * 4, cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    const int total = h_out[np];
    if (total > cap) {
        c->err = "CreateNewMapPoints: " + std::to_string(total) + " points exceed cap " + std::to_string(cap);
        return RGBL_E_CAPACITY;
    }
    std::memcpy(created_start, h_out.data(), (size_t)(np + 1) * 4);
    if (n_matches) std::memcpy(n_matches, h_out.data() + np + 1, (size_t)np * 4);
    if (total) {
        std::memcpy(idx1, h_out.data() + 2 * np + 1, (size_t)total * 4);
        std::memcpy(idx2, h_out.data() + 2 * np + 1 + M, (size_t)total * 4);
        std::memcpy(x3d, h_out.data() + out_ints, (size_t)total * 12);
    }
    return RGBL_OK;
}

}  // extern "C"
