// LocalMapping-thread kernels (SURVEY 8(f) row 3): MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:329-403) for a batch
// of map points and ORBmatcher::SearchForTriangulation (src/ORBmatcher.cc:907-1146) between two key frames.  Both are
// embarrassingly parallel in this version of the reference (vbMatched2 is never set, so the key-frame-1 features are
// independent): one warp per map point / per feature, __popc Hamming, warp reductions.
#include <algorithm>
#include <cstring>
#include <vector>

#include "rgbl_ctx.h"

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
struct TriParams { float F12[9]; float ep[2]; float scale2[RGBL_MAX_LEVELS]; float sigma2[RGBL_MAX_LEVELS]; int only_stereo, coarse; };

// One warp per key-frame-1 feature that shares a vocabulary node with key frame 2.  The reference's scan keeps a candidate when
// dist <= TH_LOW and dist <= bestDist and the geometric tests pass, so it ends with the LAST candidate of minimum distance among
// those passing the tests: min over (dist << 20 | 0xfffff - position).
__global__ void __launch_bounds__(256) triangulation_search_kernel(int n_q, const int* __restrict__ q_feat, const int* __restrict__ q_cbeg,
                                                                   const int* __restrict__ q_cend, const int* __restrict__ node_feat2, TriFrame A,
                                                                   TriFrame B, TriParams prm, int* __restrict__ match12, uint8_t* __restrict__ bins) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= n_q) return;
    const int idx1 = q_feat[q];
    const rgbl_keypoint kp1 = A.keys[idx1];
    const bool stereo1 = A.uright[idx1] >= 0.f;
    // epipolar line of kp1 in image 2 (Pinhole::epipolarConstrain, src/CameraModels/Pinhole.cpp:114-117)
    const float la = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, prm.F12[0]), __fmul_rn(kp1.y, prm.F12[3])), prm.F12[6]);
    const float lb = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, prm.F12[1]), __fmul_rn(kp1.y, prm.F12[4])), prm.F12[7]);
    const float lc = __fadd_rn(__fadd_rn(__fmul_rn(kp1.x, prm.F12[2]), __fmul_rn(kp1.y, prm.F12[5])), prm.F12[8]);
    const float den = __fadd_rn(__fmul_rn(la, la), __fmul_rn(lb, lb));
    unsigned best = 0xffffffffu;
    const int cb = q_cbeg[q], ce = q_cend[q];
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
            const float ex = __fsub_rn(prm.ep[0], kp2.x), ey = __fsub_rn(prm.ep[1], kp2.y);
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
        match12[idx1] = m; bins[idx1] = bin;
    }
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
        if (tid < 32) {
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
    for (int i = 0; i < 9; ++i) prm.F12[i] = F12[i];
    prm.ep[0] = ep[0]; prm.ep[1] = ep[1];
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

}  // extern "C"
