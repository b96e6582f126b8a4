// Tracking-thread matcher kernels for sm_90a.
//   grid build          Frame::AssignFeaturesToGrid / PosInGrid          src/Frame.cc:475-506, 815-825
//   candidate search    Frame::GetFeaturesInArea + DescriptorDistance    src/Frame.cc:747-813, src/ORBmatcher.cc:2058-2074
//   SearchByProjection(CurrentFrame, LastFrame, th, bMono)               src/ORBmatcher.cc:1676-1887
//   SearchByProjection(F, vpMapPoints, th, bFarPoints, thFarPoints)      src/ORBmatcher.cc:43-213
//   Frame::isInFrustum + MapPoint::PredictScale                          src/Frame.cc:602-664, src/MapPoint.cc:531-545
//
// The reference loops are sequential and greedy: a feature claimed by an earlier map point (with
// Observations() > 0) is skipped by later ones, so results depend on iteration order.  Here the
// distance work is data-parallel (collect kernels: one warp per query, __popc Hamming over the 64x48 grid's
// CSR ranges; every query's candidates sorted by key and appended to one dense run) and the greedy order is
// reproduced afterwards by an exact "serial dictatorship" resolution (resolve_kernel, one CTA, everything in
// shared memory): in rounds, a waiting query becomes final as soon as it is the lowest-index waiting query
// among those that list its best and its second-best available feature - the set of available features only
// shrinks until its turn, so those two are then still its best two.  The lowest waiting query is always final,
// so the loop terminates; on real data a handful of rounds suffice.  Candidate order (which decides ties) is the
// reference's: grid column, then row, then keypoint index = ascending position in the column-major CSR.
// tests/test_resolution_model.py checks the scheme against the sequential loops; DESIGN.md 5b has the measurements
// that shaped the kernel (no shared-memory atomics per round, no data-dependent loops in the decision).
#include <cfloat>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

constexpr int kGridCells = kGridCols * kGridRows;
constexpr int kThHigh = 100;          // ORBmatcher::TH_HIGH
constexpr int kHistoLength = 30;      // ORBmatcher::HISTO_LENGTH
constexpr uint32_t kPosMask = (1u << 20) - 1u;
// A candidate entry, as the collect kernels write it and the resolution reads it: hi word = key (distance << 20 | scan position: ascending key =
// the reference's preference order incl. ties), lo word = rotation bin << 24 | octave << 20 | frame feature (< 2^20).
typedef unsigned long long MatchEntry;
__device__ __forceinline__ MatchEntry ent_make(uint32_t key, unsigned bin, unsigned oc, unsigned ft) { return ((MatchEntry)key << 32) | (bin << 24) | ((oc & 0xfu) << 20) | ft; }
__device__ __forceinline__ uint32_t ent_key(MatchEntry e) { return (uint32_t)(e >> 32); }
__device__ __forceinline__ int ent_ft(MatchEntry e) { return (int)((unsigned)e & 0xfffffu); }
__device__ __forceinline__ int ent_oc(MatchEntry e) { return (int)(((unsigned)e >> 20) & 0xfu); }
__device__ __forceinline__ int ent_bin(MatchEntry e) { return (int)((unsigned)e >> 24); }
__device__ __forceinline__ unsigned rotation_bin(float q_angle, float f_angle) {          // src/ORBmatcher.cc:1820-1828 (rot, bin = round(rot * factor))
    float rot = __fsub_rn(q_angle, f_angle);
    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
    int b = (int)roundf(__fmul_rn(rot, 1.0f / 30));
    if (b == 30) b = 0;
    return (unsigned)b & 0xffu;
}
// where a collect kernel writes the candidates of query q: entries + (parallel) the slot of each entry in its feature's inverse list
struct ListOut {
    MatchEntry* lists; uint16_t* slots; int list_cap; int* list_n;      // per-query staging lists (list_cap entries each) while a query's candidates are collected
    // ... and the finished lists of ALL queries appended to one dense run (entry, slot, owning query): what the single-CTA resolution reads,
    // coalesced - its share of the L2 bandwidth is one SM's, and 2-4 k scattered sectors cost it ~10 k cycles.  total = entries so far
    // (zero between launches), base[q] = where query q's list starts.
    MatchEntry* dense; uint16_t* dense_slot; int* dense_q; int* base; int* total;
    int* inv_cnt;                    // per frame feature: entries listing it so far (global atomics here, many CTAs: the single-CTA resolution
                                     // then builds its inverse index feature -> queries without any shared-memory atomic; zero between launches)
    int* overflow;
};
constexpr int kListUnsorted = 1 << 30;        // flag in list_n[q]: the list is in scan order, not ascending by key (more than 32 candidates)
constexpr int kListCountMask = kListUnsorted - 1;

// ---- grid --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) grid_build_kernel(FrameDev f, int kp_stride, int* __restrict__ cell_start /*kGridCells+1*/,
                                                          int* __restrict__ csr_idx, int* __restrict__ kp_cell) {
    __shared__ int cnt[kGridCells];
    __shared__ int off[kGridCells + 1];
    const int tid = threadIdx.x;
    {   // batched launch: one CTA per frame
        const size_t b = blockIdx.x;
        f.n += b; f.keys += b * kp_stride;
        cell_start += b * (kGridCells + 1); csr_idx += b * kp_stride; kp_cell += b * kp_stride;
    }
    const int n = *f.n;
    for (int c = tid; c < kGridCells; c += 1024) cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += 1024) {
        const rgbl_keypoint kp = f.keys[i];
        const int px = (int)roundf(__fmul_rn(__fsub_rn(kp.x, f.min_x), f.inv_w));
        const int py = (int)roundf(__fmul_rn(__fsub_rn(kp.y, f.min_y), f.inv_h));
        int c = -1;
        if (px >= 0 && px < kGridCols && py >= 0 && py < kGridRows) { c = px * kGridRows + py; atomicAdd(&cnt[c], 1); }
        kp_cell[i] = c;
    }
    __syncthreads();
    {   // block-wide exclusive scan of the 3072 cell counts: 3 consecutive cells per thread + warp/block scan
        __shared__ int wsum[32];
        const int c0 = tid * 3;
        const int a0 = cnt[c0], a1 = cnt[c0 + 1], a2 = cnt[c0 + 2];
        const int mine = a0 + a1 + a2;
        int incl = mine;
        const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int v = wsum[lane], w = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
            wsum[lane] = w - v;                      // exclusive prefix of the warp totals
        }
        __syncthreads();
        const int base = wsum[warp] + incl - mine;
        off[c0] = base; off[c0 + 1] = base + a0; off[c0 + 2] = base + a0 + a1;
        if (tid == 1023) off[kGridCells] = base + mine;
    }
    __syncthreads();
    for (int c = tid; c <= kGridCells; c += 1024) cell_start[c] = off[c];
    for (int c = tid; c < kGridCells; c += 1024) cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += 1024) {
        const int c = kp_cell[i];
        if (c >= 0) csr_idx[off[c] + atomicAdd(&cnt[c], 1)] = i;
    }
    __syncthreads();
    // insertion order inside a cell is ascending keypoint index: sort each (tiny) cell list
    for (int c = tid; c < kGridCells; c += 1024) {
        const int b = off[c], e = off[c + 1];
        for (int a = b + 1; a < e; ++a) {
            const int v = csr_idx[a];
            int k = a - 1;
            while (k >= b && csr_idx[k] > v) { csr_idx[k + 1] = csr_idx[k]; --k; }
            csr_idx[k + 1] = v;
        }
    }
}

// ---- shared helpers ------------------------------------------------------------------------------
__device__ __forceinline__ int hamming256(const uint4 a0, const uint4 a1, const uint8_t* __restrict__ b) {
    const uint4 b0 = __ldg(reinterpret_cast<const uint4*>(b)), b1 = __ldg(reinterpret_cast<const uint4*>(b) + 1);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

struct CellRange { int min_cx, max_cx, min_cy, max_cy; bool ok; };

__device__ __forceinline__ CellRange cell_range(const FrameDev& f, float x, float y, float r) {
    CellRange c; c.ok = false;
    c.min_cx = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, f.min_x), r), f.inv_w)));
    if (c.min_cx >= kGridCols) return c;
    c.max_cx = min(kGridCols - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, f.min_x), r), f.inv_w)));
    if (c.max_cx < 0) return c;
    c.min_cy = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, f.min_y), r), f.inv_h)));
    if (c.min_cy >= kGridRows) return c;
    c.max_cy = min(kGridRows - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, f.min_y), r), f.inv_h)));
    if (c.max_cy < 0) return c;
    c.ok = true;
    return c;
}

// One warp scans the candidate cells of a query and appends every admissible candidate as
// key = dist << 20 | csr_pos to the query's list (warp-aggregated append into a global pool).
// `keep_max` = largest distance that can still influence the decision.
template <class Filter>
__device__ __forceinline__ int warp_collect(const FrameDev& f, const int* __restrict__ cell_start,
                                            const int* __restrict__ csr_idx, const CellRange cr, float x, float y,
                                            float r, int min_level, int max_level, const uint4 d0, const uint4 d1,
                                            int keep_max, const ListOut& out, int q, Filter admit,
                                            bool want_bin = false, float q_angle = 0.f) {
    MatchEntry* __restrict__ list = out.lists + (size_t)q * out.list_cap;
    uint16_t* __restrict__ slots = out.slots + (size_t)q * out.list_cap;
    const int list_cap = out.list_cap;
    const int lane = threadIdx.x & 31;
    const bool check_levels = (min_level > 0) || (max_level >= 0);
    int count = 0;
    // The cell columns of the search window are contiguous CSR segments (column-major grid).  Walking them one by one costs a
    // chain of dependent global loads per column (cell bounds -> index -> keypoint -> descriptor); instead the lanes fetch all
    // segment bounds at once, scan their lengths and then stride over the CONCATENATED candidate range, so a typical window
    // (3-7 columns, a few dozen candidates) is one or two trips.  Order of the candidates = ascending CSR position, as before.
    const int ncol = cr.max_cx - cr.min_cx + 1;
    for (int c0 = 0; c0 < ncol; c0 += 32) {
        const int nc = min(32, ncol - c0);
        int seg_b = 0, seg_len = 0;
        if (lane < nc) {
            const int ix = cr.min_cx + c0 + lane;
            seg_b = cell_start[ix * kGridRows + cr.min_cy];
            seg_len = cell_start[ix * kGridRows + cr.max_cy + 1] - seg_b;
        }
        int incl = seg_len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        for (int t0 = 0; t0 < total; t0 += 32) {
            const int t = min(t0 + lane, total - 1);
            int lo = 0, hi = 31;                                  // first segment whose inclusive count exceeds t (uniform 5 steps)
#pragma unroll
            for (int step = 0; step < 5; ++step) {
                const int mid = (lo + hi) >> 1;
                const int v = __shfl_sync(0xffffffffu, incl, mid);
                if (v > t) hi = mid; else lo = mid + 1;
            }
            const int sb = __shfl_sync(0xffffffffu, seg_b, lo), sl = __shfl_sync(0xffffffffu, seg_len, lo), si = __shfl_sync(0xffffffffu, incl, lo);
            const int p = sb + (t - (si - sl));
            bool keep = false;
            MatchEntry key = 0;
            if (t0 + lane < total) {
                const int idx = csr_idx[p];
                const rgbl_keypoint kp = f.keys[idx];
                bool ok = true;
                if (check_levels) {
                    if (kp.octave < min_level) ok = false;
                    if (max_level >= 0 && kp.octave > max_level) ok = false;
                }
                if (ok) {
                    const float dx = __fsub_rn(kp.x, x), dy = __fsub_rn(kp.y, y);
                    ok = fabsf(dx) < r && fabsf(dy) < r;
                }
                if (ok) ok = admit(idx);
                if (ok) {
                    const int d = hamming256(d0, d1, f.desc + (size_t)idx * 32);
                    if (d <= keep_max) {
                        keep = true;
                        key = ent_make(((uint32_t)d << 20) | (uint32_t)p, want_bin ? rotation_bin(q_angle, kp.angle) : 0u, (unsigned)kp.octave, (unsigned)idx);
                    }
                }
            }
            const uint32_t m = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const int o = count + __popc(m & ((1u << lane) - 1u));
                if (o < list_cap) { list[o] = key; slots[o] = (uint16_t)atomicAdd(&out.inv_cnt[ent_ft(key)], 1); }       // only stored entries count
            }
            count += __popc(m);
        }
    }
    return count;
}

// The resolution reads a query's candidates best first (ascending key = distance, then scan position): called by the whole warp after
// its list is complete, sorts lists of <= 32 keys in place by ranking (keys of one list are unique) and returns the value for list_n[q].
__device__ __forceinline__ int warp_finish_list(const ListOut& lo, int q, int count) {
    MatchEntry* __restrict__ list = lo.lists + (size_t)q * lo.list_cap;
    uint16_t* __restrict__ slots = lo.slots + (size_t)q * lo.list_cap;
    const int n = min(count, lo.list_cap);
    if (n == 0) return 0;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == 0) { base = atomicAdd(lo.total, n); lo.base[q] = base; }
    base = __shfl_sync(0xffffffffu, base, 0);
    __syncwarp();                                       // the list was written by other lanes of this warp
    if (n > 32) {                                       // left in scan order (flagged), copied as it is
        for (int i = lane; i < n; i += 32) { lo.dense[base + i] = list[i]; lo.dense_slot[base + i] = slots[i]; lo.dense_q[base + i] = q; }
        return n | kListUnsorted;
    }
    const MatchEntry k = lane < n ? list[lane] : ~0ull;
    const uint16_t sl = lane < n ? slots[lane] : (uint16_t)0;
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += (__shfl_sync(0xffffffffu, k, j) < k) ? 1 : 0;
    __syncwarp();
    if (lane < n) {
        list[rank] = k; slots[rank] = sl;               // the staging list stays valid (sorted): the global-memory fallback of the resolution reads it
        lo.dense[base + rank] = k; lo.dense_slot[base + rank] = sl; lo.dense_q[base + rank] = q;
    }
    return n;
}

// ---- SearchByProjection(CurrentFrame, LastFrame): candidate phase --------------------------------
template <bool kLanes>
__global__ void __launch_bounds__(256) search_last_collect_kernel(Laned<FrameDev> f_l, Laned<const int*> cell_start_l, Laned<const int*> csr_idx_l,
                                                                  Laned<LastFrameDev> lf_l, Laned<SearchLastParams> prm_l, Laned<ListOut> out_l) {
    pdl_wait(); pdl_trigger();
    const unsigned ln_ = blockIdx.y;
    const FrameDev& f = lane_arg<kLanes>(f_l, ln_);
    const int* __restrict__ cell_start = lane_arg<kLanes>(cell_start_l, ln_);
    const int* __restrict__ csr_idx = lane_arg<kLanes>(csr_idx_l, ln_);
    const LastFrameDev& lf = lane_arg<kLanes>(lf_l, ln_);
    const SearchLastParams& prm = lane_arg<kLanes>(prm_l, ln_);
    const ListOut& out = lane_arg<kLanes>(out_l, ln_);
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= lf.n) return;
    int count = 0;
    if (lf.valid[q]) {
        const float p[3] = {lf.xw[3 * q], lf.xw[3 * q + 1], lf.xw[3 * q + 2]};
        float xc[3];
        const float* T = prm.cur_pose_dev ? prm.cur_pose_dev : prm.cur_pose;
        se3f_rotate(T, p, xc);
        xc[0] = __fadd_rn(xc[0], T[4]); xc[1] = __fadd_rn(xc[1], T[5]); xc[2] = __fadd_rn(xc[2], T[6]);
        const float invzc = (float)__ddiv_rn(1.0, (double)xc[2]);
        bool ok = !(invzc < 0);
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(f.fx, xc[0]), xc[2]), f.cx);
        const float v = __fadd_rn(__fdiv_rn(__fmul_rn(f.fy, xc[1]), xc[2]), f.cy);
        if (ok && (u < f.min_x || u > f.max_x)) ok = false;
        if (ok && (v < f.min_y || v > f.max_y)) ok = false;
        if (ok) {
            const int oct = lf.octave[q];
            const float radius = __fmul_rn(prm.th, f.scale[oct]);
            int lo, hi;
            const int fwd = prm.flags_dev ? prm.flags_dev[0] : prm.forward, bwd = prm.flags_dev ? prm.flags_dev[1] : prm.backward;
            if (fwd) { lo = oct; hi = -1; }
            else if (bwd) { lo = 0; hi = oct; }
            else { lo = oct - 1; hi = oct + 1; }
            const CellRange cr = cell_range(f, u, v, radius);
            if (cr.ok) {
                const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(lf.desc + (size_t)q * 32));
                const uint4 d1 = __ldg(reinterpret_cast<const uint4*>(lf.desc + (size_t)q * 32) + 1);
                const float ur = __fsub_rn(u, __fmul_rn(f.bf, invzc));
                const float* uright = f.uright;
                count = warp_collect(f, cell_start, csr_idx, cr, u, v, radius, lo, hi, d0, d1, kThHigh,
                                     out, q, [&](int idx) {
                                         const float urt = uright[idx];
                                         if (urt > 0.f) { if (fabsf(__fsub_rn(ur, urt)) > radius) return false; }
                                         return true;
                                     }, prm.check_orientation != 0, lf.angle[q]);
            }
        }
    }
    const int ln = warp_finish_list(out, q, count);
    if (lane == 0) {
        out.list_n[q] = ln;
        if (count > out.list_cap) atomicExch(out.overflow, 3);
    }
}

// ---- SearchByProjection(F, vpMapPoints): candidate phase ---------------------------------------------
// Resident chain only (ho.ring.valid != nullptr): the first CTAs of the grid also hand the LAST frame's points over to the local map ring
// (MapPoint::UpdateNormalAndDepth with one observation, src/MapPoint.cc:437-490; ring slot = frames inserted so far mod K) - a streaming
// copy of ~100 bytes per point that a single CTA (the resolution kernel's tail, where it used to be) pays 4 us for.  Nothing in this
// kernel or in the resolution reads the ring (the edges take local points from the query copy), the frame counter is advanced afterwards.
struct RingHandOverDev {
    LocalRingDev ring; const float* last_xw; int n_last_cap; const uint8_t* last_valid; const int* last_octave; const uint8_t* last_desc; const float* last_pose;
};

template <bool kLanes>
__global__ void __launch_bounds__(256) search_local_collect_kernel(Laned<FrameDev> f_l, Laned<const int*> cell_start_l, Laned<const int*> csr_idx_l,
                                                                   Laned<LocalPointsDev> lp_l, SearchLocalParams prm, Laned<ListOut> out_l,
                                                                   Laned<RingHandOverDev> ho_l) {
    pdl_wait(); pdl_trigger();
    const unsigned ln_ = blockIdx.y;
    const FrameDev& f = lane_arg<kLanes>(f_l, ln_);
    const int* __restrict__ cell_start = lane_arg<kLanes>(cell_start_l, ln_);
    const int* __restrict__ csr_idx = lane_arg<kLanes>(csr_idx_l, ln_);
    const LocalPointsDev& lp = lane_arg<kLanes>(lp_l, ln_);
    const ListOut& out = lane_arg<kLanes>(out_l, ln_);
    const RingHandOverDev& ho = lane_arg<kLanes>(ho_l, ln_);
    if (ho.ring.valid) {
        const int j = blockIdx.x * 256 + threadIdx.x;
        if (j < ho.ring.cap) {
            const size_t p = (size_t)(*ho.ring.count % ho.ring.K) * ho.ring.cap + j;
            uint8_t v = 0;
            if (j < ho.n_last_cap && ho.last_valid[j]) {
                const float P[3] = {ho.last_xw[3 * j], ho.last_xw[3 * j + 1], ho.last_xw[3 * j + 2]};
                const int loct = ho.last_octave[j];
                const uint4 d0 = reinterpret_cast<const uint4*>(ho.last_desc + (size_t)j * 32)[0];
                const uint4 d1 = reinterpret_cast<const uint4*>(ho.last_desc + (size_t)j * 32)[1];
                float T[7], qinv[4], Ow[3];
#pragma unroll
                for (int k = 0; k < 7; ++k) T[k] = ho.last_pose[k];
                se3f_inverse(T, qinv, Ow);                 // KeyFrame::GetCameraCenter of the frame the points were created from
                const float PC[3] = {__fsub_rn(P[0], Ow[0]), __fsub_rn(P[1], Ow[1]), __fsub_rn(P[2], Ow[2])};
                const float dist = sqrtf(eig_sum3(__fmul_rn(PC[0], PC[0]), __fmul_rn(PC[1], PC[1]), __fmul_rn(PC[2], PC[2])));
                ho.ring.xw[3 * p] = P[0]; ho.ring.xw[3 * p + 1] = P[1]; ho.ring.xw[3 * p + 2] = P[2];
                ho.ring.normal[3 * p] = __fdiv_rn(PC[0], dist); ho.ring.normal[3 * p + 1] = __fdiv_rn(PC[1], dist); ho.ring.normal[3 * p + 2] = __fdiv_rn(PC[2], dist);
                const float mx = __fmul_rn(dist, f.scale[loct]);
                ho.ring.mf_max[p] = mx;
                ho.ring.mf_min[p] = __fdiv_rn(mx, f.scale[f.n_levels - 1]);
                uint4* dd = reinterpret_cast<uint4*>(ho.ring.desc + p * 32);
                dd[0] = d0; dd[1] = d1;
                v = 1;
            }
            ho.ring.valid[p] = v;
        }
    }
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= (lp.n_dev ? min(*lp.n_dev, lp.n) : lp.n)) return;
    int count = 0;
    bool active = lp.in_view[q] != 0;
    if (active && prm.far_points && lp.depth[q] > prm.th_far) active = false;
    if (active) {
        const int pl = lp.level[q];
        float r = ((double)lp.view_cos[q] > 0.998) ? 2.5f : 4.0f;
        if (prm.use_factor) r = __fmul_rn(r, prm.th);
        const float rad = __fmul_rn(r, f.scale[pl]);
        const float x = lp.proj_x[q], y = lp.proj_y[q];
        const CellRange cr = cell_range(f, x, y, rad);
        if (cr.ok) {
            const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(lp.desc + (size_t)q * 32));
            const uint4 d1 = __ldg(reinterpret_cast<const uint4*>(lp.desc + (size_t)q * 32) + 1);
            const float xr = lp.proj_xr[q];
            const float* uright = f.uright;
            count = warp_collect(f, cell_start, csr_idx, cr, x, y, rad, pl - 1, pl, d0, d1, prm.keep_max,
                                 out, q, [&](int idx) {
                                     const float urt = uright[idx];
                                     if (urt > 0.f) { if (fabsf(__fsub_rn(xr, urt)) > rad) return false; }
                                     return true;
                                 });
        }
    }
    const int ln = warp_finish_list(out, q, count);
    if (lane == 0) {
        out.list_n[q] = ln;
        if (count > out.list_cap) atomicExch(out.overflow, 3);
    }
}

// ---- greedy resolution (single CTA) -------------------------------------------------------------------
// mode 0: last-frame search (best <= TH_HIGH wins, rotation histogram);  mode 1: local-map search
// (best / second best with levels, ratio test).  state[f]: 0 free, 1 blocked (holds a point with
// observations), 2 holds a 0-observation point (may be re-claimed).  match[f]: -1 untouched,
// >= 0 query index, -2 cleared by the rotation check.
// Optional tail of resolve_kernel for the resident tracking chain: the matched features become PoseOptimization edges in
// keypoint order (what Optimizer::PoseOptimization's loop over pFrame->mvpMapPoints produces, src/Optimizer.cc:857-990).
// Doing it here saves a launch per frame and reads the match table while it is still in shared memory.
struct ChainEdgesDev {
    const rgbl_keypoint* kps; const float* uright; const float* last_xw;
    float* exw; float* eobs; float* einfo; uint8_t* est; int* eidx; int* n_edges;      // n_edges == nullptr: disabled
};
// TrackLocalMap form of that tail (local search of the chain): the edge list of the SECOND PoseOptimization = (inliers of the first search)
// + (local matches) in keypoint order (src/Optimizer.cc:857-990); the edges take local points from the query copy tlm_prepare made (lq_xw).
// It also advances the ring's frame counter (the points of the last frame were copied into the ring by the collect kernel, RingHandOverDev).
struct ChainTlmDev {
    const int* match_last;           // nullptr: disabled.  Feature -> point of the last frame (outliers of the first optimisation cleared)
    const float* lq_xw;              // world coordinates of the compacted local queries
    int* ring_count;                 // frames inserted into the local map ring so far
    int* n_local_matches;
};

// One CTA per lane (blockIdx.y); the lane's arguments are read once into registers (Laned, rgbl_kernels.h).
template <bool kLanes>
__global__ void __launch_bounds__(1024) resolve_kernel(int mode, int n_q, Laned<const int*> n_q_dev_l, Laned<FrameDev> f_l,
                                                       Laned<ListOut> lo_l,
                                                       Laned<const uint8_t*> obs_pos_l,
                                                       Laned<const float*> q_angle_l, float nn_ratio,
                                                       int check_orientation, int th_accept,
                                                       Laned<const float*> f_angle_l, Laned<uint8_t*> state_l,
                                                       Laned<int*> minq_l, Laned<int*> choice_l,
                                                       Laned<uint8_t*> resolved_l, Laned<int*> match_l,
                                                       Laned<int*> n_matches_l, Laned<int*> rounds_out_l, int dyn_bytes,
                                                       Laned<ChainEdgesDev> ce_l, Laned<ChainTlmDev> tl_l) {
    pdl_wait(); pdl_trigger();
    const unsigned ln_ = blockIdx.y;
    const int* __restrict__ n_q_dev = lane_arg<kLanes>(n_q_dev_l, ln_);
    const FrameDev& f = lane_arg<kLanes>(f_l, ln_);
    const ListOut& lo = lane_arg<kLanes>(lo_l, ln_);
    const uint8_t* __restrict__ obs_pos = lane_arg<kLanes>(obs_pos_l, ln_);
    const float* __restrict__ q_angle = lane_arg<kLanes>(q_angle_l, ln_);
    const float* __restrict__ f_angle = lane_arg<kLanes>(f_angle_l, ln_);
    uint8_t* __restrict__ state = lane_arg<kLanes>(state_l, ln_);
    int* __restrict__ minq = lane_arg<kLanes>(minq_l, ln_);
    int* __restrict__ choice = lane_arg<kLanes>(choice_l, ln_);
    uint8_t* __restrict__ resolved = lane_arg<kLanes>(resolved_l, ln_);
    int* __restrict__ match = lane_arg<kLanes>(match_l, ln_);
    int* __restrict__ n_matches = lane_arg<kLanes>(n_matches_l, ln_);
    int* __restrict__ rounds_out = lane_arg<kLanes>(rounds_out_l, ln_);
    const ChainEdgesDev& ce = lane_arg<kLanes>(ce_l, ln_);
    const ChainTlmDev& tl = lane_arg<kLanes>(tl_l, ln_);
    const MatchEntry* __restrict__ lists = lo.lists;
    const int list_cap = lo.list_cap;
    const int* __restrict__ list_n = lo.list_n;
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ int hist[kHistoLength];
    __shared__ int keep_bin[3];
    __shared__ int s_nm;
    __shared__ int s_wsum[32];
    __shared__ int s_total;
    __shared__ int s_cnt[2];
#ifdef RESOLVE_DEBUG
#endif
    const int tid = threadIdx.x;
#ifdef RESOLVE_DEBUG
    long long tq[12]; for (int i_ = 0; i_ < 12; ++i_) tq[i_] = 0; tq[0] = clock64(); int dbg_block_rounds = 0;
#define RQ(i) tq[i] = clock64()
#else
#define RQ(i)
#endif
    if (n_q_dev) n_q = *n_q_dev;
    const int n_f = *f.n;
    if (tid == 0) s_nm = 0;

    // ---- working set into shared memory: the rounds below are a chain of barriers around short dependent loads, so their
    // cost is the latency of those loads; with the candidate entries (key, feature, octave), the feature states and the
    // lowest-lister table on chip a round costs a few hundred cycles instead of several L2 round trips.  Falls back to the global-memory
    // rounds when the problem does not fit.
    const int E = *lo.total;              // entries of all queries (appended to one dense run by the collect kernel); cleared below for the next launch
    RQ(1);
    const size_t need = (size_t)12 * (n_f + 1) + (size_t)4 * (n_q + 1) + (size_t)12 * (E + 4) + (size_t)12 * n_q + (size_t)n_f + (size_t)2 * n_q + (size_t)4 * n_q + 64;
    const bool on_chip = need <= (size_t)dyn_bytes;
    const bool orient = mode != 1 && check_orientation;
    int rounds = 0, nm_local = 0;          // nm_local: accepted minus rotation-rejected matches of this thread
    int* ch = choice;                      // chosen feature per query (shared memory on the on-chip path)
    uint8_t* bins = resolved;              // rotation bin per query (the global flags array is free after the rounds)
    int* mt = match;                       // match table (shared memory on the on-chip path, written out at the end)
    if (on_chip) {
        unsigned long long* s_ent = reinterpret_cast<unsigned long long*>(dyn);
        int* s_ioff = reinterpret_cast<int*>(s_ent + E + 4);   // inverse index: the queries that list feature ft are s_iq[s_ioff[ft] .. s_ioff[ft + 1])
        int* s_icur = s_ioff + n_f + 1;                  // per feature: entry count (from the collect kernel), later the lowest waiting lister
        int* s_iq = s_icur + n_f;
        int* s_match = s_iq + E + 4;
        int* s_off = s_match + n_f;                      // query q's entries are s_ent[s_off[q] .. s_end[q])
        int* s_end = s_off + n_q + 1;
        int* s_choice = s_end + n_q;
        int* s_list = s_choice + n_q;                    // two compact lists of waiting queries
        uint8_t* s_state = reinterpret_cast<uint8_t*>(s_list + 2 * (size_t)n_q);
        uint8_t* s_res = s_state + n_f;    // bit 0: resolved, bit 1: the query's point has observations, bit 2: list not sorted by key
        uint8_t* s_bin = s_res + n_q;
        ch = s_choice; bins = s_bin; mt = s_match;
        // The set-up below is a handful of phases separated by barriers; what it reads from global memory does not depend on any of them, so
        // every load is ISSUED here, before the first barrier (the first 4 k entries of the dense run stay in registers until the inverse
        // offsets exist): the whole set-up then pays two rounds of global latency (the total, everything else) instead of one per phase.
        MatchEntry pe_[4]; int ps_[4], pq_[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int en = tid + u * 1024;
            pe_[u] = (en < E) ? lo.dense[en] : 0ull; ps_[u] = (en < E) ? (int)lo.dense_slot[en] : 0; pq_[u] = (en < E) ? lo.dense_q[en] : 0;
        }
        for (int i = tid; i < n_f; i += 1024) { s_state[i] = state[i]; s_match[i] = -1; s_icur[i] = lo.inv_cnt[i]; lo.inv_cnt[i] = 0; }      // the counts are clean for the next launch
        if (tid < 4) s_ent[E + tid] = 0xffffffff00000000ull;     // padding: worst key, feature 0
        for (int q = tid; q < n_q; q += 1024) {
            const int ln = list_n[q], cnt = ln & kListCountMask, b0 = lo.base[q];          // (base of an empty list is never used)
            s_off[q] = b0; s_end[q] = b0 + cnt;
            s_res[q] = (uint8_t)((cnt == 0 ? 1 : 0) | (obs_pos[q] ? 2 : 0) | ((ln & kListUnsorted) ? 4 : 0));
            s_choice[q] = -1;
        }
        __syncthreads();                                     // everybody has read the entry total
        if (tid == 0) *lo.total = 0;
        // ---- inverse index feature -> queries (who lists this feature), built WITHOUT shared-memory atomics: the collect kernels counted
        // the entries per feature with global atomics (many CTAs, negligible there) and gave every entry its slot; here a scan of the
        // counts and one pass over the entries.  (Shared atomics on scattered addresses retire at 2 cycles per lane: the first formulation's
        // per-round atomicMin proposals cost ~2 E cycles per round, an index built with them ~4 E.)
        {
            const int perf = (n_f + 1023) >> 10;
            const int fb_ = min(n_f, tid * perf), fe_ = min(n_f, fb_ + perf);
            int mine_f = 0;
            for (int i = fb_; i < fe_; ++i) mine_f += s_icur[i];
            int incl_f = mine_f;
            const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl_f, o); if (lane >= o) incl_f += t; }
            __syncthreads();                                 // s_wsum is still read by the offsets scan above
            if (lane == 31) s_wsum[warp] = incl_f;
            __syncthreads();
            if (warp == 0) {
                int v = s_wsum[lane], w = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
                s_wsum[lane] = w - v;
            }
            __syncthreads();
            int o = incl_f - mine_f + s_wsum[warp];
            for (int i = fb_; i < fe_; ++i) { s_ioff[i] = o; o += s_icur[i]; s_icur[i] = -1; }      // the count is consumed: the slot becomes the 'lowest waiting lister' cache (-1 = unknown)
            if (tid == 1023) s_ioff[n_f] = o;
            __syncthreads();
        }
        // one thread per ENTRY of the dense run: entry, slot and owning query are three coalesced loads
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int en = tid + u * 1024;
            if (en < E) { s_ent[en] = pe_[u]; s_iq[s_ioff[ent_ft(pe_[u])] + ps_[u]] = pq_[u]; }
        }
        for (int en = tid + 4096; en < E; en += 1024) {
            const MatchEntry e = lo.dense[en];
            s_ent[en] = e;
            s_iq[s_ioff[ent_ft(e)] + lo.dense_slot[en]] = lo.dense_q[en];
        }
        __syncthreads();
        RQ(2);
        RQ(5);
        // ---- rounds.  Phase A (thread per FEATURE): the lowest-index query that still waits among those listing the feature - what the
        // atomicMin proposals of the first formulation computed, now a read-only walk over the feature's (short) inverse list.
        // Phase B (thread per waiting QUERY): its best and second-best AVAILABLE candidates; the set of available candidates can only shrink
        // until the query's turn, so if it is the lowest waiting lister of those two they are still its best two then and the decision
        // is final (tests/test_resolution_model.py checks this rule against the sequential loops).  With the list sorted by key the scan
        // stops at the second available entry; lists of more than 32 candidates (left in scan order) are read to the end.
        int* s_minq = s_icur;                    // the counts are dead after the index is built
        // lowest-index query that still waits among the listers of ft (0x7fffffff: none).  The waiting set only shrinks, so a cached lister
        // that still waits is still the lowest: the inverse list is walked again only when the cached one has become final (kDead: nobody
        // waits for this feature any more, or it is taken for good).  Call only where nobody writes s_res concurrently.
        constexpr int kDead = -2;
        auto lowest_waiting = [&](int ft) -> int {
            const int c = s_minq[ft];
            if (c == kDead) return 0x7fffffff;
            if (c >= 0 && !(s_res[c] & 1)) return c;
            int m = 0x7fffffff;
            const int e = s_ioff[ft + 1];
            for (int k = s_ioff[ft]; k < e; ++k) { const int o = s_iq[k]; if (!(s_res[o] & 1)) m = min(m, o); }
            s_minq[ft] = (m == 0x7fffffff) ? kDead : m;
            return m;
        };
        struct Pick { uint32_t best, best2; int lvl, lvl2, fb, fb2, bb; };
        auto pick = [&](int q) -> Pick {         // reads only
            Pick P{0xffffffffu, 0xffffffffu, -1, -1, -1, -1, 0};
            const int k0 = s_off[q], e = s_end[q];
            if (!(s_res[q] & 4)) {
                // The first four entries at once, branch-free: the two best available candidates are almost always among them, and a
                // data-dependent loop here makes the 32 lanes of a warp take 32 different paths (measured: ~4 k cycles per round for ANY
                // number of waiting queries).  The loop below only continues where four entries were not enough.
                MatchEntry en[4]; uint8_t st[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) en[u] = s_ent[k0 + u];                       // s_ent is padded: reading past a short list is harmless
#pragma unroll
                for (int u = 0; u < 4; ++u) st[u] = (k0 + u < e) ? s_state[ent_ft(en[u])] : (uint8_t)1;
                int found = 0, first = e;                // first: position of the first available entry
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const bool av = st[u] != 1;
                    if (av && found == 0) { P.best = ent_key(en[u]); P.fb = ent_ft(en[u]); P.bb = ent_bin(en[u]); P.lvl = ent_oc(en[u]); first = k0 + u; }
                    if (av && found == 1) { P.best2 = ent_key(en[u]); P.fb2 = ent_ft(en[u]); P.lvl2 = ent_oc(en[u]); }
                    found += av ? 1 : 0;
                }
                const int want = (mode == 0) ? 1 : 2;
                for (int k = k0 + 4; found < want && k < e; ++k) {
                    const MatchEntry x = s_ent[k];
                    const int ft = ent_ft(x);
                    if (s_state[ft] == 1) continue;
                    if (found == 0) { P.best = ent_key(x); P.fb = ft; P.bb = ent_bin(x); P.lvl = ent_oc(x); first = k; }
                    else { P.best2 = ent_key(x); P.fb2 = ft; P.lvl2 = ent_oc(x); }
                    ++found;
                }
                // a taken feature stays taken: the entries before the first available one never matter again (the queries that wait
                // longest are the contested ones, whose best candidates went to lower indices - without this they re-walk them every round)
                if (first > k0) s_off[q] = first;
                if (mode == 0) { P.best2 = 0xffffffffu; P.fb2 = -1; P.lvl2 = -1; }
            } else {
                for (int k = k0; k < e; ++k) {
                    const MatchEntry en = s_ent[k];
                    const int ft = ent_ft(en);
                    if (s_state[ft] == 1) continue;
                    const uint32_t key = ent_key(en);
                    const int oc = ent_oc(en);
                    if (key < P.best) { P.best2 = P.best; P.lvl2 = P.lvl; P.fb2 = P.fb; P.best = key; P.lvl = oc; P.fb = ft; P.bb = ent_bin(en); }
                    else if (key < P.best2) { P.best2 = key; P.lvl2 = oc; P.fb2 = ft; }
                }
                if (mode == 0) { P.best2 = 0xffffffffu; P.fb2 = -1; }
            }
            return P;
        };
        auto commit = [&](int q, const Pick& P) {    // the query is final: accept / reject tests and the state update
            const uint8_t flags = s_res[q];
            s_res[q] = flags | 1;
            if (P.fb < 0) return;
            const int bd = (int)(P.best >> 20);
            bool accept = bd <= th_accept;
            if (mode == 1 && accept) {
                const int bd2 = (P.best2 == 0xffffffffu) ? 256 : (int)(P.best2 >> 20);
                if (P.lvl == P.lvl2 && (float)bd > __fmul_rn(nn_ratio, (float)bd2)) accept = false;
            }
            if (mode == 2 && accept) {            // SearchByBoW: bestDist1 < mfNNratio * bestDist2 (src/ORBmatcher.cc:324)
                const int bd2 = (P.best2 == 0xffffffffu) ? 256 : (int)(P.best2 >> 20);
                accept = (float)bd < __fmul_rn(nn_ratio, (float)bd2);
            }
            if (accept) {
                s_choice[q] = P.fb; s_bin[q] = (uint8_t)P.bb;
                atomicMax(&s_match[P.fb], q);            // owner of a feature = the last (highest-index) query that chose it
                // In a block round this write races with the state reads of other queries deciding in the same phase (compute-sanitizer
                // racecheck reports it); it is benign: only 0/2 -> 1 matters to a reader, and a query q' that reads state[fb] has fb in
                // its list, and the winner q < q' was the lowest waiting lister of fb when the round began.  If q' sees the old value it
                // waits one more round (s_minq[fb] = q != q') and then sees 1; if it sees the new value it skips fb now, exactly what
                // the sequential scan does after q took fb.  Either way q' ends with the same feature.
                if (flags & 2) s_state[P.fb] = 1; else if (s_state[P.fb] == 0) s_state[P.fb] = 2;
                ++nm_local;
            }
        };

        // Block rounds over a COMPACT list of the waiting queries: a warp pays for its slowest lane, so with the waiting queries scattered
        // over all 32 warps every warp would run the full decision in every round; packed, round r touches ceil(waiting / 32) warps.
        int cur = 0, n_act;
        {
            if (tid == 0) { s_cnt[0] = 0; s_cnt[1] = 0; }
            __syncthreads();
            for (int q0 = 0; q0 < n_q; q0 += 1024) {
                const int q = q0 + tid;
                const bool w = q < n_q && !(s_res[q] & 1);
                const unsigned m = __ballot_sync(0xffffffffu, w);
                int base = 0;
                if ((tid & 31) == 0 && m) base = atomicAdd(&s_cnt[0], __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (w) s_list[base + __popc(m & ((1u << (tid & 31)) - 1u))] = q;
            }
            __syncthreads();
            n_act = s_cnt[0];
        }
#ifdef RESOLVE_DEBUG
        long long tr_[24]; int na_[8]; int nr_ = 0;
#endif
        while (n_act > 32) {
#ifdef RESOLVE_DEBUG
            if (nr_ < 8) { tr_[3 * nr_] = clock64(); na_[nr_] = n_act; }
#endif
            const int* lst = s_list + (size_t)cur * n_q;
            int* lst_next = s_list + (size_t)(cur ^ 1) * n_q;
            if (tid == 0) s_cnt[cur ^ 1] = 0;
            for (int ft = tid; ft < n_f; ft += 1024) {           // phase A
                if (s_minq[ft] == kDead) continue;
                if (s_state[ft] == 1) s_minq[ft] = kDead; else (void)lowest_waiting(ft);
            }
            __syncthreads();
#ifdef RESOLVE_DEBUG
            if (nr_ < 8) tr_[3 * nr_ + 1] = clock64();
#endif
            for (int i0 = 0; i0 < n_act; i0 += 1024) {           // phase B
                const int i = i0 + tid;
                const int q = i < n_act ? lst[i] : -1;
                bool w = false;
                if (q >= 0) {
                    const Pick P = pick(q);
                    w = P.fb >= 0 && (s_minq[P.fb] != q || (P.fb2 >= 0 && s_minq[P.fb2] != q));
                    if (!w) commit(q, P);
                }
                const unsigned m = __ballot_sync(0xffffffffu, w);
                int base = 0;
                if ((tid & 31) == 0 && m) base = atomicAdd(&s_cnt[cur ^ 1], __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (w) lst_next[base + __popc(m & ((1u << (tid & 31)) - 1u))] = q;
            }
            ++rounds;
            cur ^= 1;
            __syncthreads();
#ifdef RESOLVE_DEBUG
            if (nr_ < 8) { tr_[3 * nr_ + 2] = clock64(); ++nr_; }
#endif
            n_act = s_cnt[cur];
        }
#ifdef RESOLVE_DEBUG
        if (tid == 0) for (int r_ = 0; r_ < nr_; ++r_) printf("  block round %d: waiting %d  phase A %lld  phase B %lld\n", r_, na_[r_], tr_[3 * r_ + 1] - tr_[3 * r_], tr_[3 * r_ + 2] - tr_[3 * r_ + 1]);
#endif
        RQ(6);
#ifdef RESOLVE_DEBUG
        dbg_block_rounds = rounds;
#endif
        // <= 32 waiting queries: warp 0 finishes alone.  A lane checks its (at most two) features' inverse lists itself; checks and commits
        // of a round are separated by warp syncs, so every check sees the state the round began with.
        if (n_act > 0 && tid < 32) {
            int q = tid < n_act ? s_list[(size_t)cur * n_q + tid] : -1;
            for (;;) {
                bool waiting = false;
                Pick P{};
                if (q >= 0) {
                    P = pick(q);
                    waiting = (P.fb >= 0 && lowest_waiting(P.fb) < q) || (P.fb2 >= 0 && lowest_waiting(P.fb2) < q);
                }
                __syncwarp();
                if (q >= 0 && !waiting) { commit(q, P); q = -1; }
                ++rounds;
                __syncwarp();
                if (!__any_sync(0xffffffffu, waiting)) break;
            }
        }
        __syncthreads();
        RQ(3);
        for (int i = tid; i < n_f; i += 1024) state[i] = s_state[i];
        __syncthreads();
    } else {
    __syncthreads();
    if (tid == 0) *lo.total = 0;
    for (int i = tid; i < n_f; i += 1024) { match[i] = -1; lo.inv_cnt[i] = 0; }
    for (int q = tid; q < n_q; q += 1024) { choice[q] = -1; resolved[q] = ((list_n[q] & kListCountMask) == 0); }
    __syncthreads();
    for (;;) {
        bool any_unresolved = false;
        for (int i = tid; i < n_f; i += 1024) minq[i] = 0x7fffffff;
        __syncthreads();
        for (int q = tid; q < n_q; q += 1024) {
            if (resolved[q]) continue;
            const MatchEntry* l = lists + (size_t)q * list_cap;
            const int n = list_n[q] & kListCountMask;
            for (int k = 0; k < n; ++k) {
                const int ft = ent_ft(l[k]);
                if (state[ft] != 1) atomicMin(&minq[ft], q);
            }
        }
        __syncthreads();
        for (int q = tid; q < n_q; q += 1024) {
            if (resolved[q]) continue;
            const MatchEntry* l = lists + (size_t)q * list_cap;
            const int n = list_n[q] & kListCountMask;
            uint32_t best = 0xffffffffu, best2 = 0xffffffffu;     // smallest / second smallest (dist, order) keys
            int lvl = -1, lvl2 = -1, fb = -1;
            bool depends_ok = true;
            for (int k = 0; k < n; ++k) {
                const uint32_t key = ent_key(l[k]);
                const int ft = ent_ft(l[k]);
                if (state[ft] == 1) continue;
                if (mode >= 1 && minq[ft] != q) depends_ok = false;
                if (mode == 0) {
                    if (key < best) { best = key; fb = ft; }
                } else {
                    // reference scan order = ascending csr position; emulate "dist < bestDist" / "else if dist < bestDist2"
                    // order-independently: best = min by (dist, pos); second = min dist among the rest (level of the
                    // FIRST candidate in scan order reaching that distance)
                    const int oc = ent_oc(l[k]);
                    if (key < best) { best2 = best; lvl2 = lvl; best = key; lvl = oc; fb = ft; }
                    else if (key < best2) { best2 = key; lvl2 = oc; }
                }
            }
            if (best == 0xffffffffu) { resolved[q] = 1; continue; }
            const bool final_ok = (mode == 0) ? (minq[fb] == q) : depends_ok;
            if (!final_ok) { any_unresolved = true; continue; }
            resolved[q] = 1;
            const int bd = (int)(best >> 20);
            bool accept = bd <= th_accept;
            if (mode == 1 && accept) {
                const int bd2 = (best2 == 0xffffffffu) ? 256 : (int)(best2 >> 20);
                if (lvl == lvl2 && (float)bd > __fmul_rn(nn_ratio, (float)bd2)) accept = false;
            }
            if (mode == 2 && accept) {            // SearchByBoW: bestDist1 < mfNNratio * bestDist2 (src/ORBmatcher.cc:324)
                const int bd2 = (best2 == 0xffffffffu) ? 256 : (int)(best2 >> 20);
                accept = (float)bd < __fmul_rn(nn_ratio, (float)bd2);
            }
            if (accept) {
                choice[q] = fb;
                if (obs_pos[q]) state[fb] = 1; else if (state[fb] == 0) state[fb] = 2;
                ++nm_local;
            }
        }
        ++rounds;
        if (!__syncthreads_or(any_unresolved)) break;
    }
    }
    // owner of a feature = the last (highest-index) query that chose it (the on-chip rounds record it when a query commits)
    if (!on_chip) for (int q = tid; q < n_q; q += 1024) if (ch[q] >= 0) atomicMax(&mt[ch[q]], q);
    if (orient) {
        for (int b = tid; b < kHistoLength; b += 1024) hist[b] = 0;
        __syncthreads();
        const float factor = 1.0f / kHistoLength;
        for (int q0 = 0; q0 < n_q; q0 += 1024) {          // uniform trip count: the warp-level vote below needs all lanes
            const int q = q0 + tid;
            const int c = q < n_q ? ch[q] : -1;
            const bool valid = c >= 0;
            int bin = 63;                                   // lanes without a match share one key (MATCH.ANY iterates over the distinct values of a warp)
            if (valid) {
                if (on_chip) {
                    bin = bins[q];                          // computed with the candidate entry
                } else {
                    float rot = __fsub_rn(q_angle[q], f_angle ? f_angle[c] : f.keys[c].angle);
                    if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
                    bin = (int)roundf(__fmul_rn(rot, factor));
                    if (bin == kHistoLength) bin = 0;
                    bins[q] = (uint8_t)bin;
                }
            }
            // nearly every match falls into one or two bins: aggregate equal bins inside the warp, one atomic per group
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (valid && (tid & 31) == __ffs(peers) - 1) atomicAdd(&hist[bin], __popc(peers));
        }
        __syncthreads();
        if (tid < 32) {
            // ORBmatcher::ComputeThreeMaxima (src/ORBmatcher.cc:2012-2053).  The reference scans the bins in index order with
            // strict '>' updates of (max1, max2, max3): the result is the three largest NON-EMPTY bins ordered by (count
            // descending, index ascending).  Done here as three warp arg-max reductions over count << 8 | (255 - index)
            // instead of a 30-step serial scan (the scan alone was ~4k cycles of one thread).
            const int cnt = tid < kHistoLength ? hist[tid] : 0;
            int key = cnt > 0 ? ((cnt << 8) | (255 - tid)) : 0;
            int top_i[3], top_c[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                int m = key;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
                top_c[r] = m >> 8; top_i[r] = m > 0 ? 255 - (m & 0xff) : -1;
                if (key == m) key = 0;                      // keys are unique (index in the low byte) unless 0
            }
            int i1 = top_i[0], i2 = top_i[1], i3 = top_i[2];
            if ((float)top_c[1] < __fmul_rn(0.1f, (float)top_c[0])) { i2 = -1; i3 = -1; }
            else if ((float)top_c[2] < __fmul_rn(0.1f, (float)top_c[0])) i3 = -1;
            if (tid == 0) { keep_bin[0] = i1; keep_bin[1] = i2; keep_bin[2] = i3; }
        }
        __syncthreads();
        for (int q = tid; q < n_q; q += 1024) {
            const int c = ch[q];
            if (c < 0) continue;
            const int bin = bins[q];
            if (bin != keep_bin[0] && bin != keep_bin[1] && bin != keep_bin[2]) { mt[c] = -2; --nm_local; }
        }
    }
    RQ(7);
    if (on_chip) {
        __syncthreads();
        for (int i = tid; i < n_f; i += 1024) match[i] = mt[i];
    }
    RQ(8);
    if (ce.n_edges) {                     // ordered compaction of the matched features into edges
        // Two chunks of 1024 features per trip (a KITTI frame is one trip): everything an edge needs is loaded for both chunks before the
        // positions are known, so the trip pays ONE round of global latency (two in the TrackLocalMap form, whose first-search matches
        // live in global memory); the positions come from warp ballots and a 64-entry scan.
        __shared__ int s_wcnt[2][32];
        __shared__ int s_nloc;
        const bool tlm = tl.match_last != nullptr;
        if (tid == 0) s_nloc = 0;
        __syncthreads();
        const int lane = tid & 31, warp = tid >> 5;
        if (tlm && tid == 0) *tl.ring_count = *tl.ring_count + 1;      // the points of the last frame were handed over by the collect kernel
        RQ(9);
        int run = 0, nloc = 0;            // edges before this trip (same value in every thread); local matches of this thread
        for (int b = 0; b < n_f; b += 2048) {
            int m[2]; float kx[2], ky[2], ur[2], xw[2][3]; int oc[2]; unsigned bal[2]; const float* src[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int i = b + c * 1024 + tid;
                m[c] = -1; src[c] = ce.last_xw;
                if (i < n_f) {
                    if (tlm) {
                        const int ma = tl.match_last[i];
                        const int mb = ma < 0 ? mt[i] : -1;
                        if (mb >= 0) ++nloc;
                        m[c] = ma >= 0 ? ma : mb;
                        if (ma < 0) src[c] = tl.lq_xw;
                    } else {
                        m[c] = mt[i];
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int i = b + c * 1024 + tid;
                kx[c] = ky[c] = ur[c] = xw[c][0] = xw[c][1] = xw[c][2] = 0.f; oc[c] = 0;
                if (m[c] >= 0) {
                    kx[c] = ce.kps[i].x; ky[c] = ce.kps[i].y; oc[c] = ce.kps[i].octave; ur[c] = ce.uright[i];
                    xw[c][0] = src[c][3 * m[c]]; xw[c][1] = src[c][3 * m[c] + 1]; xw[c][2] = src[c][3 * m[c] + 2];
                }
            }
#pragma unroll
            for (int c = 0; c < 2; ++c) { bal[c] = __ballot_sync(0xffffffffu, m[c] >= 0); if (lane == 0) s_wcnt[c][warp] = __popc(bal[c]); }
            __syncthreads();
            if (warp == 0) {              // exclusive scan of the 64 warp counts in chunk-major order
                const int v0 = s_wcnt[0][lane], v1 = s_wcnt[1][lane];
                int i0 = v0, i1 = v1;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t0 = __shfl_up_sync(0xffffffffu, i0, o), t1 = __shfl_up_sync(0xffffffffu, i1, o);
                    if (lane >= o) { i0 += t0; i1 += t1; }
                }
                const int tot0 = __shfl_sync(0xffffffffu, i0, 31), tot1 = __shfl_sync(0xffffffffu, i1, 31);
                s_wcnt[0][lane] = i0 - v0; s_wcnt[1][lane] = tot0 + i1 - v1;
                if (lane == 0) s_total = tot0 + tot1;
            }
            __syncthreads();
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                if (m[c] < 0) continue;
                const int i = b + c * 1024 + tid;
                const int e = run + s_wcnt[c][warp] + __popc(bal[c] & ((1u << lane) - 1u));
                ce.exw[3 * e] = xw[c][0]; ce.exw[3 * e + 1] = xw[c][1]; ce.exw[3 * e + 2] = xw[c][2];
                ce.eobs[3 * e] = kx[c]; ce.eobs[3 * e + 1] = ky[c]; ce.eobs[3 * e + 2] = ur[c];
                const float sc = f.scale[oc[c]];
                ce.einfo[e] = __fdiv_rn(1.0f, __fmul_rn(sc, sc));            // mvInvLevelSigma2 (src/ORBextractor.cc:421-429)
                ce.est[e] = ur[c] >= 0.f;
                ce.eidx[e] = i;
            }
            run += s_total;
            __syncthreads();              // s_wcnt / s_total are rewritten by the next trip
        }
        if (tlm) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) nloc += __shfl_down_sync(0xffffffffu, nloc, o);
            if (lane == 0 && nloc) atomicAdd(&s_nloc, nloc);
            __syncthreads();
        }
        if (tid == 0) { *ce.n_edges = run; if (tlm) *tl.n_local_matches = s_nloc; }
    }
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) nm_local += __shfl_down_sync(0xffffffffu, nm_local, o);
        if ((tid & 31) == 0 && nm_local != 0) atomicAdd(&s_nm, nm_local);
    }
    __syncthreads();
    if (tid == 0) { *n_matches = s_nm; if (rounds_out) *rounds_out = rounds; }
#ifdef RESOLVE_DEBUG
    if (tid == 0) printf("resolve mode=%d n_q=%d n_f=%d E=%d on_chip=%d rounds=%d (block %d) nm=%d | scan=%lld fill=%lld index=%lld rounds=%lld (block %lld tail %lld) epilogue=%lld (owner+orient %lld, match out %lld, hand-over %lld, edges+rest %lld)\n", mode, n_q, n_f, E, (int)on_chip, rounds, dbg_block_rounds, s_nm,
                         tq[1] - tq[0], tq[2] - tq[1], tq[5] - tq[2], tq[3] - tq[5], tq[6] - tq[5], tq[3] - tq[6], clock64() - tq[3], tq[7] - tq[3], tq[8] - tq[7], tq[9] ? tq[9] - tq[8] : 0, clock64() - (tq[9] ? tq[9] : tq[8]));

#endif
}

// ---- ORBmatcher::Fuse, the search part (src/ORBmatcher.cc:1176-1303): one warp per map point --------------------------
struct FusePointsDev { int n; const uint8_t* valid; const float* xw; const float* normal; const float* mf_min; const float* mf_max; const uint8_t* desc; };

__global__ void __launch_bounds__(256) fuse_search_kernel(FrameDev f, const int* __restrict__ cell_start, const int* __restrict__ csr_idx,
                                                          FusePointsDev mp, const float* __restrict__ Tcw, const float* __restrict__ Ow, float th,
                                                          int* __restrict__ best_idx, int* __restrict__ best_dist) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= mp.n) return;
    unsigned best = 0xffffffffu;
    if (mp.valid[q]) {
        const float P[3] = {mp.xw[3 * q], mp.xw[3 * q + 1], mp.xw[3 * q + 2]};
        float Pc[3];
        se3f_rotate(Tcw, P, Pc);
        Pc[0] = __fadd_rn(Pc[0], Tcw[4]); Pc[1] = __fadd_rn(Pc[1], Tcw[5]); Pc[2] = __fadd_rn(Pc[2], Tcw[6]);
        bool ok = !(Pc[2] < 0.0f);
        const float invz = __fdiv_rn(1.0f, Pc[2]);
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(f.fx, Pc[0]), Pc[2]), f.cx);
        const float v = __fadd_rn(__fdiv_rn(__fmul_rn(f.fy, Pc[1]), Pc[2]), f.cy);
        ok = ok && (u >= f.min_x && u < f.max_x && v >= f.min_y && v < f.max_y);                     // KeyFrame::IsInImage
        const float ur = __fsub_rn(u, __fmul_rn(f.bf, invz));
        const float PO[3] = {__fsub_rn(P[0], Ow[0]), __fsub_rn(P[1], Ow[1]), __fsub_rn(P[2], Ow[2])};
        const float dist3D = sqrtf(eig_sum3(__fmul_rn(PO[0], PO[0]), __fmul_rn(PO[1], PO[1]), __fmul_rn(PO[2], PO[2])));
        const float mf_max = mp.mf_max[q];
        ok = ok && !(dist3D < __fmul_rn(0.8f, mp.mf_min[q]) || dist3D > __fmul_rn(1.2f, mf_max));
        const float* Pn = mp.normal + 3 * q;
        const float dotn = eig_sum3(__fmul_rn(PO[0], Pn[0]), __fmul_rn(PO[1], Pn[1]), __fmul_rn(PO[2], Pn[2]));
        ok = ok && !((double)dotn < 0.5 * (double)dist3D);
        if (ok) {
            const float ratio = __fdiv_rn(mf_max, dist3D);
            const float lg = (float)log((double)ratio);          // correctly-rounded stand-in for glibc logf (as in frustum_kernel)
            int level = (int)ceilf(__fdiv_rn(lg, f.log_scale_factor));
            if (level < 0) level = 0; else if (level >= f.n_levels) level = f.n_levels - 1;
            const float radius = __fmul_rn(th, f.scale[level]);
            const CellRange cr = cell_range(f, u, v, radius);
            if (cr.ok) {
                const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(mp.desc + (size_t)q * 32));
                const uint4 d1 = __ldg(reinterpret_cast<const uint4*>(mp.desc + (size_t)q * 32) + 1);
                for (int ix = cr.min_cx; ix <= cr.max_cx; ++ix) {
                    const int b = cell_start[ix * kGridRows + cr.min_cy], e = cell_start[ix * kGridRows + cr.max_cy + 1];
                    for (int p = b + lane; p < e; p += 32) {
                        const int idx = csr_idx[p];
                        const rgbl_keypoint kp = f.keys[idx];
                        if (!(fabsf(__fsub_rn(kp.x, u)) < radius && fabsf(__fsub_rn(kp.y, v)) < radius)) continue;     // GetFeaturesInArea
                        if (kp.octave < level - 1 || kp.octave > level) continue;
                        const float sc = f.scale[kp.octave];
                        const float inv_sigma2 = __fdiv_rn(1.0f, __fmul_rn(sc, sc));                                   // mvInvLevelSigma2
                        const float ex = __fsub_rn(u, kp.x), ey = __fsub_rn(v, kp.y);
                        const float urt = f.uright[idx];
                        if (urt >= 0.f) {
                            const float er = __fsub_rn(ur, urt);
                            const float e2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er));
                            if ((double)__fmul_rn(e2, inv_sigma2) > 7.8) continue;
                        } else {
                            const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                            if ((double)__fmul_rn(e2, inv_sigma2) > 5.99) continue;
                        }
                        const int d = hamming256(d0, d1, f.desc + (size_t)idx * 32);
                        best = min(best, ((unsigned)d << 20) | (unsigned)p);         // strict '<' in scan order = min of (dist, position)
                    }
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) {
        best_idx[q] = best == 0xffffffffu ? -1 : csr_idx[best & kPosMask];
        best_dist[q] = best == 0xffffffffu ? 256 : (int)(best >> 20);
    }
}

// ---- Frame::isInFrustum for a list of local map points ----------------------------------------------
__global__ void __launch_bounds__(256) frustum_kernel(FrameDev f, FrustumParams prm, int n, const float* __restrict__ xw,
                                                      const float* __restrict__ normal, const float* __restrict__ mf_min,
                                                      const float* __restrict__ mf_max, uint8_t* __restrict__ in_view,
                                                      float* __restrict__ px, float* __restrict__ py,
                                                      float* __restrict__ pxr, float* __restrict__ depth,
                                                      int* __restrict__ level, float* __restrict__ view_cos) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float P[3] = {xw[3 * i], xw[3 * i + 1], xw[3 * i + 2]};
    const FrustumOut o = frustum_point(f, prm, P, normal + 3 * i, mf_min[i], mf_max[i]);
    in_view[i] = o.in_view; px[i] = o.px; py[i] = o.py; pxr[i] = o.pxr; depth[i] = o.depth; level[i] = o.level; view_cos[i] = o.view_cos;
}

// ---- SearchByBoW(KF, F): candidates = the F features of the same vocabulary node -----------------------------------
__global__ void __launch_bounds__(256) bow_collect_kernel(int n_q, const int* __restrict__ q_feat, const int* __restrict__ q_cbeg,
                                                          const int* __restrict__ q_cend, const uint8_t* __restrict__ kf_desc,
                                                          const uint8_t* __restrict__ f_desc, const int* __restrict__ f_node_feat,
                                                          const float* __restrict__ q_angle, const float* __restrict__ f_angle, int check_orientation,
                                                          int keep_max, ListOut out) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= n_q) return;
    const uint8_t* dq = kf_desc + (size_t)q_feat[q] * 32;
    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(dq)), d1 = __ldg(reinterpret_cast<const uint4*>(dq) + 1);
    const int b = q_cbeg[q], e = q_cend[q];
    MatchEntry* list = out.lists + (size_t)q * out.list_cap;
    uint16_t* slots = out.slots + (size_t)q * out.list_cap;
    const int list_cap = out.list_cap;
    const float qa = check_orientation ? q_angle[q] : 0.f;
    int count = 0;
    for (int p0 = b; p0 < e; p0 += 32) {
        const int p = p0 + lane;
        bool keep = false;
        MatchEntry key = 0;
        if (p < e) {
            const int ft = f_node_feat[p];
            const int d = hamming256(d0, d1, f_desc + (size_t)ft * 32);
            if (d <= keep_max) {
                keep = true;
                key = ent_make(((uint32_t)d << 20) | (uint32_t)p, check_orientation ? rotation_bin(qa, f_angle[ft]) : 0u, 0u, (unsigned)ft);
            }
        }
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        if (keep) { const int o = count + __popc(m & ((1u << lane) - 1u)); if (o < list_cap) { list[o] = key; slots[o] = (uint16_t)atomicAdd(&out.inv_cnt[ent_ft(key)], 1); } }
        count += __popc(m);
    }
    const int ln = warp_finish_list(out, q, count);
    if (lane == 0) { out.list_n[q] = ln; if (count > out.list_cap) atomicExch(out.overflow, 3); }
}

// ---- SearchByProjection(CurrentFrame, KeyFrame, sAlreadyFound, th, ORBdist): candidate phase -------------------------
__global__ void __launch_bounds__(256) search_reloc_collect_kernel(FrameDev f, const int* __restrict__ cell_start,
                                                                   const int* __restrict__ csr_idx, RelocPointsDev rp,
                                                                   SearchRelocParams prm, ListOut out) {
    const int q = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= rp.n) return;
    int count = 0;
    if (rp.valid[q]) {
        const float p[3] = {rp.xw[3 * q], rp.xw[3 * q + 1], rp.xw[3 * q + 2]};
        float xc[3];
        se3f_rotate(prm.cur_pose, p, xc);
        xc[0] = __fadd_rn(xc[0], prm.cur_pose[4]); xc[1] = __fadd_rn(xc[1], prm.cur_pose[5]); xc[2] = __fadd_rn(xc[2], prm.cur_pose[6]);
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(f.fx, xc[0]), xc[2]), f.cx);
        const float v = __fadd_rn(__fdiv_rn(__fmul_rn(f.fy, xc[1]), xc[2]), f.cy);
        bool ok = !(u < f.min_x || u > f.max_x) && !(v < f.min_y || v > f.max_y);     // note: no positive-depth test in the reference
        if (ok) {
            const float PO[3] = {__fsub_rn(p[0], prm.Ow[0]), __fsub_rn(p[1], prm.Ow[1]), __fsub_rn(p[2], prm.Ow[2])};
            const float dist = sqrtf(eig_sum3(__fmul_rn(PO[0], PO[0]), __fmul_rn(PO[1], PO[1]), __fmul_rn(PO[2], PO[2])));
            if (!(dist < __fmul_rn(0.8f, rp.mf_min[q]) || dist > __fmul_rn(1.2f, rp.mf_max[q]))) {
                const float ratio = __fdiv_rn(rp.mf_max[q], dist);
                const float lg = (float)log((double)ratio);
                int pl = (int)ceilf(__fdiv_rn(lg, f.log_scale_factor));
                if (pl < 0) pl = 0; else if (pl >= f.n_levels) pl = f.n_levels - 1;
                const float radius = __fmul_rn(prm.th, f.scale[pl]);
                const CellRange cr = cell_range(f, u, v, radius);
                if (cr.ok) {
                    const uint4 d0 = __ldg(reinterpret_cast<const uint4*>(rp.desc + (size_t)q * 32));
                    const uint4 d1 = __ldg(reinterpret_cast<const uint4*>(rp.desc + (size_t)q * 32) + 1);
                    count = warp_collect(f, cell_start, csr_idx, cr, u, v, radius, pl - 1, pl + 1, d0, d1, prm.orb_dist,
                                         out, q, [](int) { return true; }, prm.check_orientation != 0, rp.angle[q]);
                }
            }
        }
    }
    const int ln = warp_finish_list(out, q, count);
    if (lane == 0) { out.list_n[q] = ln; if (count > out.list_cap) atomicExch(out.overflow, 3); }
}

// ---- resident tracking chain (TrackWithMotionModel-style glue between the reference functions) ----------------
// Every keypoint of the last frame that has a LiDAR depth acts as a map point: Frame::UnprojectStereo
// (src/Frame.cc:1137-1150) with the last pose, descriptor = the keypoint's own descriptor.
template <bool kLanes>
__global__ void __launch_bounds__(256) chain_prep_kernel(Laned<ChainPrepDev> cp_l, Laned<const float*> last_pose_l) {
    const ChainPrepDev& cp = lane_arg<kLanes>(cp_l, blockIdx.y);
    const float* __restrict__ last_pose = lane_arg<kLanes>(last_pose_l, blockIdx.y);
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i == 0) chain_prep_motion(cp, last_pose);
    float Rwc[9], Ow[3];
    chain_pose_matrices(last_pose, Rwc, Ow);
    if (i < cp.cap) chain_prep_item(cp, Rwc, Ow, i);
}


// ---- launchers ---------------------------------------------------------------------------------------
// dynamic shared memory of resolve_kernel (opt-in above 48 KB, set once per device)
static int resolve_dyn_bytes() {
    constexpr int kBytes = 160 * 1024;
    static bool done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && !done[dev]) {
        cudaFuncSetAttribute(resolve_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBytes);
        cudaFuncSetAttribute(resolve_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBytes);
        done[dev] = true;
    }
    return kBytes;
}

// one-time function attributes of this file's kernels (call before capturing their launches into a CUDA graph)
void prepare_match_kernels() { (void)resolve_dyn_bytes(); }

void launch_grid_build(cudaStream_t st, const FrameDev& f, int* cell_start, int* csr_idx, int* kp_cell) {
    grid_build_kernel<<<1, 1024, 0, st>>>(f, 0, cell_start, csr_idx, kp_cell);
}

void launch_grid_build_batch(cudaStream_t st, const FrameDev& f, int n_frames, int kp_stride, int* cell_start, int* csr_idx, int* kp_cell) {
    if (n_frames <= 0) return;
    grid_build_kernel<<<n_frames, 1024, 0, st>>>(f, kp_stride, cell_start, csr_idx, kp_cell);
}

static ListOut list_out(const MatchScratch& s) {
    return ListOut{s.lists, s.slots, s.list_cap, s.list_n, s.dense, s.dense_slot, s.dense_q, s.base, s.total, s.inv_cnt, s.overflow};
}

void launch_search_last(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const int*>& cell_start, const Laned<const int*>& csr_idx,
                        const Laned<LastFrameDev>& lf, const Laned<SearchLastParams>& prm, const Laned<MatchScratch>& s, const Laned<uint8_t*>& state,
                        const Laned<int*>& match, const Laned<int*>& n_matches, const Laned<ChainEdgesOut>* edges, int lanes) {
    const LastFrameDev lf0 = lf.base;
    if (lf0.n <= 0) return;
    const bool pdl = chain_launch_pdl();
    const Laned<ListOut> lo = laned_of(lanes, [&](int l) { return list_out(lane_value(s, l)); });
    launch_kernel(lanes > 1 ? search_last_collect_kernel<true> : search_last_collect_kernel<false>, dim3((lf0.n + 7) / 8, lanes), dim3(256), 0, st, pdl, f, cell_start, csr_idx, lf, prm, lo);
    const auto ls = [&](int l) { return lane_value(s, l); };
    const Laned<ChainEdgesDev> ce = laned_of(lanes, [&](int l) {
        if (!edges) return ChainEdgesDev{};
        const FrameDev fl = lane_value(f, l); const LastFrameDev ll = lane_value(lf, l); const ChainEdgesOut e = lane_value(*edges, l);
        return ChainEdgesDev{fl.keys, fl.uright, ll.xw, e.exw, e.eobs, e.einfo, e.est, e.eidx, e.n_edges};
    });
    launch_kernel(lanes > 1 ? resolve_kernel<true> : resolve_kernel<false>, dim3(1, lanes), dim3(1024), (size_t)resolve_dyn_bytes(), st, pdl, 0, lf0.n, Laned<const int*>(), f, lo,
                  laned_of(lanes, [&](int l) { return lane_value(lf, l).obs_pos; }), laned_of(lanes, [&](int l) { return lane_value(lf, l).angle; }), 0.f,
                  prm.base.check_orientation, kThHigh, Laned<const float*>(), state, laned_of(lanes, [&](int l) { return ls(l).minq; }),
                  laned_of(lanes, [&](int l) { return ls(l).choice; }), laned_of(lanes, [&](int l) { return ls(l).resolved; }), match, n_matches,
                  laned_of(lanes, [&](int l) { return ls(l).rounds; }), resolve_dyn_bytes(), ce, Laned<ChainTlmDev>());
}

void launch_search_local(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const int*>& cell_start, const Laned<const int*>& csr_idx,
                         const Laned<LocalPointsDev>& lp, const SearchLocalParams& prm, const Laned<MatchScratch>& s, const Laned<uint8_t*>& state,
                         const Laned<int*>& match, const Laned<int*>& n_matches, const Laned<ChainTlmTail>* tail, int lanes) {
    const int n_lp = lp.base.n;
    if (n_lp <= 0) return;
    const Laned<RingHandOverDev> ho = laned_of(lanes, [&](int l) {
        if (!tail) return RingHandOverDev{};
        const ChainTlmTail t = lane_value(*tail, l);
        return RingHandOverDev{t.ring, t.last_xw, t.n_last_cap, t.last_valid, t.last_octave, t.last_desc, t.last_pose};
    });
    const int n_q_cta = (n_lp + 7) / 8, n_ho_cta = tail ? (tail->base.ring.cap + 255) / 256 : 0;
    const int n_cta = n_q_cta > n_ho_cta ? n_q_cta : n_ho_cta;
    const bool pdl = chain_launch_pdl();
    const auto ls = [&](int l) { return lane_value(s, l); };
    const Laned<ListOut> lo = laned_of(lanes, [&](int l) { return list_out(ls(l)); });
    launch_kernel(lanes > 1 ? search_local_collect_kernel<true> : search_local_collect_kernel<false>, dim3(n_cta, lanes), dim3(256), 0, st, pdl, f, cell_start, csr_idx, lp, prm, lo, ho);
    const Laned<ChainEdgesDev> ce = laned_of(lanes, [&](int l) {
        if (!tail) return ChainEdgesDev{};
        const FrameDev fl = lane_value(f, l); const ChainTlmTail t = lane_value(*tail, l);
        return ChainEdgesDev{fl.keys, fl.uright, t.last_xw, t.edges.exw, t.edges.eobs, t.edges.einfo, t.edges.est, t.edges.eidx, t.edges.n_edges};
    });
    const Laned<ChainTlmDev> tl = laned_of(lanes, [&](int l) {
        if (!tail) return ChainTlmDev{};
        const ChainTlmTail t = lane_value(*tail, l);
        return ChainTlmDev{t.match_last, t.lq_xw, t.ring.count, t.n_local_matches};
    });
    launch_kernel(lanes > 1 ? resolve_kernel<true> : resolve_kernel<false>, dim3(1, lanes), dim3(1024), (size_t)resolve_dyn_bytes(), st, pdl, 1, n_lp,
                  laned_of(lanes, [&](int l) { return lane_value(lp, l).n_dev; }), f, lo, laned_of(lanes, [&](int l) { return lane_value(lp, l).obs_pos; }),
                  Laned<const float*>(), prm.nn_ratio, 0, kThHigh, Laned<const float*>(), state, laned_of(lanes, [&](int l) { return ls(l).minq; }),
                  laned_of(lanes, [&](int l) { return ls(l).choice; }), laned_of(lanes, [&](int l) { return ls(l).resolved; }), match, n_matches,
                  laned_of(lanes, [&](int l) { return ls(l).rounds; }), resolve_dyn_bytes(), ce, tl);
}

void launch_search_bow(cudaStream_t st, const FrameDev& f, int n_q, const int* q_feat, const int* q_cbeg, const int* q_cend,
                       const uint8_t* kf_desc, const uint8_t* f_desc, const float* q_angle, const float* f_angle, const int* f_node_feat,
                       float nn_ratio, int keep_max, int check_orientation, const uint8_t* obs_pos, MatchScratch s, uint8_t* state, int* match,
                       int* n_matches) {
    if (n_q <= 0) return;
    bow_collect_kernel<<<(n_q + 7) / 8, 256, 0, st>>>(n_q, q_feat, q_cbeg, q_cend, kf_desc, f_desc, f_node_feat, q_angle, f_angle, check_orientation, keep_max,
                                                    ListOut{s.lists, s.slots, s.list_cap, s.list_n, s.dense, s.dense_slot, s.dense_q, s.base, s.total, s.inv_cnt, s.overflow});
    resolve_kernel<false><<<1, 1024, resolve_dyn_bytes(), st>>>(2, n_q, nullptr, f, ListOut{s.lists, s.slots, s.list_cap, s.list_n, s.dense, s.dense_slot, s.dense_q, s.base, s.total, s.inv_cnt, s.overflow}, obs_pos, q_angle, nn_ratio,
                                       check_orientation, 50 /* TH_LOW */, f_angle, state, s.minq, s.choice, s.resolved, match, n_matches, s.rounds, resolve_dyn_bytes(), ChainEdgesDev{}, ChainTlmDev{});
}

void launch_search_reloc(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, const RelocPointsDev& rp,
                         const SearchRelocParams& prm, const uint8_t* obs_pos, MatchScratch s, uint8_t* state, int* match, int* n_matches) {
    if (rp.n <= 0) return;
    search_reloc_collect_kernel<<<(rp.n + 7) / 8, 256, 0, st>>>(f, cell_start, csr_idx, rp, prm, ListOut{s.lists, s.slots, s.list_cap, s.list_n, s.dense, s.dense_slot, s.dense_q, s.base, s.total, s.inv_cnt, s.overflow});
    resolve_kernel<false><<<1, 1024, resolve_dyn_bytes(), st>>>(0, rp.n, nullptr, f, ListOut{s.lists, s.slots, s.list_cap, s.list_n, s.dense, s.dense_slot, s.dense_q, s.base, s.total, s.inv_cnt, s.overflow}, obs_pos, rp.angle, 0.f,
                                       prm.check_orientation, prm.orb_dist, nullptr, state, s.minq, s.choice, s.resolved, match, n_matches, s.rounds, resolve_dyn_bytes(), ChainEdgesDev{}, ChainTlmDev{});
}

void launch_fuse_search(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, int n, const uint8_t* valid, const float* xw,
                        const float* normal, const float* mf_min, const float* mf_max, const uint8_t* desc, const float* Tcw, const float* Ow, float th,
                        int* best_idx, int* best_dist) {
    if (n <= 0) return;
    fuse_search_kernel<<<(n + 7) / 8, 256, 0, st>>>(f, cell_start, csr_idx, FusePointsDev{n, valid, xw, normal, mf_min, mf_max, desc}, Tcw, Ow, th,
                                                  best_idx, best_dist);
}

void launch_chain_prep(cudaStream_t st, const Laned<ChainPrepDev>& cp, const Laned<const float*>& last_pose, int lanes) {
    if (lanes > 1) chain_prep_kernel<true><<<dim3((cp.base.cap + 255) / 256, lanes), 256, 0, st>>>(cp, last_pose);
    else chain_prep_kernel<false><<<dim3((cp.base.cap + 255) / 256, 1), 256, 0, st>>>(cp, last_pose);
}

void launch_frustum(cudaStream_t st, const FrameDev& f, const FrustumParams& prm, int n, const float* xw, const float* normal,
                    const float* mf_min, const float* mf_max, uint8_t* in_view, float* px, float* py, float* pxr, float* depth,
                    int* level, float* view_cos) {
    if (n <= 0) return;
    frustum_kernel<<<(n + 255) / 256, 256, 0, st>>>(f, prm, n, xw, normal, mf_min, mf_max, in_view, px, py, pxr, depth, level, view_cos);
}

}  // namespace rgbl
