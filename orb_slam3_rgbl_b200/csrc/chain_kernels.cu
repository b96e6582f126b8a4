// Resident tracking chain, TrackLocalMap half (src/Tracking.cc:2983-3050, 3377-3460): after TrackWithMotionModel's
// SearchByProjection(last frame) + PoseOptimization, the reference discards the outliers, projects the local map points that are not
// matched yet (Frame::isInFrustum, src/Frame.cc:602-664), searches them (ORBmatcher::SearchByProjection(F, vpMapPoints, th),
// src/ORBmatcher.cc:43-213) and runs PoseOptimization again on all the frame's map points.  The kernel below is the
// device-side glue between those reference functions (the functions themselves are match_kernels.cu / pose_kernels.cu):
//   tlm_prepare_kernel : outlier discard (src/Tracking.cc:2944-2966) -> isInFrustum over the local map -> ORDERED compaction of the
//                        visible points into the query arrays of the local search (the order of vpMapPoints decides ties);
//   (PoseOptimization's edge list in keypoint order from (inliers of the first search) + (local matches), src/Optimizer.cc:857-990, and the
//    hand-over of the last frame's points into the local map are the tail of the local search's resolution kernel: match_kernels.cu, ChainTlmDev.)
// The local map of the harness is a ring of the K frames before the last one, each contributing its LiDAR-depth keypoints unprojected
// with the frame's final pose; slot = frame counter mod K, points inside a slot in keypoint order.
#include "rgbl_kernels.h"
#include "rgbl_device.cuh"

namespace rgbl {
namespace {

// ---- ordered compaction over SEVERAL CTAs in one launch: "publish and look back" -------------------------------------------------
// The single-CTA versions of the two kernels below walked their input in chunks of 1024 with three block barriers and one round of
// dependent global loads per chunk, all of it latency.  Here every CTA handles one chunk, publishes
// its count in a slot array and reads the counts of the CTAs before it: one global round trip instead of a chain of them.
//   slot value 0 = not published yet, count + 1 otherwise; the CTA that takes the LAST ticket of `done` (after its own look-back, so every
//   reader is through) zeroes the slots and the ticket counter again: the array is clean for the next launch on the stream.
// CTAs of a 1-D grid start in index order and the grids here are a few dozen CTAs, so a CTA only ever waits for CTAs that are already
// running; the wait is bounded all the same (a stuck wait raises the chain's overflow flag instead of hanging the GPU).
constexpr int kTlmThreads = 256;
constexpr int kLbSlots = 1024;             // capacity of one slot array (CTAs per launch)
constexpr int kSpinLimit = 1 << 22;

struct Lookback { int* slots; int* done; int* fail; };

__device__ __forceinline__ int lb_load(const int* p) { return *reinterpret_cast<const volatile int*>(p); }

// called by every thread of the CTA after `count` (the CTA's total, valid in thread 0) is known; returns the sum of the counts of all
// CTAs with a smaller index among the first `n_part` CTAs.  Two block barriers.
__device__ __forceinline__ int lb_exclusive_base(const Lookback& lb, int count, int* s_base) {
    const int tid = threadIdx.x, b = blockIdx.x;
    if (tid == 0) atomicExch(lb.slots + b, count + 1);
    if (tid < 32) {
        int sum = 0;
        for (int j = tid; j < b; j += 32) {
            int v = lb_load(lb.slots + j), spins = 0;
            while (v == 0 && ++spins < kSpinLimit) v = lb_load(lb.slots + j);
            if (v == 0) { atomicExch(lb.fail, kTlmWaitFailed); v = 1; }
            sum += v - 1;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (tid == 0) *s_base = sum;
    }
    __syncthreads();
    return *s_base;
}

// ticket after the CTA is done with the slot array; true for the CTA that has to clean up (call from ONE thread)
__device__ __forceinline__ bool lb_last_ticket(int* counter, int n_part) { return atomicAdd(counter, 1) == n_part - 1; }

// warp-ballot block scan for kTlmThreads threads: exclusive position of `flag` inside the CTA, CTA total in `total` (all threads)
__device__ __forceinline__ int block_rank(int flag, int* s_wsum, int& total) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_wsum[warp] = __popc(m);
    __syncthreads();
    int base = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kTlmThreads / 32; ++w) { const int v = s_wsum[w]; all += v; if (w < warp) base += v; }
    total = all;
    return base + __popc(m & ((1u << lane) - 1u));
}

// grid = n_blocks frustum CTAs (one ring point per thread) + ONE extra CTA (the last) for the slot states of the local search.
// Sequence lanes: lane s = blockIdx.y with its own slot array.  CTAs are dispatched in linear order (lane-major), and a CTA waits only for
// CTAs of its own lane with a smaller x, so still only for CTAs with a smaller linear index.
template <bool kLanes>
__global__ void __launch_bounds__(kTlmThreads) tlm_prepare_kernel(Laned<FrameDev> f_l, Laned<const float*> pose_l, Laned<LocalRingDev> ring_l, float cos_limit,
                                                                  Laned<const int*> n_edges_l, Laned<const int*> e_idx_l,
                                                                  Laned<const uint8_t*> e_outlier_l, Laned<uint8_t*> state_l,
                                                                  Laned<int*> match_last_l, Laned<LocalQueriesDev> lq_l, Laned<Lookback> lb_l) {
    pdl_wait(); pdl_trigger();
    const unsigned ln_ = blockIdx.y;
    const FrameDev& f = lane_arg<kLanes>(f_l, ln_);
    const float* __restrict__ pose = lane_arg<kLanes>(pose_l, ln_);
    const LocalRingDev& ring = lane_arg<kLanes>(ring_l, ln_);
    const int* __restrict__ n_edges = lane_arg<kLanes>(n_edges_l, ln_);
    const int* __restrict__ e_idx = lane_arg<kLanes>(e_idx_l, ln_);
    const uint8_t* __restrict__ e_outlier = lane_arg<kLanes>(e_outlier_l, ln_);
    uint8_t* __restrict__ state = lane_arg<kLanes>(state_l, ln_);
    int* __restrict__ match_last = lane_arg<kLanes>(match_last_l, ln_);
    const LocalQueriesDev& lq = lane_arg<kLanes>(lq_l, ln_);
    const Lookback& lb = lane_arg<kLanes>(lb_l, ln_);
    __shared__ int s_wsum[kTlmThreads / 32];
    __shared__ int s_base;
    const int tid = threadIdx.x;
    const int n_part = (int)gridDim.x - 1;
    if ((int)blockIdx.x == n_part) {
        // slot states for the local search: a slot is occupied exactly when it holds a map point of the first search that survived the
        // rotation check (match >= 0; the resolution kernel keeps its working states on chip) ...
        const int n_f = *f.n;
        for (int i = tid; i < n_f; i += kTlmThreads) state[i] = match_last[i] >= 0 ? 1 : 0;
        __syncthreads();
        // ... and was not an outlier of the first PoseOptimization: those slots are free again (mvpMapPoints[i] = NULL, src/Tracking.cc:2951-2953)
        const int ne = *n_edges;
        for (int e = tid; e < ne; e += kTlmThreads)
            if (e_outlier[e]) { const int i = e_idx[e]; state[i] = 0; match_last[i] = -1; }
        return;
    }
    // Frame::SetPose -> UpdatePoseMatrices (src/Frame.cc:562-569): mRcw = mTcw.rotationMatrix(), mtcw, mOw = Twc.translation(); every thread
    // derives them from the 7 pose floats itself (a few dozen operations) rather than waiting for one thread behind a barrier
    FrustumParams prm;
    {
        float T[7];
#pragma unroll
        for (int i = 0; i < 7; ++i) T[i] = pose[i];
        quatf_to_matrix(T, prm.Rcw);
        float qinv[4];
        se3f_inverse(T, qinv, prm.Ow);
        prm.tcw[0] = T[4]; prm.tcw[1] = T[5]; prm.tcw[2] = T[6];
        prm.cos_limit = cos_limit;
    }
    const int n_ring = ring.K * ring.cap;
    const int p = (int)blockIdx.x * kTlmThreads + tid;
    FrustumOut o{};
    int flag = 0;
    float P[3] = {0.f, 0.f, 0.f};
    if (p < n_ring && ring.valid[p]) {
        P[0] = ring.xw[3 * p]; P[1] = ring.xw[3 * p + 1]; P[2] = ring.xw[3 * p + 2];
        o = frustum_point(f, prm, P, ring.normal + 3 * p, ring.mf_min[p], ring.mf_max[p]);
        flag = o.in_view;
    }
    int total = 0;
    const int rank = block_rank(flag, s_wsum, total);
    const int base = lb_exclusive_base(lb, total, &s_base);
    const int pos = base + rank;
    if (flag && pos < lq.cap) {
        lq.in_view[pos] = 1; lq.obs_pos[pos] = 1;
        lq.proj_x[pos] = o.px; lq.proj_y[pos] = o.py; lq.proj_xr[pos] = o.pxr; lq.depth[pos] = o.depth; lq.level[pos] = o.level;
        lq.view_cos[pos] = o.view_cos; lq.src[pos] = p;
        lq.xw[3 * pos] = P[0]; lq.xw[3 * pos + 1] = P[1]; lq.xw[3 * pos + 2] = P[2];      // the edge list takes the point from here, not from the ring
        const uint4* d = reinterpret_cast<const uint4*>(ring.desc + (size_t)p * 32);
        uint4* dd = reinterpret_cast<uint4*>(lq.desc + (size_t)pos * 32);
        dd[0] = d[0]; dd[1] = d[1];
    }
    if (tid == 0) {
        if ((int)blockIdx.x == n_part - 1) *lq.n = min(base + total, lq.cap);
        if (lb_last_ticket(lb.done, n_part)) {
            for (int j = 0; j < n_part; ++j) lb.slots[j] = 0;
            *lb.done = 0;
        }
    }
}

}  // namespace

// lb: kLbSlots + 8 zero-initialised ints owned by the caller; fail: the chain's overflow flag
int tlm_lookback_ints() { return kLbSlots + 8; }

void launch_tlm_prepare(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const float*>& pose, const Laned<LocalRingDev>& ring, float cos_limit,
                        const Laned<const int*>& n_edges, const Laned<const int*>& e_idx, const Laned<const uint8_t*>& e_outlier, const Laned<uint8_t*>& state,
                        const Laned<int*>& match_last, const Laned<LocalQueriesDev>& lq, int* lb, const Laned<int*>& fail, int lanes) {
    const int n_part = (ring.base.K * ring.base.cap + kTlmThreads - 1) / kTlmThreads;
    const Laned<Lookback> l = laned_of(lanes, [&](int s) {
        int* slots = lb + (size_t)s * tlm_lookback_ints();
        return Lookback{slots, slots + kLbSlots, lane_value(fail, s)};
    });
    launch_kernel(lanes > 1 ? tlm_prepare_kernel<true> : tlm_prepare_kernel<false>, dim3(n_part + 1, lanes), dim3(kTlmThreads), 0, st, chain_launch_pdl(), f, pose, ring, cos_limit, n_edges, e_idx, e_outlier, state, match_last, lq, l);
}

}  // namespace rgbl
