// Context of librgbl_b200.so: memory plan, streams, profiling state (shared by api.cu, api_track.cu, api_bow.cu, api_ba.cu and
// api_mapping.cu).
#ifndef RGBL_CTX_H
#define RGBL_CTX_H

#include <algorithm>
#include <cstddef>
#include <string>
#include <vector>

#include "rgbl_kernels.h"
#include "rgbl_owned.h"

namespace rgbl {

enum Stage { ST_PYRAMID = 0, ST_FAST, ST_COMPACT, ST_BLUR, ST_DESCRIBE, ST_DEPTH_PROJECT, ST_DEPTH_DILATE, ST_DEPTH_GATHER,
             ST_MATCH, ST_POSE, ST_QUADTREE, kNumStages };
static const char* const kStageNames[kNumStages] = {"pyramid", "fast", "compact", "blur", "describe", "depth_project",
                                              "depth_resolve_dilate", "depth_gather", "match", "pose", "quadtree"};

constexpr int kMatchListCap = 512;    // admissible candidates kept per map point (overflow is reported)
static_assert(RGBL_MAX_SEQUENCES == kMaxLanes, "the header's sequence bound is the chain's lane bound");

// the inputs of a resident upload or a staged slot: RGB-L (image + point cloud), RGB-D (image + uint16 depth plane), stereo (left and
// right image of a pair: rectified, or raw when the context rectifies them)
enum class InputKind { rgbl, rgbd, stereo };

// The camera-input setting (rgbl_set_input_resize / _channels, rgbl_set_stereo_rectification): images of w x h (Settings' original camera
// size; the context's unless `resize`, which resizes RGB-D and stereo input to it) and ch bytes per pixel (1, or 3 / 4 interleaved) whose
// channel 0 has the gray weight w0 (gray_of: 9798 with Camera.RGB = 1, else 3735); unrectified stereo pairs with `rectify`.  Derived by
// input_changed (api.cu): the row pitches of an image (bytes) and an input-size depth image (elements), the depth resize's integer factors.
struct InputSetting {
    int w = 0, h = 0, ch = 1, w0 = 3735; bool resize = false, rectify = false;
    int pitch = 0, kx = 0, ky = 0; size_t depth_pitch = 0;
    size_t plane_bytes() const { return (size_t)pitch * h; }     // one input image, without the frame slot around it
    size_t depth_elems() const { return depth_pitch * h; }       // one input-size depth image
};

// What the loaded batch holds for the kernels that write level 0 (api.cu: level0_writer): its images as raw planes at img (plane z at
// img + z * pitch * input.h, ch bytes per pixel, gray weight w0 of channel 0; ch = 0: the upload wrote level 0 itself), recorded per
// upload as a PNG stream may be gray or in R, G, B order, and depth, the input-size depth images the depth resize reads.  Each is a
// working buffer (d_raw_img, d_depth16_raw) or a staged slot's planes, read in place.
struct LoadedInput { const uint8_t* img = nullptr; int ch = 0, w0 = 0, pitch = 0; const uint16_t* depth = nullptr; };

// Words of TrackBufs::scalars (device, 16 ints) the tracking entry points use: the frame size FrameDev::n points at, a search's match
// count and resolution rounds (adjacent: read back as one pair), PoseOptimization's inlier count.
constexpr int kDevFrameN = 0, kDevMatches = 1, kDevRounds = 2, kDevPoseInliers = 8;
// Words of Ctx::h_scalars (pinned, 16 ints).  Every call that uses them is synchronous, so each owns its words for its own duration only:
//   api_track.cu   the words named here; kHostFusePose: ints 4..13 as ten floats (pose, camera centre) of rgbl_fuse_search
//   api_bow.cu     [0..2] ComputeBoW's counts, [8] a frame's keypoint count;   api_mapping.cu   [0] a match count
//   api_ba.cu      all 16 as eight doubles (a trial's scalars), [12] the solver's status
constexpr int kHostFrameN = 0, kHostMatches = 4, kHostRounds = 5, kHostFusePose = 4, kHostPoseInliers = 8;
static_assert(kDevRounds == kDevMatches + 1 && kHostRounds == kHostMatches + 1, "a search's match count and rounds are read back as one pair");

// State that persists between the chains of one sequence (device, TrackBufs::carry), next to the carried frame's arrays: its keypoint
// count and pose, the local map ring's frame counter, the pose of the frame before it.  The chain hands member addresses to its kernels.
struct ChainCarry { int n_sel; float pose[7]; int ring_count; float prev_pose[7]; };
static_assert(sizeof(ChainCarry) == 16 * 4 && offsetof(ChainCarry, pose) == 4 && offsetof(ChainCarry, ring_count) == 32 &&
              offsetof(ChainCarry, prev_pose) == 36, "ChainCarry is 16 packed 32-bit words");

// Counters of one chain over nF frames in `lanes` sequence lanes of m = nF / lanes frames: TrackBufs::ch_counts on the device, a slot of
// Ctx::h_chain_i on the host (one copy brings all of them back).  Four blocks of nF ints in batch order (lane s's frame k at s * m + k), then
// one tail of 8 ints per lane: edges of the first and the second PoseOptimization, the forward / backward flags of the last-frame search,
// the overflow word (matcher list overflow, or kTlmWaitFailed), the local search's query count.
struct ChainCounts { int *n_matches, *n_inliers, *n_local_matches, *n_inliers_first, *n_edges, *n_edges2, *flags, *overflow, *n_queries; };
constexpr size_t chain_count_ints(size_t nF, size_t lanes) { return 4 * nF + 8 * lanes; }
// lane s's counters (its frame 0 and its tail)
inline ChainCounts chain_counts(int* base, size_t nF, size_t m, size_t s) {
    int* head = base + s * m;
    int* tail = base + 4 * nF + 8 * s;
    return {head, head + nF, head + 2 * nF, head + 3 * nF, tail, tail + 1, tail + 2, tail + 4, tail + 5};
}
// Poses of one chain in a slot of Ctx::h_chain_f: the pose given for frame 0 of each lane (kMaxLanes x 7, read by a chain that starts a
// sequence), then the nF results in batch order
constexpr size_t kChainPose0Floats = 7 * (size_t)kMaxLanes;
constexpr size_t chain_pose_floats(size_t nF) { return kChainPose0Floats + nF * 7; }

// Launch parameters of a chain: with the context's buffers and its settings fixed at rgbl_create, everything the enqueue of the chain
// reads (api_track.cu: enqueue_chain takes this struct and nothing else of the call).
// lanes: sequence lanes (rgbl_set_sequences), m = nF / lanes frames each.
struct ChainPlan { int nF, cap, mono, cont, K, prev_valid, lanes, m; float th, th_local, nn_local, fx, fy, cx, cy, bf, bounds[4]; };
// capacity of the query arrays of the chain's local search: the queries are compacted, at most every point of the local map ring
inline int local_query_cap(const ChainPlan& p) { return std::max(p.K * p.cap, 1); }
// The chain's per-lane layout: every TrackBufs buffer the chain writes holds plan.lanes lanes, lane s of a buffer at base + s * stride
// (elements).  ensure_chain_resources grows each buffer to lanes x its stride and chain_lane (api_track.cu) carves lane s with these and
// nothing else.  The batch's frames (the slot snapshot, the grids, ch_poses, ch_counts) are in batch order: lane s's frame k is s * m + k.
struct ChainLaneStrides {
    size_t kp;         // per keypoint of a frame (cap): state, match, match_local, minq, e_*, c_kps, c_depth; x 3: e_xw, e_obs, pose_work; x 32: c_desc
    size_t inv;        // inv_cnt: cap per-feature counters + the dense run's entry total
    size_t q;          // queries (max(cap, local query cap)): q_*, list_n, list_base, choice, resolved; x 3: q_f3*; x kMatchListCap: lists, dense*
    size_t ring;       // local map ring (K x cap): r_valid, r_min, r_max; x 3: r_xw, r_normal; x 32: r_desc
    size_t lq;         // local queries (local query cap): planes of lq_u8 / lq_f / lq_i (kLq*Planes each), x 32: lq_desc
    size_t scalars;    // TrackBufs::scalars: 16 words
    size_t lookback;   // tlm_prepare's slot array: tlm_lookback_ints()
    size_t pose_tmp;   // ch_poses after the nF results: pose after TrackWithMotionModel | predicted pose (14 floats)
};
inline ChainLaneStrides chain_lane_strides(const ChainPlan& p) {
    const size_t cap = (size_t)p.cap, lq = (size_t)local_query_cap(p);
    return {cap, cap + 1, std::max(cap, lq), (size_t)p.K * cap, lq, 16, (size_t)tlm_lookback_ints(), 14};
}
// Key of a slot's CUDA graph: the plan, and Ctx::scratch_generation for the buffer addresses.  Compared with memcmp: value-initialise it.
struct ChainGraphKey { ChainPlan plan; unsigned long long generation; };
static_assert(sizeof(ChainPlan) % sizeof(unsigned long long) == 0, "no padding in ChainGraphKey");

// Lazily grown device scratch of the tracking entry points (api_track.cu).
struct TrackBufs {
    DeviceArray<rgbl_keypoint> keys; DeviceArray<float> uright; DeviceArray<uint8_t> desc, state;
    DeviceArray<int> csr_idx, kp_cell, cell_start, match, minq, scalars;
    DeviceArray<unsigned long long> lists, dense; DeviceArray<uint16_t> list_slots, dense_slot;
    DeviceArray<int> inv_cnt;                            // + 1: the entry total of the dense run (both zero between launches)
    DeviceArray<int> dense_q, list_base, list_n, choice;
    DeviceArray<uint8_t> resolved, q_u8a, q_u8b, q_desc; DeviceArray<float> q_f3a, q_f3b, q_f[7]; DeviceArray<int> q_i;
    DeviceArray<double> pose_work;
    // resident tracking chain
    DeviceArray<float> ch_poses, e_xw, e_obs, e_info; DeviceArray<int> ch_counts, e_idx; DeviceArray<uint8_t> e_st, e_lvl, e_out;
    // chain-owned snapshot of the batch's frame outputs (so that the next batch's frame construction may overwrite the
    // context's buffers while the chain of this batch is still running) + per-frame grids built in one launch
    DeviceArray<rgbl_keypoint> s_kps; DeviceArray<uint8_t> s_desc; DeviceArray<float> s_depth, s_uright;
    DeviceArray<int> s_nsel, b_cell_start, b_csr_idx, b_kp_cell;
    // state that persists between the chains of one sequence: the carried last frame and the local map ring (chain_kernels.cu)
    DeviceArray<rgbl_keypoint> c_kps; DeviceArray<uint8_t> c_desc; DeviceArray<float> c_depth;
    DeviceArray<ChainCarry> carry;                       // one element per sequence lane
    DeviceArray<uint8_t> r_valid, r_desc, lq_u8, lq_desc; DeviceArray<float> r_xw, r_normal, r_min, r_max, lq_f; DeviceArray<int> lq_i, match_local;
    DeviceArray<int> lookback;                           // slot arrays of the multi-CTA compactions (chain_kernels.cu), kept zero between launches
    // ComputeBoW
    DeviceArray<int> bw_i;                               // f_word | f_node | bow_word | fv_node | fv_start | fv_feature | scratch | counts
    DeviceArray<double> bw_d;                            // f_weight | bow_value
};

struct Ctx {
    rgbl_config cfg{};
    OrbTables tab{};
    std::vector<LevelGeom> levels;
    std::vector<CellInfo> cells;
    std::vector<LinCoef> coefs;
    size_t frame_bytes = 0;
    int n_cells = 0;
    int cap_kp = 0;              // keypoints per frame capacity (nfeatures + 3 per level)
    bool qt_device_ok = false;   // the context's geometry fits the device quad-tree (every level: quota + 3 <= 1024, 1 <= nIni <= 64, shared memory)
    int qt_max_nodes = 0;        // largest node list of any level's quad-tree (selects the half-size tree state: two trees per SM)
    int dense_cap = 0;           // candidates per batch capacity
    std::string err;

    Stream st, st_aux;
    Event ev_pyr, ev_blur, ev_t0, ev_t1;

    // device
    DeviceArray<LevelGeom> d_levels;
    DeviceArray<CellInfo> d_cells;
    DeviceArray<LinCoef> d_coefs;
    DeviceArray<uint8_t> d_pyr, d_blur;
    DeviceArray<uint32_t> d_slots;
    DeviceArray<int> d_counts, d_cell_off, d_level_cnt, d_frame_total, d_overflow;
    DeviceArray<uint32_t> d_dense;
    DeviceArray<SelKp> d_sel;
    DeviceArray<int> d_n_sel;
    DeviceArray<rgbl_keypoint> d_kps, d_kps_un, d_kps_in;
    DeviceArray<int> d_n_kp_in;
    DeviceArray<uint8_t> d_desc;
    DeviceArray<float> d_pts;
    DeviceArray<float> d_pts_raw;   // lazily allocated: raw (x, y, z, r) records awaiting de-interleave
    // png_kernels.cu (lazily allocated): inflated-but-still-filtered scanlines, pinned + device, one slot of png_raw_stride bytes per frame;
    // the reconstructed row above each 512-row band; status word (bad filter type)
    PinnedArray<uint8_t> h_png_raw; DeviceArray<uint8_t> d_png_raw;
    DeviceArray<uint32_t> d_png_band;
    DeviceArray<int> d_png_status; PinnedArray<int> h_png_status;
    size_t png_raw_stride = 0;
    // RGB-D (lazily allocated by the first RGB-D call): one uint16 depth plane per frame slot as imread returns it (CV_16U), row pitch
    // depth16_pitch elements (64-byte rows); scaled to metric depth by the gather
    DeviceArray<uint16_t> d_depth16;
    size_t depth16_pitch = 0;
    // Frame::ComputeStereoMatches scratch (lazily allocated by the first stereo call, sized once for max(1, max_batch / 2) pairs): per
    // pair the row index (row starts, row lists of stereo_row_index_cap entries) and the matched SADs.  Never reallocated and never
    // referenced by the chain's CUDA graphs, so it needs no scratch_generation bump.
    DeviceArray<int> d_stereo_row_start, d_stereo_row_idx, d_stereo_sad;
    int stereo_idx_cap = 0;
    InputSetting input;
    // stereo rectification (stereo_kernels.cu).  d_rect_xy / d_rect_a: OpenCV's fixed-point form of the left and right maps, H rows of
    // rect_pitch entries per camera, allocated by the first setting and never reallocated.
    DeviceArray<uint32_t> d_rect_xy; DeviceArray<uint16_t> d_rect_a;
    int rect_pitch = 0;
    DeviceArray<LinCoef> d_resize_coefs;      // the input resize's cv::resize tables of the two axes (x: W entries, then y: H entries)
    // The raw planes of uploads and PNG decodes (LoadedInput): max_batch input-size images or depth images, allocated by the first upload
    // that needs them and reallocated when a later one needs more.  No chain graph references them, so they need no scratch_generation bump.
    DeviceArray<uint8_t> d_raw_img; DeviceArray<uint16_t> d_depth16_raw;
    LoadedInput loaded;
    DeviceArray<int> d_n_pts;
    DeviceArray<uint32_t> d_idx_map;
    DeviceArray<float> d_raw, d_processed, d_depth, d_uright;
    DeviceArray<uint8_t> d_scratch;   // padded-level export
    size_t scratch_bytes = 0;
    uint32_t stamp = 0;

    // pinned host
    PinnedArray<int> h_level_cnt, h_frame_total, h_overflow, h_n_sel, h_n_pts;
    PinnedArray<uint32_t> h_dense;
    PinnedArray<SelKp> h_sel;

    // profiling (rgbl_profile_*): CUDA events on the launching stream around every stage
    bool prof_on = false, prof_serial = false;   // prof_serial: stage timings without stream overlap (the aux-stream work is joined before the quad-tree)
    Event ev_b[kNumStages], ev_e[kNumStages];
    bool st_used[kNumStages] = {};
    Event ev_rsd_b, ev_rsd_e; bool rsd_used = false;   // the depth resize on the aux stream, billed to depth_gather besides the gather itself
    int st_pending_launches[kNumStages] = {};
    double st_ms[kNumStages] = {};
    long st_launches[kNumStages] = {};
    long st_calls[kNumStages] = {};
    double host_quadtree_ms = 0.0;
    long total_launches = 0;

    // device quad-tree (quadtree_kernels.cu)
    bool device_quadtree = false, host_counts_valid = false;
    LevelTensorMaps level_tms{};                 // level_tma_kernels.cu; level_tma: the fused TMA tile kernel replaces launch_pyramid + launch_blur (RGBL_LEVEL_TMA=0: off)
    bool level_tma = false;
    // cell strips of the FAST kernel (fast_strip.cuh)
    std::vector<StripInfo> strips;
    DeviceArray<StripInfo> d_strips;
    int strip_rows_cap = 0, strip_list_cap = 0;
    DeviceArray<unsigned short> qt_perm_a, qt_perm_b, qt_node_a, qt_node_b; DeviceArray<unsigned long long> qt_scan; DeviceArray<unsigned char> qt_quad;
    QtScratchDev qt_scr{};                       // view of the six arrays above, as the quad-tree launcher takes it
    DeviceArray<uint32_t> d_sel_lvl;
    DeviceArray<int> d_n_sel_lvl, d_lvl_region;

    TrackBufs trk;
    // grow-only device arena of the mapping-thread entry points (local BA, SearchForTriangulation, distinctive descriptors): those
    // calls are synchronous, so one buffer serves them in turn and no call pays a device allocation or free (both synchronise)
    DeviceArray<char> map_arena;
    PinnedArray<int> h_scalars;  // 16 ints
    int last_match_rounds = 0;

    // asynchronous tracking chain (rgbl_resident_track_begin / _end): own high-priority stream, pinned result staging
    Stream st_trk;
    // Up to two chains may be queued (slots 0 / 1, FIFO): the second one is enqueued behind the first on the tracking stream,
    // so the device never waits for the host between two batches.  Per slot: snapshot buffers (TrackBufs::s_*, b_*, carved by
    // slot), pinned result staging, completion and profiling events.
    Event ev_snap, ev_chain_b[2], ev_chain_e[2], ev_chain_done[2];
    int chain_pending = 0;       // chains in flight (0..2)
    int chain_head = 0;          // slot of the oldest chain in flight
    int chain_frames[2] = {}, chain_lanes[2] = {1, 1}, chain_launches[2] = {}, chain_first[2] = {}, chain_graph_launches[2] = {};
    long chain_tracked_frames = 0;               // frames that went through the chain (frame 0 of a non-continuing chain is given, not tracked)
    bool chain_has_carry = false; int carry_K = 0, carry_cap = 0, carry_lanes = 1;
    // sequence lanes (rgbl_set_sequences): batches hold `lanes` sequences of consecutive frames; lane_pose0[s] = lane s's start pose when
    // lane_pose0_set (else every lane starts at rgbl_chain_params::pose0)
    int lanes = 1; bool lane_pose0_set = false; float lane_pose0[kMaxLanes][7] = {};
    bool carry_prev_valid = false;               // the carried sequence also holds the pose BEFORE its last frame (constant-velocity motion model)
    PinnedArray<int> h_chain_ovf;                // per slot: the two frame-construction overflow flags of the tracked batch
    // The chain's CUDA graphs hold raw pointers into the buffers of this context.  Every buffer that can be reallocated after
    // rgbl_create (TrackBufs, the mapping arena, the pinned chain staging) therefore grows only through OwnedArray::grow with this
    // counter, and the counter is part of the graphs' key: any reallocation re-captures them.
    unsigned long long scratch_generation = 1;
    bool chain_timing_on = false, chain_graphs_on = true;   // RGBL_CHAIN_TIMING / RGBL_CHAIN_GRAPH, read at rgbl_create
    bool chain_pdl_on = true;                               // RGBL_CHAIN_PDL=0: ordinary launches between the chain's kernels
    Event chain_tev[8];
    PinnedArray<float> h_chain_f;  // per slot: chain_pose_floats(h_chain_cap)
    PinnedArray<int> h_chain_i;    // per slot: chain_count_ints(h_chain_cap), laid out by chain_counts(slot's base, the chain's frames)
    size_t h_chain_cap = 0;      // frames per slot
    // the chain of a slot as an instantiated CUDA graph (re-captured when any launch parameter or scratch pointer changes)
    GraphExec chain_exec[2];
    ChainGraphKey chain_key[2] = {};
    bool chain_timing_recorded = false;      // RGBL_CHAIN_TIMING development aid: chain_tev hold the timings of a chain

    // staged input slots of the sequence runners (rgbl_resident_stage / rgbl_track_sequence, rgbl_resident_stage_rgbd /
    // rgbl_track_sequence_rgbd, rgbl_resident_stage_stereo / rgbl_track_sequence_stereo): level-0 planes + clouds (RGB-L), uint16 depth
    // planes (RGB-D) or the left then the right level-0 planes (stereo: n_frames pairs, 2 n_frames planes) of whole batches
    static constexpr int kMaxStageSlots = 8;
    struct StageSlot {
        DeviceArray<uint8_t> img; DeviceArray<float> pts; DeviceArray<int> n_pts; DeviceArray<uint16_t> depth;
        int n_frames = 0, max_pts = 0; InputKind kind = InputKind::rgbl; InputSetting input;   // input: the setting it was staged with
    };
    StageSlot stage[kMaxStageSlots];

    // camera model of Frame::UndistortKeyPoints / ComputeImageBounds (rgbl_set_camera_distortion): undistort = (k1 != 0); cam_bounds =
    // mnMinX, mnMaxX, mnMinY, mnMaxY of that camera ((0, W, 0, H) when k1 == 0)
    bool undistort = false;
    UndistortDev cam_un{};
    float cam_bounds[4] = {};
    // mvKeysUn and image bounds of the frames in the device buffers, set by each batched frame construction: frames_undistorted ->
    // d_kps_un ([max_batch][cap_kp]) holds mvKeysUn, else mvKeysUn == mvKeys (d_kps).  The tracking chain reads these.
    bool frames_undistorted = false;
    float frame_bounds[4] = {};

    int last_frames = 0;         // frames valid in the device buffers
    int resident_frames = 0, resident_max_pts = 0;   // stereo: resident_frames pairs in slots [0, 2 resident_frames)
    InputKind resident_kind = InputKind::rgbl;      // what the uploaded frames are
    bool blur_valid = false;
};

// returns the context's mapping arena with at least `bytes` bytes (nullptr on allocation failure)
inline char* mapping_arena(Ctx* c, size_t bytes) {
    return c->map_arena.grow(bytes, c->scratch_generation, bytes + bytes / 4 + (1 << 20)) ? c->map_arena.get() : nullptr;
}

// the mapping arena with at least `bytes` bytes, carved into 256-byte aligned arrays in call order (base == nullptr: allocation failed)
struct ArenaCarve {
    char* base; size_t cap, used = 0;
    ArenaCarve(Ctx* c, size_t bytes) : base(mapping_arena(c, bytes)), cap(bytes) {}
    template <class T> T* take(size_t n) { used = (used + 255) & ~(size_t)255; T* p = reinterpret_cast<T*>(base + used); used += n * sizeof(T); return p; }
};

#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            c->err = std::string(#call) + ": " + cudaGetErrorString(e_);                           \
            return RGBL_E_CUDA;                                                                    \
        }                                                                                          \
    } while (0)


// Entry guard of every call that must not run beside a tracking chain: the context exists and no chain is in flight.  (Only
// rgbl_resident_track_begin* / _end*, which queue and collect the chains, run with one pending.)
inline int require_idle(Ctx* c) {
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    return RGBL_OK;
}

// frames per half of the per-slot buffers: the context's full batch (frame construction refuses larger ones), so that the halves never
// move while a chain is in flight
inline size_t slot_frames(const Ctx* c) { return (size_t)std::max(c->last_frames, c->cfg.max_batch); }

// A slot's half of the per-slot buffers: the snapshot of the batch's frame outputs, the per-frame grids, the pinned result staging.
struct ChainSlot {
    rgbl_keypoint* s_kps; uint8_t* s_desc; float* s_depth; float* s_uright; int* s_nsel;
    int* b_cell_start; int* b_csr_idx; int* b_kp_cell;
    float* h_f; int* h_i;
};
inline ChainSlot chain_slot(Ctx* c, int slot) {
    TrackBufs& t = c->trk;
    const size_t nF = slot_frames(c), tot = nF * c->cap_kp, cs = nF * (kGridCols * kGridRows + 1);
    return {t.s_kps + slot * tot, t.s_desc + slot * tot * 32, t.s_depth + slot * tot, t.s_uright + slot * tot, t.s_nsel + slot * nF,
            t.b_cell_start + slot * cs, t.b_csr_idx + slot * tot, t.b_kp_cell + slot * tot,
            c->h_chain_f + slot * chain_pose_floats(c->h_chain_cap), c->h_chain_i + slot * chain_count_ints(c->h_chain_cap, kMaxLanes)};
}

// The query arrays of the chain's local search (one lane): planes of n_lq elements in lq_u8 (2), lq_f (8: five scalars, then xyz) and lq_i (2)
constexpr int kLqU8Planes = 2, kLqFPlanes = 8, kLqIPlanes = 2;
inline LocalQueriesDev local_queries(uint8_t* u8, float* f, int* i, uint8_t* desc, int n_lq, int* n) {
    const size_t s = (size_t)n_lq;
    LocalQueriesDev lq{};
    lq.cap = n_lq; lq.n = n; lq.in_view = u8; lq.obs_pos = u8 + s;
    lq.proj_x = f; lq.proj_y = f + s; lq.proj_xr = f + 2 * s; lq.depth = f + 3 * s; lq.view_cos = f + 4 * s; lq.xw = f + 5 * s;
    lq.level = i; lq.src = i + s; lq.desc = desc;
    return lq;
}

// n elements between host and device memory on the context's main stream; n == 0 issues nothing (the pointers may then be null).  The
// element size comes from the host pointer's type; the device side (a DeviceArray or a pointer into one) converts to it.
template <class T> struct SameAs { using type = T; };
template <class T> inline cudaError_t h2d(Ctx* c, typename SameAs<T>::type* dst, const T* src, size_t n) {
    return n ? cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, c->st) : cudaSuccess;
}
template <class T> inline cudaError_t d2h(Ctx* c, T* dst, const typename SameAs<T>::type* src, size_t n) {
    return n ? cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, c->st) : cudaSuccess;
}

// profiling helpers (api.cu)
void stage_begin(Ctx* c, int stage, cudaStream_t st);
void stage_end(Ctx* c, int stage, cudaStream_t st, int launches);
void prof_collect(Ctx* c);

// Frame::ComputeStereoMatches for the pairs (l0 + p, r0 + p), p < n_pairs, of the last batched extraction, on the main stream and billed to
// the match stage (api.cu): mvDepth / mvuRight of the left slots in d_depth / d_uright.  Allocates the stereo scratch on first use.
int stereo_matches(Ctx* c, int l0, int r0, int n_pairs, float mb, float mbf);

}  // namespace rgbl
#endif
