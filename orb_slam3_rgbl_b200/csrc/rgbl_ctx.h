// Context of librgbl_b200.so: memory plan, streams, profiling state (shared by api.cu and api_track.cu).
#ifndef RGBL_CTX_H
#define RGBL_CTX_H

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

// the inputs of a resident upload or a staged slot: RGB-L (image + point cloud), RGB-D (image + uint16 depth plane), stereo (left and
// right image of a pair: rectified, or raw when the context rectifies them)
enum class InputKind { rgbl, rgbd, stereo };

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
    DeviceArray<uint32_t> c_misc;                        // n_sel | pose[7] | ring frame counter
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
    // stereo rectification (rgbl_set_stereo_rectification, stereo_kernels.cu).  d_rect_xy / d_rect_a: OpenCV's fixed-point form of the
    // left and right maps, H rows of rect_pitch entries per camera, allocated by the first setting and never reallocated.  d_rect_raw:
    // max_batch raw planes in level 0's layout (row pitch levels[0].pitch), allocated by the first stereo upload with rectification on;
    // host uploads and PNG decodes of pairs write there instead of level 0.  rect_src: the raw planes of the uploaded pairs (d_rect_raw,
    // or a staged slot's planes).  No chain graph references these buffers, so they need no scratch_generation bump.
    bool rectify = false;
    DeviceArray<uint32_t> d_rect_xy; DeviceArray<uint16_t> d_rect_a;
    int rect_pitch = 0;
    DeviceArray<uint8_t> d_rect_raw;
    const uint8_t* rect_src = nullptr;
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
    int st_pending_launches[kNumStages] = {};
    double st_ms[kNumStages] = {};
    long st_launches[kNumStages] = {};
    long st_calls[kNumStages] = {};
    double host_quadtree_ms = 0.0;
    long total_launches = 0;

    // device quad-tree (quadtree_kernels.cu)
    bool device_quadtree = false, host_counts_valid = false;
    // strip formulation of the FAST kernel (fast_strip.cuh); selected with RGBL_FAST_STRIPS=1
    LevelTensorMaps level_tms{};                 // level_tma_kernels.cu; level_tma: the fused TMA tile kernel replaces launch_pyramid + launch_blur (RGBL_LEVEL_TMA=0: off)
    bool level_tma = false;
    bool fast_strips = false, describe_staged = false, dilate_v2 = false;   // RGBL_DESCRIBE_STAGED=1: describe_warp_kernels.cu
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
    int chain_frames[2] = {}, chain_launches[2] = {}, chain_first[2] = {}, chain_graph_launches[2] = {};
    long chain_tracked_frames = 0;               // frames that went through the chain (frame 0 of a non-continuing chain is given, not tracked)
    bool chain_has_carry = false; int carry_K = 0, carry_cap = 0;
    bool carry_prev_valid = false;               // the carried sequence also holds the pose BEFORE its last frame (constant-velocity motion model)
    PinnedArray<int> h_chain_ovf;                // per slot: the two frame-construction overflow flags of the tracked batch
    // The chain's CUDA graphs hold raw pointers into the buffers of this context.  Every buffer that can be reallocated after
    // rgbl_create (TrackBufs, the mapping arena, the pinned chain staging) therefore grows only through OwnedArray::grow with this
    // counter, and the counter is part of the graphs' key: any reallocation re-captures them.
    unsigned long long scratch_generation = 1;
    bool chain_timing_on = false, chain_graphs_on = true;   // RGBL_CHAIN_TIMING / RGBL_CHAIN_GRAPH, read at rgbl_create
    bool chain_pdl_on = true;                               // RGBL_CHAIN_PDL=0: ordinary launches between the chain's kernels
    Event chain_tev[8];
    PinnedArray<float> h_chain_f;  // per slot: pose0 (7) | poses (cap * 7)
    PinnedArray<int> h_chain_i;    // per slot: n_matches | n_inliers | n_local_matches | n_inliers_first | n_edges x2, flags[2], overflow, n_queries
    size_t h_chain_cap = 0;      // frames per slot
    // the chain of a slot as an instantiated CUDA graph (re-captured when any launch parameter or scratch pointer changes)
    struct ChainGraphKey { int nF, cap, mono, cont, K, prev_valid; float th, th_local, nn_local, fx, fy, cx, cy, bf, bounds[4]; unsigned long long generation; };
    GraphExec chain_exec[2];
    ChainGraphKey chain_key[2] = {};
    bool chain_timing_recorded = false;      // RGBL_CHAIN_TIMING development aid: chain_tev hold the timings of a chain

    // staged input slots of the sequence runners (rgbl_resident_stage / rgbl_track_sequence, rgbl_resident_stage_rgbd /
    // rgbl_track_sequence_rgbd, rgbl_resident_stage_stereo / rgbl_track_sequence_stereo): level-0 planes + clouds (RGB-L), uint16 depth
    // planes (RGB-D) or the left then the right level-0 planes (stereo: n_frames pairs, 2 n_frames planes) of whole batches
    static constexpr int kMaxStageSlots = 8;
    struct StageSlot { DeviceArray<uint8_t> img; DeviceArray<float> pts; DeviceArray<int> n_pts; DeviceArray<uint16_t> depth; int n_frames = 0, max_pts = 0; InputKind kind = InputKind::rgbl; };
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


// profiling helpers (api.cu)
void stage_begin(Ctx* c, int stage, cudaStream_t st);
void stage_end(Ctx* c, int stage, cudaStream_t st, int launches);
void prof_collect(Ctx* c);

// Frame::ComputeStereoMatches for the pairs (l0 + p, r0 + p), p < n_pairs, of the last batched extraction, on the main stream and billed to
// the match stage (api.cu): mvDepth / mvuRight of the left slots in d_depth / d_uright.  Allocates the stereo scratch on first use.
int stereo_matches(Ctx* c, int l0, int r0, int n_pairs, float mb, float mbf);

}  // namespace rgbl
#endif
