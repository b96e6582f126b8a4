// Context of librgbl_b200.so: memory plan, streams, profiling state (shared by api.cu and api_track.cu).
#ifndef RGBL_CTX_H
#define RGBL_CTX_H

#include <string>
#include <vector>

#include "rgbl_kernels.h"

namespace rgbl {

enum Stage { ST_PYRAMID = 0, ST_FAST, ST_COMPACT, ST_BLUR, ST_DESCRIBE, ST_DEPTH_PROJECT, ST_DEPTH_DILATE, ST_DEPTH_GATHER,
             ST_MATCH, ST_POSE, ST_QUADTREE, kNumStages };
static const char* const kStageNames[kNumStages] = {"pyramid", "fast", "compact", "blur", "describe", "depth_project",
                                              "depth_resolve_dilate", "depth_gather", "match", "pose", "quadtree"};

constexpr int kMatchListCap = 512;    // admissible candidates kept per map point (overflow is reported)

// Lazily grown device scratch of the tracking entry points (api_track.cu).
struct TrackBufs {
    rgbl_keypoint* keys = nullptr; size_t cap_keys = 0;
    float* uright = nullptr; size_t cap_uright = 0;
    uint8_t* desc = nullptr; size_t cap_desc = 0;
    int* csr_idx = nullptr; size_t cap_csr = 0;
    int* kp_cell = nullptr; size_t cap_kpcell = 0;
    int* cell_start = nullptr; size_t cap_cellstart = 0;
    uint8_t* state = nullptr; size_t cap_state = 0;
    int* match = nullptr; size_t cap_match = 0;
    int* minq = nullptr; size_t cap_minq = 0;
    int* scalars = nullptr; size_t cap_scalars = 0;
    unsigned long long* lists = nullptr; size_t cap_lists = 0;
    uint16_t* list_slots = nullptr; size_t cap_list_slots = 0;
    int* inv_cnt = nullptr; size_t cap_inv_cnt = 0;           // + 1: the entry total of the dense run (both zero between launches)
    unsigned long long* dense = nullptr; size_t cap_dense = 0;
    uint16_t* dense_slot = nullptr; size_t cap_dense_slot = 0;
    int *dense_q = nullptr, *list_base = nullptr; size_t cap_dense_q = 0, cap_list_base = 0;
    int* list_n = nullptr; size_t cap_listn = 0;
    int* choice = nullptr; size_t cap_choice = 0;
    uint8_t* resolved = nullptr; size_t cap_resolved = 0;
    uint8_t *q_u8a = nullptr, *q_u8b = nullptr, *q_desc = nullptr; size_t cap_q_u8a = 0, cap_q_u8b = 0, cap_q_desc = 0;
    float *q_f3a = nullptr, *q_f3b = nullptr; size_t cap_q_f3a = 0, cap_q_f3b = 0;
    float* q_f[7] = {}; size_t cap_q_f[7] = {};
    int* q_i = nullptr; size_t cap_q_i = 0;
    double* pose_work = nullptr; size_t cap_pose_work = 0;
    // resident tracking chain
    float* ch_poses = nullptr; size_t cap_ch_poses = 0;
    int* ch_counts = nullptr; size_t cap_ch_counts = 0;
    float *e_xw = nullptr, *e_obs = nullptr, *e_info = nullptr; size_t cap_e_xw = 0, cap_e_obs = 0, cap_e_info = 0;
    uint8_t *e_st = nullptr, *e_lvl = nullptr, *e_out = nullptr; size_t cap_e_st = 0, cap_e_lvl = 0, cap_e_out = 0;
    int* e_idx = nullptr; size_t cap_e_idx = 0;
    // chain-owned snapshot of the batch's frame outputs (so that the next batch's frame construction may overwrite the
    // context's buffers while the chain of this batch is still running) + per-frame grids built in one launch
    rgbl_keypoint* s_kps = nullptr; size_t cap_s_kps = 0;
    uint8_t* s_desc = nullptr; size_t cap_s_desc = 0;
    float *s_depth = nullptr, *s_uright = nullptr; size_t cap_s_depth = 0, cap_s_uright = 0;
    int* s_nsel = nullptr; size_t cap_s_nsel = 0;
    int *b_cell_start = nullptr, *b_csr_idx = nullptr, *b_kp_cell = nullptr; size_t cap_b_cell_start = 0, cap_b_csr_idx = 0, cap_b_kp_cell = 0;
    // state that persists between the chains of one sequence: the carried last frame and the local map ring (chain_kernels.cu)
    rgbl_keypoint* c_kps = nullptr; size_t cap_c_kps = 0;
    uint8_t* c_desc = nullptr; size_t cap_c_desc = 0;
    float* c_depth = nullptr; size_t cap_c_depth = 0;
    uint32_t* c_misc = nullptr; size_t cap_c_misc = 0;      // n_sel | pose[7] | ring frame counter
    uint8_t *r_valid = nullptr, *r_desc = nullptr; size_t cap_r_valid = 0, cap_r_desc = 0;
    float *r_xw = nullptr, *r_normal = nullptr, *r_min = nullptr, *r_max = nullptr; size_t cap_r_xw = 0, cap_r_normal = 0, cap_r_min = 0, cap_r_max = 0;
    uint8_t *lq_u8 = nullptr, *lq_desc = nullptr; size_t cap_lq_u8 = 0, cap_lq_desc = 0;
    float* lq_f = nullptr; size_t cap_lq_f = 0;
    int *lq_i = nullptr, *match_local = nullptr; size_t cap_lq_i = 0, cap_match_local = 0;
    int* lookback = nullptr; size_t cap_lookback = 0;     // slot arrays of the multi-CTA compactions (chain_kernels.cu), kept zero between launches
    // ComputeBoW
    int *bw_i = nullptr; size_t cap_bw_i = 0;            // f_word | f_node | bow_word | fv_node | fv_start | fv_feature | scratch | counts
    double* bw_d = nullptr; size_t cap_bw_d = 0;         // f_weight | bow_value
    void release() {
        void* all[] = {list_slots, inv_cnt, dense, dense_slot, dense_q, list_base, keys, uright, desc, csr_idx, kp_cell, cell_start, state, match, minq, scalars, lists, list_n, choice, resolved,
                       q_u8a, q_u8b, q_desc, q_f3a, q_f3b, q_f[0], q_f[1], q_f[2], q_f[3], q_f[4], q_f[5], q_f[6], q_i, pose_work, ch_poses, ch_counts, e_xw, e_obs, e_info, e_st, e_lvl, e_out, e_idx,
                       s_kps, s_desc, s_depth, s_uright, s_nsel, b_cell_start, b_csr_idx, b_kp_cell, bw_i, bw_d,
                       c_kps, c_desc, c_depth, c_misc, r_valid, r_desc, r_xw, r_normal, r_min, r_max, lq_u8, lq_desc, lq_f, lq_i, match_local, lookback};
        for (void* p : all) if (p) cudaFree(p);
    }
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

    cudaStream_t st = nullptr, st_aux = nullptr;
    cudaEvent_t ev_pyr = nullptr, ev_blur = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;

    // device
    LevelGeom* d_levels = nullptr;
    CellInfo* d_cells = nullptr;
    LinCoef* d_coefs = nullptr;
    uint8_t *d_pyr = nullptr, *d_blur = nullptr;
    uint32_t* d_slots = nullptr;
    int *d_counts = nullptr, *d_cell_off = nullptr, *d_level_cnt = nullptr, *d_frame_total = nullptr, *d_overflow = nullptr;
    uint32_t* d_dense = nullptr;
    SelKp* d_sel = nullptr;
    int* d_n_sel = nullptr;
    rgbl_keypoint *d_kps = nullptr, *d_kps_un = nullptr, *d_kps_in = nullptr;
    int* d_n_kp_in = nullptr;
    uint8_t* d_desc = nullptr;
    float* d_pts = nullptr;
    float* d_pts_raw = nullptr;   // lazily allocated: raw (x, y, z, r) records awaiting de-interleave
    // png_kernels.cu (lazily allocated): inflated-but-still-filtered scanlines, pinned + device, one slot of png_raw_stride bytes per frame;
    // the reconstructed row above each 512-row band; status word (bad filter type)
    uint8_t *h_png_raw = nullptr, *d_png_raw = nullptr;
    uint32_t* d_png_band = nullptr;
    int *d_png_status = nullptr, *h_png_status = nullptr;
    size_t png_raw_stride = 0;
    // RGB-D (lazily allocated by the first RGB-D call): one uint16 depth plane per frame slot as imread returns it (CV_16U), row pitch
    // depth16_pitch elements (64-byte rows); scaled to metric depth by the gather
    uint16_t* d_depth16 = nullptr;
    size_t depth16_pitch = 0;
    int* d_n_pts = nullptr;
    uint32_t* d_idx_map = nullptr;
    float *d_raw = nullptr, *d_processed = nullptr, *d_depth = nullptr, *d_uright = nullptr;
    uint8_t* d_scratch = nullptr;   // padded-level export
    size_t scratch_bytes = 0;
    uint32_t stamp = 0;

    // pinned host
    int *h_level_cnt = nullptr, *h_frame_total = nullptr, *h_overflow = nullptr, *h_n_sel = nullptr, *h_n_pts = nullptr;
    uint32_t* h_dense = nullptr;
    SelKp* h_sel = nullptr;

    // profiling (rgbl_profile_*): CUDA events on the launching stream around every stage
    bool prof_on = false, prof_serial = false;   // prof_serial: stage timings without stream overlap (the aux-stream work is joined before the quad-tree)
    cudaEvent_t ev_b[kNumStages] = {}, ev_e[kNumStages] = {};
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
    StripInfo* d_strips = nullptr;
    int strip_rows_cap = 0, strip_list_cap = 0;
    QtScratchDev qt_scr{};
    uint32_t* d_sel_lvl = nullptr;
    int *d_n_sel_lvl = nullptr, *d_lvl_region = nullptr;

    TrackBufs trk;
    // grow-only device arena of the mapping-thread entry points (local BA, SearchForTriangulation, distinctive descriptors): those
    // calls are synchronous, so one buffer serves them in turn and no call pays a cudaMalloc / cudaFree (both synchronise)
    char* map_arena = nullptr; size_t map_arena_cap = 0;
    int* h_scalars = nullptr;    // pinned, 16 ints
    int last_match_rounds = 0;

    // asynchronous tracking chain (rgbl_resident_track_begin / _end): own high-priority stream, pinned result staging
    cudaStream_t st_trk = nullptr;
    // Up to two chains may be queued (slots 0 / 1, FIFO): the second one is enqueued behind the first on the tracking stream,
    // so the device never waits for the host between two batches.  Per slot: snapshot buffers (TrackBufs::s_*, b_*, carved by
    // slot), pinned result staging, completion and profiling events.
    cudaEvent_t ev_snap = nullptr, ev_chain_b[2] = {}, ev_chain_e[2] = {}, ev_chain_done[2] = {};
    int chain_pending = 0;       // chains in flight (0..2)
    int chain_head = 0;          // slot of the oldest chain in flight
    int chain_frames[2] = {}, chain_launches[2] = {}, chain_first[2] = {}, chain_graph_launches[2] = {};
    long chain_tracked_frames = 0;               // frames that went through the chain (frame 0 of a non-continuing chain is given, not tracked)
    bool chain_has_carry = false; int carry_K = 0, carry_cap = 0;
    bool carry_prev_valid = false;               // the carried sequence also holds the pose BEFORE its last frame (constant-velocity motion model)
    int* h_chain_ovf = nullptr;                  // pinned, per slot: the two frame-construction overflow flags of the tracked batch
    unsigned long long scratch_generation = 1;   // bumped by every reallocation of this context's tracking scratch
    bool chain_timing_on = false, chain_graphs_on = true;   // RGBL_CHAIN_TIMING / RGBL_CHAIN_GRAPH, read at rgbl_create
    bool chain_pdl_on = true;                               // RGBL_CHAIN_PDL=0: ordinary launches between the chain's kernels
    cudaEvent_t chain_tev[8] = {};
    float* h_chain_f = nullptr;  // pinned, per slot: pose0 (7) | poses (cap * 7)
    int* h_chain_i = nullptr;    // pinned, per slot: n_matches | n_inliers | n_local_matches | n_inliers_first | n_edges x2, flags[2], overflow, n_queries
    size_t h_chain_cap = 0;      // frames per slot
    // the chain of a slot as an instantiated CUDA graph (re-captured when any launch parameter or scratch pointer changes)
    struct ChainGraphKey { int nF, cap, mono, cont, K, prev_valid; float th, th_local, nn_local, fx, fy, cx, cy, bf, bounds[4]; unsigned long long generation; };
    cudaGraphExec_t chain_exec[2] = {};
    ChainGraphKey chain_key[2] = {};
    const void* chain_timing_ev = nullptr;   // RGBL_CHAIN_TIMING development aid

    // staged input slots of the sequence runners (rgbl_resident_stage / rgbl_track_sequence, rgbl_resident_stage_rgbd /
    // rgbl_track_sequence_rgbd): level-0 planes + clouds (RGB-L) or uint16 depth planes (RGB-D) of whole batches
    static constexpr int kMaxStageSlots = 8;
    struct StageSlot { uint8_t* img = nullptr; float* pts = nullptr; int* n_pts = nullptr; uint16_t* depth = nullptr; std::vector<int> h_n_pts; int n_frames = 0, max_pts = 0; bool rgbd = false; };
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
    int resident_frames = 0, resident_max_pts = 0;
    bool resident_rgbd = false;  // the uploaded frames are RGB-D frames (image + depth plane), not RGB-L ones
    bool blur_valid = false;
};

// returns the context's mapping arena with at least `bytes` bytes (nullptr on allocation failure)
inline char* mapping_arena(Ctx* c, size_t bytes) {
    if (bytes > c->map_arena_cap) {
        if (c->map_arena) cudaFree(c->map_arena);
        c->map_arena = nullptr; c->map_arena_cap = 0;
        const size_t want = bytes + bytes / 4 + (1 << 20);
        if (cudaMalloc((void**)&c->map_arena, want) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        c->map_arena_cap = want;
    }
    return c->map_arena;
}

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

}  // namespace rgbl
#endif
