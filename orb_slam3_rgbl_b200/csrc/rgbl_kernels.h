// Kernel launchers (defined in the .cu files) and the device-side record types.
#ifndef RGBL_KERNELS_H
#define RGBL_KERNELS_H

#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <type_traits>

#include "rgbl_internal.h"

namespace rgbl {

// Selected keypoint handed from the quad-tree to the describe kernel (level coordinates, +16 applied).
struct __align__(8) SelKp {
    uint16_t x, y;
    uint8_t level, score;
    uint16_t pad;
};

// orb_kernels.cu
void launch_pyramid(cudaStream_t st, uint8_t* pyr, size_t frame_stride, const LevelGeom* h_levels, int n_levels,
                    const LinCoef* d_coefs, int n_frames);
// cv::resize(INTER_LINEAR) of n_planes 8-bit planes, src.w x src.h -> dst.w x dst.h with the tables tabx / taby (linear_coefs): plane z at
// src_base + z * src_stride + src.off -> dst_base + z * dst_stride + dst.off; both rows 64-byte aligned (pitch % 64 == 0, 16-byte aligned bases).
// ch 3 / 4: the source planes are interleaved colour images (src.pitch in bytes), resized per channel and converted to gray (gray_of, channel 0
// weighted w0, rgbl_device.cuh) into the 8-bit destination planes
void launch_resize_planes(cudaStream_t st, const uint8_t* src_base, size_t src_stride, const LevelGeom& src, uint8_t* dst_base, size_t dst_stride,
                          const LevelGeom& dst, const LinCoef* tabx, const LinCoef* taby, int n_planes, int ch = 1, int w0 = 0);
// cvtColor to gray of n_planes interleaved colour planes of ch (3 / 4) bytes per pixel, dst.w x dst.h, laid out as for launch_resize_planes
void launch_gray_planes(cudaStream_t st, const uint8_t* src_base, size_t src_stride, const LevelGeom& src, uint8_t* dst_base, size_t dst_stride,
                        const LevelGeom& dst, int ch, int w0, int n_planes);
// fast_strip_kernels.cu: per-cell FAST with the iniTh -> minTh fallback, one CTA per strip of cells (fast_strip.cuh); survivors in
// each cell's slot array; returns -1 when the shared-memory request is refused
int launch_fast_strips(cudaStream_t st, const uint8_t* pyr, size_t frame_stride, const LevelGeom* d_levels, const CellInfo* d_cells,
                       int n_cells, const StripInfo* d_strips, int n_strips, int rows_cap, int list_cap, int ini_th, int min_th,
                       uint32_t* slots, int* counts, int* overflow, int n_frames);
void launch_compact(cudaStream_t st, const LevelGeom* d_levels, int n_levels, int n_cells, const uint32_t* slots,
                    const int* counts, int* cell_off, int* level_cnt, int* frame_total, uint32_t* dense, int dense_cap,
                    int* overflow, int n_frames);
// png_kernels.cu: cv::imread of PNG streams (host: chunks + zlib inflate; device: scanline reconstruction + cvtColor to gray) -----------
// depth16: the streams are depth images (16-bit gray only, 2 bytes per pixel); else images (8-bit gray / RGB / RGBA)
int png_inflate_batch(int n_frames, const uint8_t* const* png, const size_t* png_bytes, int w, int h, uint8_t* h_raw, size_t raw_stride, int* ch_out,
                      std::string& err, bool depth16 = false);
void launch_png_unfilter_gray(cudaStream_t st, const uint8_t* d_raw, size_t raw_stride, int w, int h, int channels, int camera_rgb, uint8_t* pyr,
                              size_t frame_stride, const LevelGeom& l0, uint32_t* band_rows, int* status, int n_frames);
// the same reconstruction of 3 / 4-channel streams with the pixels' bytes stored as they are (the file's R, G, B(, A) order) in colour planes:
// frame f at dst + f * dst_stride, rows of `pitch` bytes (a multiple of 4)
void launch_png_unfilter_pixels(cudaStream_t st, const uint8_t* d_raw, size_t raw_stride, int w, int h, int channels, uint8_t* dst, size_t dst_stride,
                                int pitch, uint32_t* band_rows, int* status, int n_frames);
// 16-bit depth PNG scanlines (ch = 2) -> uint16 depth planes (frame f at depth + f * frame_elems, row pitch pitch_elems, pitch a multiple of 32)
void launch_png_unfilter_depth16(cudaStream_t st, const uint8_t* d_raw, size_t raw_stride, int w, int h, uint16_t* depth, size_t frame_elems,
                                 size_t pitch_elems, uint32_t* band_rows, int* status, int n_frames);
// level_tma_kernels.cu: fused per-level TMA tile kernel (blur of level l + level l+1 from one read of level l) -----------------------
struct LevelTensorMaps { alignas(64) unsigned char map[RGBL_MAX_LEVELS][128]; int n_levels; };     // raw CUtensorMap objects, one per level
int make_level_tensor_maps(uint8_t* pyr, size_t frame_stride, int n_slots, const LevelGeom* levels, int n_levels, LevelTensorMaps* out);
int launch_level_tiles(cudaStream_t st, const LevelTensorMaps& tms, uint8_t* pyr, uint8_t* blur, size_t frame_stride, const LevelGeom* h_levels,
                       int n_levels, const LinCoef* d_coefs, int n_frames);
void launch_blur(cudaStream_t st, const uint8_t* pyr, uint8_t* blur, size_t frame_stride, const LevelGeom* h_levels,
                 int n_levels, int n_frames);
// describe_warp_kernels.cu: orientation + rBRIEF descriptor + keypoint record, one warp per selected keypoint with its pixel
// neighbourhoods staged in shared memory (describe_warp.cuh)
void launch_describe_staged(cudaStream_t st, const uint8_t* pyr, const uint8_t* blur, size_t frame_stride, const LevelGeom* d_levels,
                            const SelKp* sel, const int* n_sel, int cap, int max_n, const int umax[16], rgbl_keypoint* kps, uint8_t* desc,
                            int n_frames);
void launch_padded_level(cudaStream_t st, const uint8_t* pyr, size_t frame_stride, int frame, const LevelGeom& lg,
                         uint8_t* dst, int dst_pitch);

// quadtree_kernels.cu
struct QtScratchDev { unsigned short *perm_a, *perm_b, *node_a, *node_b; unsigned long long* scan; unsigned char* quad; };      // 16-bit key / node indices (quadtree_block.cuh: KeyIdx)
int quadtree_smem_bytes();
int launch_quadtree(cudaStream_t st, const uint32_t* dense, const int* level_cnt, const int* frame_total, const LevelGeom* d_levels,
                    int n_levels, const QtScratchDev& scr, uint32_t* sel_lvl, int* n_sel_lvl, const int* lvl_region, int cap_kp,
                    int* status, SelKp* sel, int* n_sel, int n_frames, int max_nodes = 1024,      // max_nodes: largest max(quota + 3, 4 nIni) over the levels
                    int dense_cap = 0x7fffffff);      // entries of `dense`: the counts may run past it after a flagged candidate-buffer overflow
int quadtree_block_host(const uint32_t* cand, int n, int width, int height, int N, uint32_t* out, int out_cap);

// depth_kernels.cu
struct DepthDev {
    float P[12];
    float min_dist, max_dist, bf, inv_scale_m;   // inv_scale_m = max_dist * ScaleFactor (the inversion constant M)
    int ku, kv;
    uint8_t mask[81];
    int method, avg_kernel;          // rgbl_depth_method, AverageFiltering kernel size
    float nn_radius;                 // NearestNeighborPixel SearchDistance
};
// raw KITTI records (x, y, z, reflectance) x n -> planar rows x | y | z | 1 (frame stride pts_stride floats in both buffers)
void launch_deinterleave_xyzr(cudaStream_t st, const float* raw, float* pts, int pts_stride, const int* n_pts, int max_n_pts, int n_frames);
void launch_depth_project(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts, int max_n_pts,
                          const DepthDev& prm, int W, int H, uint32_t* idx_map, uint32_t stamp, int n_frames);
// depth_dilate_v2.cu: depth of each pixel's winning point (raw, nullable) and its inverse dilation by the structuring element of prm
// (processed); empty tiles skip the structuring-element loop, taps as shared-memory offsets
void launch_depth_resolve_dilate_v2(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts, const DepthDev& prm, int W, int H,
                                    const uint32_t* idx_map, uint32_t stamp, float* raw, float* processed, int n_frames);
void launch_depth_average_filter(cudaStream_t st, const float* raw, int W, int H, int k, float* processed, int n_frames);
void launch_depth_nn_pixel(cudaStream_t st, const float* raw, int W, int H, const rgbl_keypoint* kps, const rgbl_keypoint* kps_un,
                           const int* n_kp, int cap, int max_n, float bf, float R, float* depth, float* uright, int n_frames);
void launch_depth_gather(cudaStream_t st, const float* processed, int W, int H, const rgbl_keypoint* kps,
                         const rgbl_keypoint* kps_un, const int* n_kp, int cap, int max_n, float bf, float* depth,
                         float* uright, int n_frames);
// Frame::UndistortKeyPoints (src/Frame.cc:837-869) of n_frames keypoint lists ([n_frames][cap], n_kp[frame] valid): kps_un = kps with pt
// replaced by the undistorted point (undistort_point, rgbl_device.cuh)
void launch_undistort_keypoints(cudaStream_t st, const UndistortDev& cam, const rgbl_keypoint* kps, const int* n_kp, int cap, int max_n,
                                rgbl_keypoint* kps_un, int n_frames);
// the same gather on uint16 RGB-D depth planes, metric depth = (float)sample * scale (Tracking::mDepthMapFactor)
void launch_depth_gather_u16(cudaStream_t st, const uint16_t* plane, size_t frame_elems, size_t pitch_elems, float scale, const rgbl_keypoint* kps,
                             const rgbl_keypoint* kps_un, const int* n_kp, int cap, int max_n, float bf, float* depth, float* uright, int n_frames);
// cv::resize(INTER_LINEAR) of n_frames CV_16U depth planes by integer factors kx = src_w / dst_w, ky = src_h / dst_h (OpenCV's float path:
// weights 1 - f, f with f in {0, 1/2}, horizontal then vertical in float32, rounded half to even): src plane f at src + f * src_frame_elems with
// row pitch src_pitch elements -> dst + f * dst_frame_elems, row pitch dst_pitch elements
void launch_resize_depth16(cudaStream_t st, const uint16_t* src, size_t src_frame_elems, size_t src_pitch, int kx, int ky, uint16_t* dst,
                           size_t dst_frame_elems, size_t dst_pitch, int dst_w, int dst_h, int n_frames);


// match_kernels.cu ---------------------------------------------------------------------------------
// Device view of the Frame members the matchers read (Nleft == -1 frames).
struct FrameDev {
    const int* n;                    // device int: number of keypoints
    const rgbl_keypoint* keys;       // mvKeysUn
    const float* uright;             // mvuRight
    const uint8_t* desc;             // mDescriptors
    float min_x, max_x, min_y, max_y, inv_w, inv_h;
    int n_levels;
    float scale[RGBL_MAX_LEVELS];
    float fx, fy, cx, cy, bf, mb, log_scale_factor;
};
struct LastFrameDev {                // LastFrame.mvpMapPoints as flat arrays (device pointers)
    int n;
    const uint8_t* valid; const float* xw; const uint8_t* desc; const int* octave; const float* angle; const uint8_t* obs_pos;
};
struct LocalPointsDev {              // vpMapPoints with the mTrack* fields isInFrustum fills
    int n;                           // query capacity of the launch; n_dev (if non-null) = the number of queries, read on the device
    const int* n_dev;
    const uint8_t* in_view; const float *proj_x, *proj_y, *proj_xr, *depth; const int* level; const float* view_cos;
    const uint8_t* desc; const uint8_t* obs_pos;
};
struct SearchLastParams { float cur_pose[7]; float th; int forward, backward, check_orientation; const float* cur_pose_dev; const int* flags_dev; };
struct SearchLocalParams { float th, nn_ratio, th_far; int use_factor, far_points, keep_max; };
struct RelocPointsDev { int n; const uint8_t* valid; const float* xw; const uint8_t* desc; const float* angle; const float *mf_min, *mf_max; };
struct SearchRelocParams { float cur_pose[7]; float Ow[3]; float th; int orb_dist, check_orientation; };
struct FrustumParams { float Rcw[9], tcw[3], Ow[3], cos_limit; };
struct MatchScratch {                 // device scratch of the matchers (match_kernels.cu)
    unsigned long long* lists; uint16_t* slots; int list_cap; int* list_n;     // per-query staging lists: 64-bit entries (MatchEntry) + inverse-list slots
    unsigned long long* dense; uint16_t* dense_slot; int* dense_q; int* base;   // all finished lists appended to one run, base[q] = start of query q
    int* total;                      // entries in the run: ZERO between launches (resolve_kernel clears it)
    int* inv_cnt;                    // per frame feature: entries listing it: ZERO between launches (resolve_kernel clears what it read)
    int* minq; int* choice; uint8_t* resolved; int* overflow; int* rounds;
};

// Sequence lanes (rgbl_set_sequences): every launch of the resident chain serves S independent sequences, lane s = blockIdx.y (the pose
// kernel: cluster s along y).  Each pointer-bearing argument of the chain's kernels is a Laned<T>: lane s's value is base + s * step, word
// by word (64-bit, wrapping).  The lanes' buffers are equally spaced (rgbl_ctx.h: ChainLaneStrides), so a pointer's step is its lane
// stride in bytes and every other field, the same in all lanes, has step zero.  A plain T converts to one lane (step zero).
constexpr int kMaxLanes = 16;
template <class T> struct Laned {
    static_assert(sizeof(T) % 8 == 0 && alignof(T) >= 8, "Laned<T>: T is made of 64-bit words");
    T base, step;
    Laned() : base(), step() {}
    Laned(const T& v) : base(v), step() {}
    Laned(const T& b, const T& st) : base(b), step(st) {}
};
template <class T> __host__ __device__ __forceinline__ T lane_value(const Laned<T>& a, unsigned s) {
    T r;
#pragma unroll
    for (size_t i = 0; i < sizeof(T) / 8; ++i) {
        unsigned long long b, d;
        memcpy(&b, reinterpret_cast<const char*>(&a.base) + 8 * i, 8);
        memcpy(&d, reinterpret_cast<const char*>(&a.step) + 8 * i, 8);
        b += (unsigned long long)s * d;
        memcpy(reinterpret_cast<char*>(&r) + 8 * i, &b, 8);
    }
    return r;
}
// lane s's argument inside a kernel instantiated for kLanes; a one-lane launch (kLanes false) reads the argument itself, as a kernel
// without lanes would
template <bool kLanes, class T> __device__ __forceinline__ auto lane_arg(const Laned<T>& a, unsigned s) -> typename std::conditional<kLanes, T, const T&>::type {
    if constexpr (kLanes) return lane_value(a, s); else return a.base;
}
// Set (never cleared here) when laned_of met lanes that are not base + s * step.  enqueue_chain fails the chain with it; a captured chain
// (the default) is then never instantiated, so none of its launches runs.
inline bool& lane_layout_broken() { static thread_local bool broken = false; return broken; }
// host: the Laned<T> of the lanes make(s) builds (make(1) - make(0) word by word; make(0) alone when the launch has one lane).  Every lane
// s >= 2 is checked against base + s * step in the low 32 bits of each word: all of a pointer's offset and every 4-byte field that starts a
// word, while the high half of a word may be the padding after such a field, whose bytes are unspecified.
template <class F> inline auto laned_of(int lanes, F make) -> Laned<decltype(make(0))> {
    using T = decltype(make(0));
    const T b = make(0);
    if (lanes < 2) return Laned<T>(b);
    const T o = make(1);
    T d;
    for (size_t i = 0; i < sizeof(T) / 8; ++i) {
        unsigned long long x, y;
        memcpy(&x, reinterpret_cast<const char*>(&o) + 8 * i, 8);
        memcpy(&y, reinterpret_cast<const char*>(&b) + 8 * i, 8);
        x -= y;
        memcpy(reinterpret_cast<char*>(&d) + 8 * i, &x, 8);
    }
    const Laned<T> r(b, d);
    for (int s = 2; s < lanes; ++s) {
        const T want = make(s), got = lane_value(r, (unsigned)s);
        for (size_t i = 0; i < sizeof(T) / 8; ++i) {
            unsigned long long x, y;
            memcpy(&x, reinterpret_cast<const char*>(&want) + 8 * i, 8);
            memcpy(&y, reinterpret_cast<const char*>(&got) + 8 * i, 8);
            if ((uint32_t)x != (uint32_t)y) lane_layout_broken() = true;
        }
    }
    return r;
}

void prepare_match_kernels();
// true while the resident chain enqueues its kernels: the chain launchers then add the programmatic-stream-serialization attribute (PDL, see
// pdl_wait in rgbl_device.cuh).  Thread-local, set and cleared by chain_begin (api_track.cu).
inline bool& chain_launch_pdl() { static thread_local bool on = false; return on; }
// kernel launch with or without that attribute
template <class... KArgs, class... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
void launch_grid_build(cudaStream_t st, const FrameDev& f, int* cell_start, int* csr_idx, int* kp_cell);
// one CTA per frame: frame b reads f.n[b], f.keys + b * kp_stride and writes cell_start + b * (cells + 1), csr_idx / kp_cell + b * kp_stride
void launch_grid_build_batch(cudaStream_t st, const FrameDev& f, int n_frames, int kp_stride, int* cell_start, int* csr_idx, int* kp_cell);
// edges != nullptr: the resolution kernel also writes the matched features as PoseOptimization edges (resident tracking chain)
struct ChainEdgesOut { float* exw; float* eobs; float* einfo; uint8_t* est; int* eidx; int* n_edges; };
// The chain's launchers take `lanes` sequence lanes (grid y); a plain argument is one lane.
void launch_search_last(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const int*>& cell_start, const Laned<const int*>& csr_idx,
                        const Laned<LastFrameDev>& lf, const Laned<SearchLastParams>& prm, const Laned<MatchScratch>& s, const Laned<uint8_t*>& state,
                        const Laned<int*>& match, const Laned<int*>& n_matches, const Laned<ChainEdgesOut>* edges = nullptr, int lanes = 1);
struct LocalRingDev;
struct ChainTlmTail;                 // below (chain_kernels.cu section): TrackLocalMap tail of the resolution kernel
void launch_search_local(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const int*>& cell_start, const Laned<const int*>& csr_idx,
                         const Laned<LocalPointsDev>& lp, const SearchLocalParams& prm, const Laned<MatchScratch>& s, const Laned<uint8_t*>& state,
                         const Laned<int*>& match, const Laned<int*>& n_matches, const Laned<ChainTlmTail>* tail = nullptr, int lanes = 1);
void launch_search_bow(cudaStream_t st, const FrameDev& f, int n_q, const int* q_feat, const int* q_cbeg, const int* q_cend,
                       const uint8_t* kf_desc, const uint8_t* f_desc, const float* q_angle, const float* f_angle, const int* f_node_feat,
                       float nn_ratio, int keep_max, int check_orientation, const uint8_t* obs_pos, MatchScratch s, uint8_t* state, int* match,
                       int* n_matches);
void launch_search_reloc(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, const RelocPointsDev& rp,
                         const SearchRelocParams& prm, const uint8_t* obs_pos, MatchScratch s, uint8_t* state, int* match, int* n_matches);
void launch_fuse_search(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, int n, const uint8_t* valid, const float* xw,
                        const float* normal, const float* mf_min, const float* mf_max, const uint8_t* desc, const float* Tcw /*7, device*/,
                        const float* Ow /*3, device*/, float th, int* best_idx, int* best_dist);
// ChainPrepDev (rgbl_device.cuh): unprojection of one frame's LiDAR-depth keypoints with its pose = the map points of the next search
struct ChainPrepDev;
void launch_chain_prep(cudaStream_t st, const Laned<ChainPrepDev>& cp, const Laned<const float*>& last_pose, int lanes = 1);
void launch_frustum(cudaStream_t st, const FrameDev& f, const FrustumParams& prm, int n, const float* xw, const float* normal,
                    const float* mf_min, const float* mf_max, uint8_t* in_view, float* px, float* py, float* pxr, float* depth,
                    int* level, float* view_cos);

// chain_kernels.cu: TrackLocalMap half of the resident tracking chain ----------------------------------
struct LocalRingDev {                // local map of the chain: K frame slots x cap points, slot = frames inserted so far mod K
    int K, cap;
    uint8_t* valid; float* xw; float* normal; float* mf_min; float* mf_max; uint8_t* desc;
    int* count;                      // frames inserted so far (device)
};
struct LocalQueriesDev {             // the in-frustum local map points, compacted in ring order (= vpMapPoints of the local search)
    int cap; int* n;
    uint8_t* in_view; uint8_t* obs_pos; float *proj_x, *proj_y, *proj_xr, *depth; int* level; float* view_cos; uint8_t* desc; int* src;
    float* xw;                       // world coordinates of the compacted points (read by the edge-list tail instead of the ring)
};
// lanes: one compaction per lane (grid y), lane s's look-back slots at lookback + s * tlm_lookback_ints()
void launch_tlm_prepare(cudaStream_t st, const Laned<FrameDev>& f, const Laned<const float*>& pose, const Laned<LocalRingDev>& ring, float cos_limit,
                        const Laned<const int*>& n_edges, const Laned<const int*>& e_idx, const Laned<const uint8_t*>& e_outlier, const Laned<uint8_t*>& state,
                        const Laned<int*>& match_last, const Laned<LocalQueriesDev>& lq, int* lookback, const Laned<int*>& fail, int lanes = 1);
// TrackLocalMap tail of the local search's resolution kernel (match_kernels.cu): the edge list of the second PoseOptimization from (inliers
// of the first search) + (local matches), and the hand-over of the last frame's points into the ring.  *n_local_matches is written.
struct ChainTlmTail {
    const int* match_last; const float* last_xw; const float* lq_xw; LocalRingDev ring; ChainEdgesOut edges; int* n_local_matches;
    int n_last_cap; const uint8_t* last_valid; const int* last_octave; const uint8_t* last_desc; const float* last_pose;
};
// tlm_prepare compacts over several CTAs in one launch; `lookback` = tlm_lookback_ints() ZERO-INITIALISED ints (the kernel leaves them zero),
// `fail` = a device flag set to kTlmWaitFailed if a CTA ever waited in vain
constexpr int kTlmWaitFailed = 9;
int tlm_lookback_ints();

// stereo_kernels.cu --------------------------------------------------------------------------------
// Frame::ComputeStereoMatches for n_pairs pairs of frame slots of one batched extraction: pair p = (left slot l0 + p, right slot r0 + p).
// Keypoints, descriptors and counts are the batch's [slot][cap] outputs; mvDepth / mvuRight of the left slot are written in place.
struct StereoBatchDev {
    const uint8_t* pyr; size_t frame_stride; const LevelGeom* levels;
    const rgbl_keypoint* kps; const uint8_t* desc; const int* n_sel; int cap;
    int l0, r0, n_rows;
    float scale[RGBL_MAX_LEVELS], inv_scale[RGBL_MAX_LEVELS];
    float mb, mbf;
    float* depth; float* uright;
    // scratch, per pair: row_start [n_rows + 1] (vRowIndices as CSR), row_idx [idx_cap], sad [cap]
    int* row_start; int* row_idx; int idx_cap; int* sad;
};
// row_idx entries one pair needs at most: a right keypoint of octave o is listed in ceil(y + r) - floor(y - r) + 1 <= 2r + 4 rows, r = 2 scale[o]
int stereo_row_index_cap(int cap, const float* scale, int n_levels, int n_rows);
void launch_stereo_matches(cudaStream_t st, const StereoBatchDev& s, int n_pairs);

// stereo_kernels.cu, rectification: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of stereo pairs with fixed-point maps -----------------
// maps = [m1l | m2l | m1r | m2r] (H x W floats each) -> per camera (left 0, right 1) H rows of `pitch` (a multiple of 4) entries:
// xy = sx | sy << 16 (int16 each), a = ay * 32 + ax
void launch_rectify_maps(cudaStream_t st, const float* maps, int W, int H, uint32_t* xy, uint16_t* a, int pitch);
struct RectifyDev {
    const uint32_t* xy; const uint16_t* a; int map_pitch;
    int W, H;                                                        // output (and map) size: the context's
    int src_W, src_H;                                                // raw plane size: the input resize's source size (0, 0: W x H)
    const uint8_t* src; size_t src_stride; int src_pitch;            // raw plane of slot s at src + s * src_stride
    int ch, w0;                                                      // ch 3 / 4: colour raw planes, remapped per channel, then gray_of(w0); else 8-bit
    uint8_t* dst; size_t dst_stride; int dst_off, dst_pitch;         // rectified plane of slot s at dst + s * dst_stride + dst_off (4-byte aligned rows)
};
// slots [0, n_pairs) through the left camera's map, [n_pairs, 2 n_pairs) through the right camera's, in one launch
void launch_rectify(cudaStream_t st, const RectifyDev& r, int n_pairs);

// pose_kernels.cu ----------------------------------------------------------------------------------
struct PoseProblemDev {
    int n;                           // edges (keypoint order)
    const int* n_dev;                // if non-null: edge count read on the device
    const float* pose_in_dev;        // if non-null: initial pose read on the device
    const float* xw; const float* obs; const float* inv_sigma2; const uint8_t* stereo;
    float fx, fy, cx, cy, bf;
    float pose_in[7];
};
// nullptr when `device` can run pose_optimize_kernel's cluster (and the non-portable size is opted in), else why it cannot;
// callers check it before launch_pose_optimize
const char* pose_cluster_unsupported(int device);
// next != nullptr: after the pose is final the kernel also runs the chain preparation of the NEXT frame's search with it
// lanes: one cluster per lane (cluster s = CTAs [0, kPoseCtas) x {s})
void launch_pose_optimize(cudaStream_t st, const Laned<PoseProblemDev>& p, const Laned<double*>& work /* n*4 doubles */, const Laned<uint8_t*>& level,
                          const Laned<uint8_t*>& outlier, const Laned<float*>& pose_out /*7*/, const Laned<int*>& n_inliers,
                          const Laned<ChainPrepDev>* next = nullptr, int lanes = 1);
// clusters of pose_optimize_kernel the device holds at once (cudaOccupancyMaxActiveClusters; 0: the query failed)
int pose_max_active_clusters(int device);

// bow_kernels.cu ------------------------------------------------------------------------------------
struct VocabDev {                    // DBoW2 vocabulary, flattened (node 0 = root)
    const int* child_begin;          // n_nodes + 1
    const int* child_index;          // children in m_nodes[i].children order
    const uint8_t* node_desc;        // n_nodes x 32
    const double* node_weight;       // WordValue
    const int* word_id;              // >= 0 for leaves
};
void launch_bow_descend(cudaStream_t st, const VocabDev& voc, int n, const uint8_t* desc, int nid_level, int* f_word, double* f_weight,
                        int* f_node);
// returns the padded key count (power of two) or -1 when n exceeds the shared-memory sort capacity
int launch_bow_assemble(cudaStream_t st, int n, const int* f_word, const double* f_weight, const int* f_node, int* bow_word,
                        double* bow_value, int* fv_node, int* fv_start, int* fv_feature, int* counts /*3*/, int* scratch);

// ba_factor.cu --------------------------------------------------------------------------------------
// S x = bp - coef for the reduced camera system of bundle adjustment (S: n x n doubles, n = 6 n_opt, lower triangle, factored in place;
// work: n doubles).  by_size: the one-CTA kernel up to kSingleCtaMaxOpt free poses, the tiled multi-CTA factorisation above.
// status[0] = 1 and x = 0 on a non-positive or non-finite pivot, else 0.  Returns the number of launches.
enum class BaSolvePath { by_size, single_cta, tiled };
constexpr int kSingleCtaMaxOpt = 64;
int ba_solve_reduced(cudaStream_t st, int n, double* S, const double* bp, const double* coef, double* x, double* work, int* status,
                     BaSolvePath path = BaSolvePath::by_size);

}  // namespace rgbl
#endif
