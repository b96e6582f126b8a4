// Kernel launchers (defined in the .cu files) and the device-side record types.
#ifndef RGBL_KERNELS_H
#define RGBL_KERNELS_H

#include <cuda_runtime.h>

#include <string>

#include "rgbl_internal.h"

namespace rgbl {

// Selected keypoint handed from the quad-tree to the describe kernel (level coordinates, +16 applied).
struct __align__(8) SelKp {
    uint16_t x, y;
    uint8_t level, score;
    uint16_t pad;
};

#if defined(__CUDACC__)
__device__ __forceinline__ uint32_t pack_cand_dev(int x, int y, int s) {
    return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)s << 24);
}
#endif

// orb_kernels.cu
void launch_pyramid(cudaStream_t st, uint8_t* pyr, size_t frame_stride, const LevelGeom* h_levels, int n_levels,
                    const LinCoef* d_coefs, int n_frames);
void launch_fast(cudaStream_t st, const uint8_t* pyr, size_t frame_stride, const LevelGeom* d_levels,
                 const CellInfo* d_cells, int n_cells, int ini_th, int min_th, uint32_t* slots, int* counts,
                 int* overflow, int n_frames);
// fast_strip_kernels.cu: strip formulation of launch_fast (same outputs); returns -1 when the shared-memory request is refused
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
void launch_describe(cudaStream_t st, const uint8_t* pyr, const uint8_t* blur, size_t frame_stride,
                     const LevelGeom* d_levels, const SelKp* sel, const int* n_sel, int cap, int max_n,
                     const int umax[16], rgbl_keypoint* kps, uint8_t* desc, int n_frames);
// describe_warp_kernels.cu: launch_describe with the pixel neighbourhoods staged in shared memory (same outputs)
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
                    int* status, SelKp* sel, int* n_sel, int n_frames, int max_nodes = 1024);      // max_nodes: largest max(quota + 3, 4 nIni) over the levels
int quadtree_block_host(const uint32_t* cand, int n, int width, int height, int N, uint32_t* out, int out_cap, int block_sort = 0);

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
void launch_depth_resolve_dilate(cudaStream_t st, const float* pts, int pts_stride, const int* n_pts,
                                 const DepthDev& prm, int W, int H, const uint32_t* idx_map, uint32_t stamp,
                                 float* raw, float* processed, int n_frames);
// depth_dilate_v2.cu: same outputs; empty tiles skip the structuring-element loop, taps as shared-memory offsets
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
void launch_search_last(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, const LastFrameDev& lf,
                        const SearchLastParams& prm, MatchScratch s, uint8_t* state, int* match, int* n_matches,
                        const ChainEdgesOut* edges = nullptr);
struct LocalRingDev;
struct ChainTlmTail;                 // below (chain_kernels.cu section): TrackLocalMap tail of the resolution kernel
void launch_search_local(cudaStream_t st, const FrameDev& f, const int* cell_start, const int* csr_idx, const LocalPointsDev& lp,
                         const SearchLocalParams& prm, MatchScratch s, uint8_t* state, int* match, int* n_matches, const ChainTlmTail* tail = nullptr);
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
void launch_chain_prep(cudaStream_t st, const ChainPrepDev& cp, const float* last_pose);
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
void launch_tlm_prepare(cudaStream_t st, const FrameDev& f, const float* pose, const LocalRingDev& ring, float cos_limit, const int* n_edges,
                        const int* e_idx, const uint8_t* e_outlier, uint8_t* state, int* match_last, const LocalQueriesDev& lq, int* lookback, int* fail);
// TrackLocalMap tail of the local search's resolution kernel (match_kernels.cu): the edge list of the second PoseOptimization from (inliers
// of the first search) + (local matches), and the hand-over of the last frame's points into the ring.  *n_local_matches is written.
struct ChainTlmTail {
    const int* match_last; const float* last_xw; const float* lq_xw; LocalRingDev ring; ChainEdgesOut edges; int* n_local_matches;
    int n_last_cap; const uint8_t* last_valid; const int* last_octave; const uint8_t* last_desc; const float* last_pose;
};
// tlm_prepare compacts over several CTAs in one launch; `lookback` = tlm_lookback_ints() ZERO-INITIALISED ints (the kernel leaves them zero),
// `fail` = a device flag set to 9 if a CTA ever waited in vain
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
    int W, H;
    const uint8_t* src; size_t src_stride; int src_pitch;            // raw plane of slot s at src + s * src_stride
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
void launch_pose_optimize(cudaStream_t st, const PoseProblemDev& p, double* work /* n*4 doubles */, uint8_t* level, uint8_t* outlier,
                          float* pose_out /*7*/, int* n_inliers, const ChainPrepDev* next = nullptr);

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

}  // namespace rgbl
#endif
