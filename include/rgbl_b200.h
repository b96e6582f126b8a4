/*
 * rgbl_b200 — C ABI of the H100-native (sm_90a) per-frame front end for ORB-SLAM3-RGBL.
 *
 * The reference has no FFI; its boundary is four C++ classes (SURVEY.md §8(b)).  Each entry point
 * below names the reference method it replaces (paths relative to the reference root).  A thin C++
 * shim with the reference's class signatures (shim/, see INTEGRATION.md) marshals cv::Mat /
 * std::vector<cv::KeyPoint> to these flat buffers.
 *
 * Conventions: plain C types; caller-allocated outputs with explicit capacities; return 0 on
 * success, negative rgbl_status on error (rgbl_last_error() gives the text); all pointers are HOST
 * pointers unless the name ends in _dev; a context is bound to one CUDA device and owns its
 * streams; calls on one context are serialised by the caller (one context per tracking thread /
 * per camera, as the reference uses one ORBextractor per camera: src/Frame.cc:122-125).
 * There is NO CPU fallback: without a usable CUDA device rgbl_create fails with RGBL_E_CUDA.
 */
#ifndef RGBL_B200_H
#define RGBL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RGBL_MAX_LEVELS 16
#define RGBL_DESC_BYTES 32

typedef enum {
    RGBL_OK = 0,
    RGBL_E_INVALID = -1,     /* bad argument */
    RGBL_E_CUDA = -2,        /* CUDA runtime/driver error (no device, launch failure, ...) */
    RGBL_E_CAPACITY = -3,    /* an output or internal buffer was too small; nothing silently dropped */
    RGBL_E_EMPTY = -4,       /* empty image: ORBextractor::operator() returns -1 (src/ORBextractor.cc:1090) */
    RGBL_E_UNSUPPORTED = -5
} rgbl_status;

typedef struct rgbl_ctx rgbl_ctx;

/* cv::KeyPoint memory layout (28 bytes): pt.x, pt.y, size, angle, response, octave, class_id. */
typedef struct {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} rgbl_keypoint;

/* ORBextractor constructor arguments, include/ORBextractor.h:48-49, src/ORBextractor.cc:409-469. */
typedef struct {
    int32_t nfeatures;
    float scale_factor;
    int32_t nlevels;
    int32_t ini_th_fast;
    int32_t min_th_fast;
} rgbl_orb_params;

/* DepthModule parameters parsed from the YAML, src/DepthModule.cc:281-601. */
typedef enum {
    RGBL_DEPTH_NONE = 0,
    RGBL_DEPTH_NEAREST_NEIGHBOR_PIXEL = 1,
    RGBL_DEPTH_AVERAGE_FILTERING = 2,
    RGBL_DEPTH_INVERSE_DILATION = 3
} rgbl_depth_method;                          /* include/DepthModule.h:33-39 */

typedef struct {
    int32_t method;                            /* rgbl_depth_method */
    float min_dist, max_dist;                  /* LiDAR.min_dist / LiDAR.max_dist */
    float bf;                                  /* Camera.bf */
    float inv_dilation_scale;                  /* ParamUpsampling_InverseDilation_ScaleFactor (1.0) */
    int32_t ku, kv;                            /* structuring element size (u = columns, v = rows) */
    uint8_t mask[81];                          /* 0/1 structuring element, row-major kv x ku (<= 9x9) */
    int32_t avg_kernel;                        /* AverageFiltering kernel size */
    float nn_search_radius;                    /* NearestNeighborPixel search distance */
} rgbl_depth_params;

typedef struct {
    int32_t device;          /* CUDA device ordinal */
    int32_t width, height;   /* image size all frames of this context share */
    int32_t max_batch;       /* frames processed per batched call (>= 1) */
    int32_t max_points;      /* LiDAR points per frame capacity */
    int32_t max_candidates;  /* FAST candidates per frame capacity; 0 = default */
    rgbl_orb_params orb;
} rgbl_config;

/* ---- lifetime ------------------------------------------------------------------------------- */
int rgbl_create(const rgbl_config* cfg, rgbl_ctx** out);
void rgbl_destroy(rgbl_ctx* ctx);
const char* rgbl_last_error(const rgbl_ctx* ctx);     /* ctx may be NULL: error of the last failed rgbl_create */
int rgbl_abi_version(void);
/* Upper bound of keypoints one frame can yield (sum over levels of max(quota+3, 4*nIni)); size kps/desc with it. */
int rgbl_keypoint_capacity(const rgbl_ctx* ctx);

/* Tables computed by ORBextractor::ORBextractor (src/ORBextractor.cc:409-469) and exposed through
 * GetScaleFactors()/GetInverseScaleFactors()/... (include/ORBextractor.h:61-81).  Host-only. */
int rgbl_orb_tables(const rgbl_orb_params* p, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                    int32_t* features_per_level, int32_t* umax16);

/* ---- ORBextractor::operator() (include/ORBextractor.h:57-59, src/ORBextractor.cc:1086-1168) ---- *
 * gray: CV_8UC1 host image.  kps/desc: capacity `cap` entries (cap >= rgbl_keypoint_capacity(ctx)
 * is always sufficient).  lap0/lap1 = vLappingArea.  *mono_index = the return value of
 * the reference operator().  Returns RGBL_E_EMPTY for an empty image.                               */
int rgbl_orb_extract(rgbl_ctx* ctx, const uint8_t* gray, int width, int height, int stride, int lap0, int lap1,
                     rgbl_keypoint* kps, uint8_t* desc, int cap, int* n_out, int* mono_index);

/* Batched form: n_frames images of identical size (offline sequences / several cameras); outputs
 * are [n_frames][cap] and n_out/mono_index[n_frames].  gray[i] are host pointers.               */
int rgbl_orb_extract_batch(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                           int lap0, int lap1, rgbl_keypoint* kps, uint8_t* desc, int cap, int* n_out, int* mono_index);

/* mvImagePyramid[level] of frame slot `frame` of the last extract call, WITH the 19 px REFLECT_101
 * border (src/ORBextractor.cc:1170-1195).  dst is (w+38) x (h+38), row stride dst_stride.        */
int rgbl_orb_get_pyramid(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride, int* w_out, int* h_out);

/* Stage introspection for parity tests (valid after an extract call). */
int rgbl_orb_get_level(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride, int* w_out, int* h_out);
int rgbl_orb_get_blurred_level(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride);
int rgbl_orb_get_candidates(rgbl_ctx* ctx, int frame, int level, int32_t* xys /* n x 3 */, int cap, int* n_out);

/* ---- DepthModule::CalculateDepthFromPcd (include/DepthModule.h:62, src/DepthModule.cc:50-79) ---- *
 * pts4xn: 4 x n planar float rows x,y,z,1 (Examples/RGB-L/rgbl_kitti.cc:168-177).  P: the 12 floats
 * of LidarProjectionMatrix (row-major 3x4), passed through unchanged (SURVEY A.6).  kps = mvKeys,
 * kps_un = mvKeysUn.  depth/uright = mvDepth/mvuRight.  raw_map/processed_map (H x W float, nullable)
 * = RawDepthMap / ProcessedDepthMap.                                                              */
int rgbl_depth_from_pcd(rgbl_ctx* ctx, const float* pts4xn, int n_pts, const float P[12], int width, int height,
                        const rgbl_depth_params* prm, const rgbl_keypoint* kps, const rgbl_keypoint* kps_un, int n_kp,
                        float* depth, float* uright, float* raw_map, float* processed_map);

/* ---- Frame::ComputeStereoFromRGBD (src/Frame.cc:1074-1095), the depth association of System::TrackRGBD ---- *
 * depth_map: H x W float32 (row stride in floats), metric depth (the caller applied DepthMapFactor, src/Tracking.cc:1538-1539).
 * d = depth_map[(int)kp.y][(int)kp.x] at the DISTORTED keypoint; depth[i] = d, uright[i] = kps_un[i].x - bf / d where d > 0, else -1. */
int rgbl_depth_from_map(rgbl_ctx* ctx, const float* depth_map, int width, int height, int stride_floats, float bf, const rgbl_keypoint* kps,
                        const rgbl_keypoint* kps_un, int n_kp, float* depth, float* uright);

/* Structuring element for Upsample_InverseDilation (src/DepthModule.cc:234-260): kind = "Rectangle",
 * "Cross", "Ellipse" (cv::getStructuringElement) or "Diamond" (include/DepthModule.h:138-161).   */
int rgbl_depth_structuring_element(const char* kind, int ku, int kv, uint8_t* mask /* kv*ku */);

/* ---- fused RGB-L frame construction, src/Frame.cc:289-377 (ExtractORB + UndistortKeyPoints + CalculateDepthFromPcd) ---- *
 * n_frames frames: image i + point cloud i -> keypoints, descriptors, mvDepth, mvuRight.  mvKeysUn comes from the context's camera
 * model (rgbl_set_camera_distortion; by default k1 == 0 as in KITTI, so mvKeysUn == mvKeys, src/Frame.cc:837-843).              */
int rgbl_frame_rgbl_batch(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                          const float* const* pts4xn, const int* n_pts, const float P[12], const rgbl_depth_params* prm,
                          rgbl_keypoint* kps, uint8_t* desc, float* depth, float* uright, int cap, int* n_out);

/* ---- tracking-thread stages ------------------------------------------------------------------------ *
 * The members of ORB_SLAM3::Frame the matchers read, for frames with Nleft == -1 (mono / stereo-rectified /
 * RGB-D / RGB-L): mvKeysUn, mvuRight, mDescriptors, image bounds (src/Frame.cc:871-899), mvScaleFactors,
 * calibration, mfLogScaleFactor.  The 64x48 grid (AssignFeaturesToGrid, src/Frame.cc:475-506) is rebuilt on
 * the device from these.                                                                                  */
typedef struct {
    int32_t n;
    const rgbl_keypoint* keys_un;
    const float* uright;
    const uint8_t* desc;
    float min_x, max_x, min_y, max_y;
    int32_t n_levels;
    const float* scale_factors;
    float fx, fy, cx, cy, bf;
    float log_scale_factor;
} rgbl_frame_view;

/* ORBmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, float th, bool bMono)
 * (include/ORBmatcher.h:51, src/ORBmatcher.cc:1676-1887).  Poses are Sophus::SE3f as (qx,qy,qz,qw,tx,ty,tz).
 * Last-frame map points i = 0..n_last-1 in LastFrame order: valid[i] = mvpMapPoints[i] != NULL &&
 * !mvbOutlier[i]; xw = GetWorldPos(); mp_desc = GetDescriptor(); last_octave/last_angle = the last frame's
 * keypoint; obs_pos[i] = Observations() > 0.  cur_state[i2] (nullable = all free): 0 free, 1 holds a point
 * with Observations() > 0, 2 holds a point without observations.  match[i2]: >= 0 index i now assigned,
 * -1 untouched, -2 cleared by the rotation-consistency check.  *n_matches = the reference's return value. */
int rgbl_search_by_projection_last(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float cur_pose[7], const float last_pose[7],
                                   int n_last, const uint8_t* valid, const float* xw, const uint8_t* mp_desc,
                                   const int32_t* last_octave, const float* last_angle, const uint8_t* obs_pos, float th, int mono,
                                   int check_orientation, const uint8_t* cur_state, int32_t* match, int* n_matches);

/* Frame::isInFrustum(MapPoint*, viewingCosLimit) for n map points (src/Frame.cc:602-664, Tracking.cc:3411).
 * Rcw row-major, tcw, Ow = Frame::mRcw/mtcw/mOw; normal = GetNormal(); mf_min/max_dist = mfMinDistance /
 * mfMaxDistance.  Outputs = mbTrackInView, mTrackProjX/Y/XR, mTrackDepth, mnTrackScaleLevel, mTrackViewCos. */
int rgbl_is_in_frustum(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float Rcw[9], const float tcw[3], const float Ow[3], int n,
                       const float* xw, const float* normal, const float* mf_min_dist, const float* mf_max_dist, float cos_limit,
                       uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr, float* track_depth, int32_t* level, float* view_cos);

/* ORBmatcher::SearchByProjection(Frame& F, const vector<MapPoint*>&, float th, bool bFarPoints, float thFarPoints)
 * (include/ORBmatcher.h:47, src/ORBmatcher.cc:43-213).  in_view[i] = mbTrackInView && !isBad(); the mTrack*
 * fields as filled by isInFrustum; nn_ratio = mfNNratio.  match/cur_state as above.                         */
int rgbl_search_by_projection_local(rgbl_ctx* ctx, const rgbl_frame_view* cur, int n, const uint8_t* in_view, const float* proj_x,
                                    const float* proj_y, const float* proj_xr, const float* track_depth, const int32_t* level,
                                    const float* view_cos, const uint8_t* mp_desc, const uint8_t* obs_pos, float th, float nn_ratio,
                                    int far_points, float th_far, const uint8_t* cur_state, int32_t* match, int* n_matches);

/* Frame::ComputeStereoMatches (src/Frame.cc:901-1071) between two frame slots of the last batched extraction (the left and
 * right image of a rectified stereo pair extracted as one batch: the reference runs its two ORBextractors on two threads,
 * src/Frame.cc:122-125).  mb = mbf / fx, mbf = Camera.bf.  depth / uright [n_left] = mvDepth / mvuRight of the left frame. */
int rgbl_stereo_matches(rgbl_ctx* ctx, int slot_left, int slot_right, float mb, float mbf, float* depth, float* uright, int cap);

/* ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>& vpMapPointMatches) (include/ORBmatcher.h:68,
 * src/ORBmatcher.cc:223-425), Nleft == -1.  pKF->mFeatVec and F.mFeatVec (DBoW2::FeatureVector = std::map<NodeId,
 * vector<unsigned>>) are passed as CSR: ascending node ids, node_start[n_nodes+1], feature indices in vector order.
 * kf_valid[i] = vpMapPointsKF[i] != NULL && !isBad().  match[idxF] = key-frame feature index whose map point is assigned
 * to F's feature idxF, or -1 (= NULL).  *n_matches = the reference's return value.                                    */
int rgbl_search_by_bow(rgbl_ctx* ctx, int n_kf, const uint8_t* kf_desc, const float* kf_angle, const uint8_t* kf_valid,
                       int n_nodes_kf, const uint32_t* kf_node_ids, const int32_t* kf_node_start, const int32_t* kf_node_feat,
                       int n_f, const uint8_t* f_desc, const float* f_angle,
                       int n_nodes_f, const uint32_t* f_node_ids, const int32_t* f_node_start, const int32_t* f_node_feat,
                       float nn_ratio, int check_orientation, int32_t* match, int* n_matches);

/* ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const set<MapPoint*>& sAlreadyFound, float th,
 * int ORBdist) (include/ORBmatcher.h:55, src/ORBmatcher.cc:1889-2010): relocalisation refinement.  Key-frame map points
 * i: valid[i] = pMP && !isBad() && !sAlreadyFound.count(pMP); kf_angle = pKF->mvKeysUn[i].angle; mf_min/max_dist =
 * mfMinDistance / mfMaxDistance.  cur_occupied[i2] != 0 <=> CurrentFrame.mvpMapPoints[i2] != NULL.  match as above.   */
int rgbl_search_by_projection_reloc(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float cur_pose[7], int n, const uint8_t* valid,
                                    const float* xw, const uint8_t* mp_desc, const float* kf_angle, const float* mf_min_dist,
                                    const float* mf_max_dist, float th, int orb_dist, int check_orientation, const uint8_t* cur_occupied,
                                    int32_t* match, int* n_matches);

/* Optimizer::PoseOptimization(Frame*) (include/Optimizer.h, src/Optimizer.cc:814-1114) for Nleft == -1 frames.
 * One edge per keypoint that has a map point, in keypoint order: xw = GetWorldPos(), obs = (kpUn.x, kpUn.y,
 * mvuRight[i]), inv_sigma2 = mvInvLevelSigma2[octave], stereo[i] = mvuRight[i] >= 0.  pose = Frame::GetPose().
 * outlier[i] = mvbOutlier; *n_inliers = the return value (0 and pose unchanged if n < 3).                   */
int rgbl_pose_optimize(rgbl_ctx* ctx, const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2,
                       const uint8_t* stereo, float fx, float fy, float cx, float cy, float bf, float pose_out[7], uint8_t* outlier,
                       int* n_inliers);

/* Resident form of the same work (device-throughput measurement, pipelined callers): inputs are
 * copied to HBM once, rgbl_resident_process can then be repeated with no host->device input traffic
 * and leaves its results in HBM until rgbl_resident_download.                                     */
int rgbl_resident_upload(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                         const float* const* pts4xn, const int* n_pts);
/* Same with the point clouds as raw KITTI .bin records, xyzr[f] = n_pts[f] x (x, y, z, reflectance) floats exactly as read from
 * the file: the element-wise re-layout of LoadPointcloudBinaryMat (Examples/RGB-L/rgbl_kitti.cc:151-185: rows x, y, z and a
 * row of ones) happens on the device.  The reference reads at most 1 000 000 floats (250 000 points) per file.             */
int rgbl_resident_upload_kitti(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                               const float* const* xyzr, const int* n_pts);
/* Same with the images as the PNG FILES' BYTES: replaces `imRGB = cv::imread(file, cv::IMREAD_UNCHANGED)` (Examples/RGB-L/rgbl_kitti.cc:87)
 * and Tracking::GrabImageRGBL's cvtColor to gray (src/Tracking.cc:1567-1580).  camera_rgb = Camera.RGB of the settings file (mbRGB: 1 ->
 * COLOR_RGB2GRAY / RGBA2GRAY, 0 -> COLOR_BGR2GRAY / BGRA2GRAY, applied to imread's B, G, R(, A) channel order like the reference does).
 * The host walks the chunks and inflates the zlib stream (entropy decoding is serial); scanline reconstruction (None / Sub / Up / Average /
 * Paeth) and the gray conversion run on the device and write level 0 of the frame slots.  Supported: 8-bit gray / RGB / RGBA,
 * non-interlaced, image size = the context's (RGBL_E_UNSUPPORTED / RGBL_E_INVALID otherwise; corrupt streams are RGBL_E_INVALID).     */
int rgbl_resident_upload_kitti_png(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb,
                                   const float* const* xyzr, const int* n_pts);
/* The decode alone: gray_out[f] = what the reference's mImGray holds for PNG stream f (height x width bytes, row stride `stride`). */
int rgbl_decode_png_gray(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb, uint8_t* const* gray_out,
                         int stride);
int rgbl_resident_process(rgbl_ctx* ctx, const float P[12], const rgbl_depth_params* prm, int* n_out /* nullable */);
int rgbl_resident_download(rgbl_ctx* ctx, rgbl_keypoint* kps, uint8_t* desc, float* depth, float* uright, int cap, int* n_out);

/* ---- Optimizer::LocalBundleAdjustment (src/Optimizer.cc:1116-1499), numerical core ------------------------------------
 * The shim gathers the local graph exactly as the reference builds it (:1210-1404): key-frame poses Tcw (local ones, the
 * fixed ones and pose_fixed = 1 for those and for the map's initial key frame), local map points, one edge per observation
 * (stereo = mvuRight >= 0, obs = (kpUn.x, kpUn.y, mvuRight), inv_sigma2 = mvInvLevelSigma2[octave]).  Runs g2o's
 * Levenberg-Marquardt with the Schur-complement solver for `iterations` (10 in the reference) and returns the optimised
 * poses / points (fixed poses unchanged) plus, per edge, the reference's erase test (:1416-1461: chi2 of the last
 * evaluated errors > 5.991 / 7.815, or non-positive depth).  Map bookkeeping (EraseMapPointMatch, SetPose, ...) stays in
 * the shim.  One Pinhole camera for all key frames (RGB-L / RGB-D / stereo rigs of the reference).                     */
int rgbl_local_bundle_adjustment(rgbl_ctx* ctx, int n_poses, const float* poses /* n_poses x 7: qx qy qz qw tx ty tz */, const uint8_t* pose_fixed,
                                 int n_points, const float* points /* n_points x 3 */, int n_edges, const int32_t* e_point, const int32_t* e_pose,
                                 const float* obs /* n_edges x 3 */, const uint8_t* stereo, const float* inv_sigma2, float fx, float fy, float cx,
                                 float cy, float bf, int iterations, float* poses_out, float* points_out, uint8_t* edge_erase,
                                 int* iterations_run /* nullable */);

/* ---- LocalMapping-thread kernels (SURVEY 8(f) row 3) -----------------------------------------------------------------
 * MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:329-403) for a batch of map points: the descriptors observed for
 * point p are desc[obs_start[p] .. obs_start[p+1]) (vDescriptors in the reference's order); best[p] = index within that list of
 * the descriptor with the least median Hamming distance to the others (first minimum), -1 for a point without observations.  */
int rgbl_distinctive_descriptors(rgbl_ctx* ctx, int n_points, const int32_t* obs_start /* n_points + 1 */, const uint8_t* desc, int32_t* best);

/* ORBmatcher::SearchForTriangulation(pKF1, pKF2, vMatchedPairs, bOnlyStereo, bCoarse) (include/ORBmatcher.h, src/ORBmatcher.cc:907-1146),
 * Nleft == -1 and one camera.  has_mp*[i] = GetMapPoint(i) != NULL; uright* = mvuRight; feature vectors as CSR like
 * rgbl_search_by_bow.  The per-pair constants are computed by the shim with the reference's own code: F12 = K1^-T [t12]x R12 K2^-1
 * (row-major, Pinhole::epipolarConstrain, src/CameraModels/Pinhole.cpp:109-112) and ep = pKF2->mpCamera->project(T2w * Cw);
 * scale_factors2 / level_sigma2_2 = pKF2->mvScaleFactors / mvLevelSigma2.  match12[idx1] = idx2 or -1 (vMatchedPairs = the
 * pairs in ascending idx1); *n_matches = the return value.                                                                 */
int rgbl_search_for_triangulation(rgbl_ctx* ctx, int n1, const uint8_t* desc1, const rgbl_keypoint* keys1, const uint8_t* has_mp1, const float* uright1,
                                  int n_nodes1, const uint32_t* node_ids1, const int32_t* node_start1, const int32_t* node_feat1,
                                  int n2, const uint8_t* desc2, const rgbl_keypoint* keys2, const uint8_t* has_mp2, const float* uright2,
                                  int n_nodes2, const uint32_t* node_ids2, const int32_t* node_start2, const int32_t* node_feat2,
                                  const float F12[9], const float ep[2], int n_levels, const float* scale_factors2, const float* level_sigma2_2,
                                  int only_stereo, int coarse, int check_orientation, int32_t* match12, int* n_matches);

/* ORBmatcher::Fuse(KeyFrame* pKF, const vector<MapPoint*>& vpMapPoints, float th, bool bRight = false) (src/ORBmatcher.cc:1148-1330),
 * the search part (:1176-1303).  kf = the key frame's members (a KeyFrame has the same grid / keypoint members as a Frame);
 * Tcw = pKF->GetPose(), Ow = pKF->GetCameraCenter(); valid[i] = pMP && !isBad() && !IsInKeyFrame(pKF); mf_min / mf_max =
 * mfMinDistance / mfMaxDistance.  best_idx[i] / best_dist[i] = bestIdx / bestDist of the reference's loop (-1 / 256 when the
 * point is rejected or has no candidate); the shim applies `bestDist <= TH_LOW` and the Replace / AddObservation bookkeeping.   */
int rgbl_fuse_search(rgbl_ctx* ctx, const rgbl_frame_view* kf, const float Tcw[7], const float Ow[3], int n, const uint8_t* valid, const float* xw,
                     const float* normal, const float* mf_min_dist, const float* mf_max_dist, const uint8_t* mp_desc, float th, int32_t* best_idx,
                     int32_t* best_dist);

/* ---- Frame::ComputeBoW (src/Frame.cc:828-835) -------------------------------------------------------------------------
 * = DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB>::transform(features, BowVector&, FeatureVector&, levelsup)
 * (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1206, per-feature descent :1218-1259, FORB::distance FORB.cpp:81-101).
 * The vocabulary is uploaded once, flattened by the shim from m_nodes: node i (0 = root) has the children
 * child_index[child_begin[i] .. child_begin[i+1]) in m_nodes[i].children order, a 32-byte descriptor, its WordValue weight and
 * word_id (>= 0 for leaves).  levels = m_L; weighting / scoring = the DBoW2 enum values of the vocabulary file header
 * (TF_IDF = 0 or TF = 1; any scoring that normalises with L1: L1_NORM = 0, CHI_SQUARE = 2, KL = 3, BHATTACHARYYA = 4; others
 * return RGBL_E_UNSUPPORTED).                                                                                            */
typedef struct rgbl_vocabulary rgbl_vocabulary;
int rgbl_vocabulary_create(rgbl_ctx* ctx, int n_nodes, const int32_t* child_begin /* n_nodes + 1 */, const int32_t* child_index,
                           const uint8_t* node_desc /* n_nodes x 32 */, const double* node_weight, const int32_t* word_id, int levels,
                           int weighting, int scoring, rgbl_vocabulary** out);
void rgbl_vocabulary_destroy(rgbl_vocabulary* voc);
/* BowVector (std::map<WordId, WordValue>) as ascending bow_word[] / bow_value[] (doubles, bit-identical to the map built by
 * addWeight + normalize(L1)); FeatureVector (std::map<NodeId, vector<unsigned>>) as CSR: ascending fv_node[], fv_start[n_fv_nodes + 1],
 * fv_feature[] in insertion order - the layout rgbl_search_by_bow takes.  All output arrays need room for n entries (fv_start: n + 1).
 * A leaf above level (levels - levelsup) leaves the reference's node id uninitialised; it is 0 (the root) here.               */
int rgbl_compute_bow(rgbl_ctx* ctx, const rgbl_vocabulary* voc, int n, const uint8_t* desc /* n x 32 */, int levelsup, int32_t* bow_word,
                     double* bow_value, int* n_words, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feature, int* n_fv_nodes);
/* same on the descriptors of frame `frame` of the last batched call, which are already in HBM */
int rgbl_resident_compute_bow(rgbl_ctx* ctx, const rgbl_vocabulary* voc, int frame, int levelsup, int32_t* bow_word, double* bow_value,
                              int* n_words, int32_t* fv_node, int32_t* fv_start, int32_t* fv_feature, int* n_fv_nodes);

/* Resident tracking chain over the frames of the last batched call, entirely on the device: for t = 1..n-1
 * SearchByProjection(frame t, frame t-1, th) -> PoseOptimization, every keypoint of frame t-1 with depth acting as a map
 * point (Frame::UnprojectStereo, src/Frame.cc:1137-1150, with the estimated pose of t-1).  Frame t is searched and its optimisation
 * started at the constant-velocity prediction mVelocity * Tcw(t-1), mVelocity = Tcw(t-1) * Tcw(t-2)^-1 (src/Tracking.cc:2904,
 * 2243-2245; Sophus SE3f products); frame 1 of a sequence has no velocity yet and starts at the pose of frame 0.
 * This is harness glue around the two reference functions (Tracking::TrackWithMotionModel, src/Tracking.cc:2888-2981,
 * stays on the host in the drop-in).  poses_out[n][7], n_matches[n], n_inliers[n]; entry 0 = (pose0, 0, 0).           */
int rgbl_resident_track(rgbl_ctx* ctx, const float pose0[7], float fx, float fy, float cx, float cy, float bf, float th, int mono,
                        float* poses_out, int* n_matches, int* n_inliers);

/* Asynchronous form of the same chain.  _begin copies the batch's frame outputs into chain-owned buffers, enqueues the chain
 * on the context's tracking stream and returns at once; _end blocks until the OLDEST queued chain has finished and writes its
 * results.  Up to two chains may be queued (FIFO): between _begin and _end the caller runs rgbl_resident_process /
 * rgbl_resident_upload / rgbl_frame_rgbl_batch for the NEXT batch and may already _begin its chain, which starts on the
 * device the moment the previous one ends (frame construction of batch i+1 overlaps the tracking of batch i, as the tracking
 * thread's pipeline does in the reference, and the device never waits for the host between two batches).  Every other
 * tracking entry point returns RGBL_E_INVALID while a chain is in flight.                                                */
int rgbl_resident_track_begin(rgbl_ctx* ctx, const float pose0[7], float fx, float fy, float cx, float cy, float bf, float th, int mono);
int rgbl_resident_track_end(rgbl_ctx* ctx, float* poses_out, int* n_matches, int* n_inliers);

/* The full per-frame tracking path of the reference for an RGB-L or RGB-D frame (the chain reads keypoints, descriptors, mvDepth and
 * mvuRight only), and batches that continue one sequence:
 *   TrackWithMotionModel (src/Tracking.cc:2888-2981): pose predicted by the constant-velocity model (:2904), SearchByProjection(frame t,
 *     frame t-1, th_last) -> PoseOptimization -> outliers discarded;
 *   TrackLocalMap (src/Tracking.cc:2983-3050 with SearchLocalPoints :3377-3460), when local_map_frames = K > 0: Frame::isInFrustum over
 *     the local map, SearchByProjection(frame t, local points, th_local, nn_ratio_local) -> PoseOptimization on all map points.  The
 *     local map of this harness = the keypoints with depth of the K frames before t-1, unprojected with their final poses, with
 *     MapPoint::UpdateNormalAndDepth's normal / scale-invariance distances for one observation (src/MapPoint.cc:437-490); it lives on
 *     the device as a ring (slot = frame counter mod K) and its points are searched in ring order.
 * continue_sequence != 0: frame 0 of this batch is tracked against the LAST frame of the previous chain of this context (keypoints,
 *   pose, the pose before it - for the velocity - and local map stay in HBM), so consecutive batches form one sequence and every frame of the batch is tracked; pose0 is
 *   ignored.  continue_sequence == 0 starts a sequence: frame 0 gets pose0 and the local map is emptied.
 * th_last: 15 (7 for System::STEREO, src/Tracking.cc:2913-2917); th_local: 3 for RGB-L / RGB-D, else 1 (:3432-3436); nn_ratio_local 0.8. */
typedef struct rgbl_chain_params {
    float pose0[7];
    float fx, fy, cx, cy, bf;
    float th_last;
    int mono;
    int continue_sequence;
    int local_map_frames;
    float th_local;
    float nn_ratio_local;
} rgbl_chain_params;
int rgbl_resident_track_begin2(rgbl_ctx* ctx, const rgbl_chain_params* prm);
/* as rgbl_resident_track_end, plus (nullable) per frame: matches of the local search, inliers after the first PoseOptimization;
 * n_inliers = inliers of the frame's last PoseOptimization.  Fails with RGBL_E_CAPACITY when the frame construction of the tracked
 * batch overflowed a capacity (the keypoint sets were truncated) or a matcher candidate list overflowed.                        */
int rgbl_resident_track_end2(rgbl_ctx* ctx, float* poses_out, int* n_matches, int* n_inliers, int* n_local_matches, int* n_inliers_first);

/* ---- Sequence runner: the loop of Examples/RGB-L/rgbl_kitti.cc:84-133 (load frame -> SLAM.TrackRGBL -> pose) for many frames per
 * call, entirely native.  Per batch of frames_per_batch consecutive frames: inputs -> frame construction -> tracking chain
 * (rgbl_chain_params; batches after the first continue the sequence) -> poses.  The chains are queued two deep, so the frame
 * construction (and host<->device copies) of batch b+1 overlap the tracking of batch b and the device never waits for the caller.
 *   host-input mode   gray != NULL: gray / pts4xn / n_pts hold one entry per frame of the call ([n_batches * frames_per_batch]);
 *                     pinned host memory makes the copies asynchronous;
 *   resident mode     gray == NULL: batch b processes the staged slot (first_slot + b) % n_slots (rgbl_resident_stage uploads a batch
 *                     into a device slot once; up to 8 slots) - device throughput without host->device input traffic.
 * Outputs (host, one entry per frame of the call): poses[.][7], n_matches, n_inliers (after the frame's last PoseOptimization),
 * n_local_matches (nullable).  kps != NULL additionally returns the frame-construction outputs of every frame ([.][cap] arrays, cap =
 * rgbl_keypoint_capacity(); n_kp[.] valid entries per frame).                                                                      */
typedef struct rgbl_sequence_io {
    int n_batches, frames_per_batch;
    int width, height, stride;
    const uint8_t* const* gray; const float* const* pts4xn; const int* n_pts;
    int n_slots, first_slot;
    float* poses; int* n_matches; int* n_inliers; int* n_local_matches;
    rgbl_keypoint* kps; uint8_t* desc; float* depth; float* uright; int cap; int* n_kp;
} rgbl_sequence_io;
int rgbl_resident_stage(rgbl_ctx* ctx, int slot, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                        const float* const* pts4xn, const int* n_pts);
int rgbl_track_sequence(rgbl_ctx* ctx, const float P[12], const rgbl_depth_params* prm, const rgbl_chain_params* chain, const rgbl_sequence_io* io);

/* ---- RGB-D: System::TrackRGBD (src/System.cc:339) -> Tracking::GrabImageRGBD (src/Tracking.cc:1518) -> RGB-D Frame constructor
 * (src/Frame.cc:200, ExtractORB + ComputeStereoFromRGBD :237 -> :1074-1095), batched and resident like the RGB-L entry points above.
 * The depth images stay uint16 in HBM (one plane per frame slot, allocated by the first RGB-D call; max_points may be 0) and are
 * scaled where ComputeStereoFromRGBD reads them: d = (float)sample * depth_scale, the per-pixel rule of GrabImageRGBD's
 * imDepth.convertTo(CV_32F, mDepthMapFactor) (:1538-1539), so the bits equal convert-then-gather.  d is read at the truncated
 * keypoint; mvDepth = d, mvuRight = kpUn.x - bf / d where d > 0, else -1 (mvKeysUn from the context's camera model,
 * rgbl_set_camera_distortion, as for RGB-L; TUM's RGB-D cameras have k1 != 0).
 * After rgbl_resident_process_rgbd, rgbl_resident_download, rgbl_resident_compute_bow and rgbl_resident_track_begin2 / _end2 work
 * unchanged (chain parameters for RGB-D: th_last 15, th_local 3).
 * depth[f]: H x W uint16 (CV_16U as imread returns it), row stride depth_stride elements.                                          */
int rgbl_resident_upload_rgbd(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                              const uint16_t* const* depth, int depth_stride);
/* Same with the files' bytes: the images as for rgbl_resident_upload_kitti_png, the depth images as 16-bit single-channel PNG
 * (cv::imread(depth_file, IMREAD_UNCHANGED), Examples/RGB-D/rgbd_kitti.cc; KITTI depth PNGs store metres x 256, TUM x 5000).
 * The depth stream must be 16-bit gray, non-interlaced, of the context's size; anything else (8-bit, 16-bit RGB, interlaced) is
 * RGBL_E_UNSUPPORTED.                                                                                                               */
int rgbl_resident_upload_rgbd_png(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb,
                                  const uint8_t* const* depth_png, const size_t* depth_png_bytes);
/* The depth decode alone: depth_out[f] = what imread(IMREAD_UNCHANGED) returns for depth PNG stream f (H x W uint16, row stride
 * `stride` elements).  Uses the depth planes of frame slots 0..n_frames-1.                                                          */
int rgbl_decode_png_depth16(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, uint16_t* const* depth_out, int stride);
/* Frame construction of the uploaded RGB-D frames.  depth_scale = Tracking::mDepthMapFactor (already 1.0f / RGBD.DepthMapFactor,
 * src/Tracking.cc:1188-1204), bf = Camera.bf (> 0).  RGBL_E_INVALID when the uploaded frames are not RGB-D frames.               */
int rgbl_resident_process_rgbd(rgbl_ctx* ctx, float depth_scale, float bf, int* n_out /* nullable */);
/* Upload one batch of RGB-D frames into staged slot `slot` for the resident mode of rgbl_track_sequence_rgbd. */
int rgbl_resident_stage_rgbd(rgbl_ctx* ctx, int slot, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                             const uint16_t* const* depth, int depth_stride);
/* The sequence runner for RGB-D (the loop of Examples/RGB-D/rgbd_kitti.cc: load image + depth -> SLAM.TrackRGBD -> pose), as
 * rgbl_track_sequence: io->pts4xn / io->n_pts must be NULL; host mode (io->gray != NULL) takes depth[] (one per frame of the call),
 * resident mode takes slots staged with rgbl_resident_stage_rgbd (a slot staged with rgbl_resident_stage is RGBL_E_INVALID, and so is
 * an RGB-D slot given to rgbl_track_sequence).                                                                                       */
int rgbl_track_sequence_rgbd(rgbl_ctx* ctx, float depth_scale, float bf, const rgbl_chain_params* chain, const rgbl_sequence_io* io,
                             const uint16_t* const* depth, int depth_stride);

/* ---- Stereo: System::TrackStereo -> Tracking::GrabImageStereo -> stereo Frame constructor (src/Frame.cc:101-197: the two ORBextractor
 * calls, then ComputeStereoMatches :901-1071), batched and resident like the RGB-D entry points above.  n_pairs rectified pairs are
 * extracted as ONE batch of 2 n_pairs frames, left images in frame slots [0, n_pairs), right ones in [n_pairs, 2 n_pairs), so
 * 2 n_pairs <= max_batch (RGBL_E_INVALID otherwise).  After rgbl_resident_process_stereo the left frames are the batch: rgbl_resident_download,
 * rgbl_resident_download_keys_un, rgbl_resident_compute_bow and rgbl_resident_track_begin2 / _end2 see them as they see RGB-L or RGB-D frames
 * (chain parameters for stereo: th_last 7, th_local 1).  A capacity overflow in the frame construction of a right frame fails _end2 with
 * RGBL_E_CAPACITY like one in a left frame.  The images must be rectified: on a context whose camera has k1 != 0
 * (rgbl_set_camera_distortion) every stereo entry point returns RGBL_E_UNSUPPORTED.                                                      */
int rgbl_resident_upload_stereo(rgbl_ctx* ctx, int n_pairs, const uint8_t* const* left, const uint8_t* const* right, int width, int height, int stride);
/* Same with the files' bytes (KITTI image_0 / image_1 PNGs), decoded as for rgbl_resident_upload_kitti_png; every stream must have the
 * context's size.                                                                                                                      */
int rgbl_resident_upload_stereo_png(rgbl_ctx* ctx, int n_pairs, const uint8_t* const* left_png, const size_t* left_bytes, const uint8_t* const* right_png,
                                    const size_t* right_bytes, int camera_rgb);
/* Frame construction of the uploaded pairs: mb = mbf / fx (the stereo Frame constructor's mb), mbf = Camera.bf; both finite and > 0.
 * ComputeStereoMatches is billed to the `match` profiling stage.  RGBL_E_INVALID when the uploaded frames are not stereo pairs.         */
int rgbl_resident_process_stereo(rgbl_ctx* ctx, float mb, float mbf, int* n_out /* nullable, [n_pairs] keypoints of the left frames */);
/* Upload one batch of n_pairs stereo pairs into staged slot `slot` for the resident mode of rgbl_track_sequence_stereo. */
int rgbl_resident_stage_stereo(rgbl_ctx* ctx, int slot, int n_pairs, const uint8_t* const* left, const uint8_t* const* right, int width, int height,
                               int stride);
/* The sequence runner for stereo (the loop of Examples/Stereo/stereo_kitti.cc: load left + right image -> SLAM.TrackStereo -> pose), as
 * rgbl_track_sequence with frames_per_batch pairs per batch: io->pts4xn / io->n_pts must be NULL; host mode (io->gray != NULL, the left
 * images) takes right[] (one per frame of the call), resident mode takes slots staged with rgbl_resident_stage_stereo (a slot of another
 * kind is RGBL_E_INVALID, and so is a stereo slot given to the other runners).                                                          */
int rgbl_track_sequence_stereo(rgbl_ctx* ctx, float mb, float mbf, const rgbl_chain_params* chain, const rgbl_sequence_io* io, const uint8_t* const* right);
/* Stereo rectification on the device: the cv::remap(im, imRect, M1, M2, INTER_LINEAR) that System::TrackStereo runs on both images before
 * GrabImageStereo when Settings::needToRectify() (src/System.cc:251 ff.; BORDER_CONSTANT 0, bit-exact with OpenCV).  m1l / m2l / m1r / m2r
 * are Settings' M1l, M2l, M1r, M2r (cv::initUndistortRectifyMap, CV_32F): H x W float32 maps at the context's size, row stride map_stride
 * floats.  They are converted once to OpenCV's fixed-point form on the device.  All four NULL turns rectification off (the default); a
 * partial set of NULLs, map_stride < width or a value that is not finite is RGBL_E_INVALID and the previous setting stays.
 * While rectification is on, the stereo entry points take the RAW images at the context's size (Settings without resize): uploads and
 * PNG decodes keep them in raw planes, staged slots hold them as they always do, and rgbl_resident_process_stereo / the stereo runner
 * remap both images of every pair into level 0 before the extraction, billed to the `pyramid` profiling stage.  PNG streams must then
 * be 8-bit gray (colour: RGBL_E_UNSUPPORTED, since the reference remaps before its conversion to gray).  The camera model
 * (rgbl_set_camera_distortion) keeps describing the rectified images, so it stays k1 = 0; mb / mbf and the chain's camera are the
 * rectified ones (Settings: P1's intrinsics, bf = b * P1(0,0)).  Setting or clearing the maps discards a pending stereo upload (the process
 * call then reports "nothing uploaded"); staged slots stay valid.                                                                       */
int rgbl_set_stereo_rectification(rgbl_ctx* ctx, const float* m1l, const float* m2l, const float* m1r, const float* m2r, int map_stride);

/* ---- Camera model of Frame::UndistortKeyPoints / ComputeImageBounds (src/Frame.cc:837-899) for every later batched frame construction
 * (rgbl_frame_rgbl_batch, rgbl_resident_process, rgbl_resident_process_rgbd, both sequence runners) and tracking chain of this context:
 * K = (fx, fy, cx, cy) (Pinhole::toK() == mK), dist = mDistCoef (k1, k2, p1, p2[, k3]), n_dist 4 or 5.  The keypoints are undistorted
 * on the device as cv::undistortPoints(mvKeys, K, mDistCoef, noArray(), mK) computes them; the chain then reads mvKeysUn and these bounds.
 * dist[0] == 0 -> mvKeysUn = mvKeys and bounds (0, W, 0, H), the reference's early return (the default).  bounds_out (nullable) = mnMinX,
 * mnMaxX, mnMinY, mnMaxY.  RGBL_E_INVALID for n_dist not 4/5, a non-finite value, fx or fy <= 0, or a chain in flight.                 */
int rgbl_set_camera_distortion(rgbl_ctx* ctx, float fx, float fy, float cx, float cy, const float* dist, int n_dist, float bounds_out[4]);
/* mvKeysUn of the last batched frame construction, laid out like rgbl_resident_download's kps ([n_frames][cap], n_out[n_frames]). */
int rgbl_resident_download_keys_un(rgbl_ctx* ctx, rgbl_keypoint* kps_un, int cap, int* n_out);

/* Keypoint distribution (DistributeOctTree) runs on the device by default (one CTA per (frame, level)); on != 0
 * selects the host implementation instead.  Both are exact.                                                     */
int rgbl_set_host_quadtree(rgbl_ctx* ctx, int on);

/* CUDA-event stopwatch on the context's main stream: mark(0) ... work ... mark(1); elapsed = device time
 * between the two marks (includes host gaps of the pipeline, excludes nothing).                      */
int rgbl_timer_mark(rgbl_ctx* ctx, int which);
int rgbl_timer_elapsed_ms(rgbl_ctx* ctx, double* ms);

/* ---- profiling: CUDA-event time per stage on the launching streams, kernel launch counts.  The
 * reference's counterpart is REGISTER_TIMES (include/Settings.h:24, src/Frame.cc:311-319).  on = 1: as the pipeline runs (the blur /
 * depth-map work of the auxiliary stream overlaps FAST's successors, so stage times overlap too); on = 2: the auxiliary stream is
 * joined before the quad-tree, so that no two kernels of the context run at the same time and every stage time is its own.   */
int rgbl_profile_enable(rgbl_ctx* ctx, int on);
int rgbl_profile_reset(rgbl_ctx* ctx);
int rgbl_profile_num_stages(void);
const char* rgbl_profile_stage_name(int stage);
int rgbl_profile_read(const rgbl_ctx* ctx, int stage, double* total_ms, int64_t* kernel_launches, int64_t* calls);
int rgbl_profile_totals(const rgbl_ctx* ctx, int64_t* kernel_launches, double* host_quadtree_ms);

/* ---- ORBmatcher::DescriptorDistance (src/ORBmatcher.cc:2058-2074).  Host-only helper. ---- */
int rgbl_descriptor_distance(const uint8_t a[32], const uint8_t b[32]);

#ifdef __cplusplus
}
#endif
#endif /* RGBL_B200_H */
