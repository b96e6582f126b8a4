// C ABI entry points of the tracking-thread stages: ORBmatcher::SearchByProjection (x2), Frame::isInFrustum and
// Optimizer::PoseOptimization.  MapPoint* / Frame objects of the reference are flat arrays here (the C++ shim
// gathers them, see INTEGRATION.md); all compute runs on the context's CUDA device.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "rgbl_ctx.h"
#include "rgbl_device.cuh"

namespace rgbl {

#define GROW(buf, need) do { if (!(buf).grow((size_t)(need), c->scratch_generation)) { c->err = "device allocation failed (tracking scratch)"; return RGBL_E_CUDA; } } while (0)

static int ensure_frame(Ctx* c, int n_frame) {
    TrackBufs& t = c->trk;
    GROW(t.keys, n_frame); GROW(t.uright, n_frame); GROW(t.desc, (size_t)n_frame * 32);
    GROW(t.csr_idx, n_frame); GROW(t.kp_cell, n_frame); GROW(t.state, n_frame);
    GROW(t.match, n_frame); GROW(t.minq, n_frame);
    if ((size_t)n_frame + 1 > t.inv_cnt.size()) {             // per-feature entry counters of the collect kernels + the entry total ([size - 1]): zero between launches
        GROW(t.inv_cnt, n_frame + 1);
        CU(cudaMemsetAsync(t.inv_cnt, 0, t.inv_cnt.size() * sizeof(int), c->st));
    }
    GROW(t.cell_start, kGridCols * kGridRows + 1);
    GROW(t.scalars, 16);
    return RGBL_OK;
}

static int ensure_queries(Ctx* c, int n_q) {
    TrackBufs& t = c->trk;
    GROW(t.lists, (size_t)n_q * kMatchListCap); GROW(t.list_slots, (size_t)n_q * kMatchListCap); GROW(t.list_n, n_q);
    GROW(t.dense, (size_t)n_q * kMatchListCap); GROW(t.dense_slot, (size_t)n_q * kMatchListCap);
    GROW(t.dense_q, (size_t)n_q * kMatchListCap); GROW(t.list_base, n_q);
    GROW(t.choice, n_q); GROW(t.resolved, n_q);
    GROW(t.q_u8a, n_q); GROW(t.q_u8b, n_q); GROW(t.q_desc, (size_t)n_q * 32);
    GROW(t.q_f3a, (size_t)n_q * 3); GROW(t.q_f3b, (size_t)n_q * 3);
    for (int k = 0; k < 7; ++k) GROW(t.q_f[k], n_q);
    GROW(t.q_i, n_q);
    return RGBL_OK;
}

// camera and image bounds of a frame as the matchers read them
static void set_camera(FrameDev& f, const float bounds[4], float fx, float fy, float cx, float cy, float bf) {
    f.min_x = bounds[0]; f.max_x = bounds[1]; f.min_y = bounds[2]; f.max_y = bounds[3];
    f.inv_w = static_cast<float>(kGridCols) / static_cast<float>(f.max_x - f.min_x);      // src/Frame.cc:351-352
    f.inv_h = static_cast<float>(kGridRows) / static_cast<float>(f.max_y - f.min_y);
    f.fx = fx; f.fy = fy; f.cx = cx; f.cy = cy; f.bf = bf;
    f.mb = bf / fx;                                                                       // src/Frame.cc:360
}

// ... of a frame view, with its level count and log scale factor.  The scale table is copied by upload_frame, which checks the level count.
static void set_view(FrameDev& f, const rgbl_frame_view* v) {
    const float bounds[4] = {v->min_x, v->max_x, v->min_y, v->max_y};
    set_camera(f, bounds, v->fx, v->fy, v->cx, v->cy, v->bf);
    f.n_levels = v->n_levels;
    f.log_scale_factor = v->log_scale_factor;
}

// uploads the frame view and builds its 64x48 grid; fills FrameDev
static int upload_frame(Ctx* c, const rgbl_frame_view* v, FrameDev& f) {
    if (!v || v->n < 0 || (v->n > 0 && (!v->keys_un || !v->uright || !v->desc)) || !v->scale_factors || v->n_levels < 1 || v->n_levels > RGBL_MAX_LEVELS) {
        c->err = "bad frame view"; return RGBL_E_INVALID;
    }
    int rc = ensure_frame(c, std::max(v->n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    CU(h2d(c, t.keys, v->keys_un, v->n));
    CU(h2d(c, t.uright, v->uright, v->n));
    CU(h2d(c, t.desc, v->desc, (size_t)v->n * 32));
    c->h_scalars[kHostFrameN] = v->n;
    CU(h2d(c, t.scalars + kDevFrameN, c->h_scalars + kHostFrameN, 1));
    f.n = t.scalars + kDevFrameN; f.keys = t.keys; f.uright = t.uright; f.desc = t.desc;
    set_view(f, v);
    for (int l = 0; l < v->n_levels; ++l) f.scale[l] = v->scale_factors[l];
    stage_begin(c, ST_MATCH, c->st);
    launch_grid_build(c->st, f, t.cell_start, t.csr_idx, t.kp_cell);
    return RGBL_OK;
}

static MatchScratch scratch(Ctx* c) {
    TrackBufs& t = c->trk;
    MatchScratch s;
    s.lists = t.lists; s.list_cap = kMatchListCap; s.list_n = t.list_n; s.minq = t.minq; s.choice = t.choice; s.resolved = t.resolved;
    s.overflow = c->d_overflow; s.rounds = t.scalars + kDevRounds; s.slots = t.list_slots; s.inv_cnt = t.inv_cnt; s.total = t.inv_cnt + (t.inv_cnt.size() - 1);
    s.dense = t.dense; s.dense_slot = t.dense_slot; s.dense_q = t.dense_q; s.base = t.list_base;
    return s;
}

// candidates kept per query by a ratio-tested search: a second-best beyond th_dist / nn_ratio can never reject (best <= th_dist <
// nn_ratio * second).  th_dist: the search's TH_HIGH or TH_LOW
static int keep_max(float th_dist, float nn_ratio) { return std::min(256, (int)std::floor(th_dist / nn_ratio) + 1); }

// the per-keypoint state of the searched frame (n keypoints): the caller's, or every keypoint free
static cudaError_t upload_state(Ctx* c, const uint8_t* cur_state, int n) {
    if (!n) return cudaSuccess;
    return cur_state ? h2d(c, c->trk.state, cur_state, n) : cudaMemsetAsync(c->trk.state, 0, n, c->st);
}

// a search without queries launches nothing that writes `match` or its two counters: no match, no round
static cudaError_t clear_search_outputs(Ctx* c, int n_frame) {
    const cudaError_t e = cudaMemsetAsync(c->trk.match, 0xff, (size_t)std::max(n_frame, 1) * sizeof(int), c->st);
    return e != cudaSuccess ? e : cudaMemsetAsync(c->trk.scalars + kDevMatches, 0, 2 * sizeof(int), c->st);
}

// Sophus::SE3f helpers on the host (float32, compiled with -ffp-contract=off): so3.hpp:358-366, se3.hpp inverse()
static void h_rotate(const float* T, const float p[3], float out[3]) {
    const float qx = T[0], qy = T[1], qz = T[2], qw = T[3];
    float uv[3] = {qy * p[2] - qz * p[1], qz * p[0] - qx * p[2], qx * p[1] - qy * p[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    const float cr[3] = {qy * uv[2] - qz * uv[1], qz * uv[0] - qx * uv[2], qx * uv[1] - qy * uv[0]};
    for (int i = 0; i < 3; ++i) out[i] = (p[i] + qw * uv[i]) + cr[i];
}

// Tcw.inverse().translation(): SO3f(conjugate) normalises in float (so3.hpp:229-231, 481-487), then invR * (t * -1) (se3.hpp:208-211)
static void h_inverse_translation(const float* T, float out[3]) {
    float inv[4] = {-T[0], -T[1], -T[2], T[3]};
    const float length = std::sqrt((inv[0] * inv[0] + inv[1] * inv[1]) + (inv[2] * inv[2] + inv[3] * inv[3]));      // Eigen 3.3: (x2 + y2) + (z2 + w2)
    for (int i = 0; i < 4; ++i) inv[i] /= length;
    const float nt[3] = {T[4] * -1.f, T[5] * -1.f, T[6] * -1.f};
    h_rotate(inv, nt, out);
}

static int finish_search(Ctx* c, int n_frame, int32_t* match, int* n_matches) {
    TrackBufs& t = c->trk;
    stage_end(c, ST_MATCH, c->st, 3);
    CU(cudaGetLastError());
    CU(d2h(c, match, t.match, n_frame));
    CU(d2h(c, c->h_scalars + kHostMatches, t.scalars + kDevMatches, 2));
    CU(d2h(c, c->h_overflow.get(), c->d_overflow, 1));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    if (*c->h_overflow) {
        cudaMemsetAsync(c->d_overflow, 0, sizeof(int), c->st);
        c->err = "matcher candidate list overflow (> 512 admissible candidates for one map point)";
        return RGBL_E_CAPACITY;
    }
    if (n_matches) *n_matches = c->h_scalars[kHostMatches];
    c->last_match_rounds = c->h_scalars[kHostRounds];
    return RGBL_OK;
}

}  // namespace rgbl

using namespace rgbl;

extern "C" {

int rgbl_search_by_projection_last(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float cur_pose[7], const float last_pose[7],
                                   int n_last, const uint8_t* valid, const float* xw, const uint8_t* mp_desc,
                                   const int32_t* last_octave, const float* last_angle, const uint8_t* obs_pos, float th, int mono,
                                   int check_orientation, const uint8_t* cur_state, int32_t* match, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!cur || !cur_pose || !last_pose || n_last < 0 || !match || (n_last > 0 && (!valid || !xw || !mp_desc || !last_octave || !last_angle || !obs_pos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n_last, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    CU(h2d(c, t.q_u8a, valid, n_last));
    CU(h2d(c, t.q_f3a, xw, (size_t)n_last * 3));
    CU(h2d(c, t.q_desc, mp_desc, (size_t)n_last * 32));
    CU(h2d(c, t.q_i, last_octave, n_last));
    CU(h2d(c, t.q_f[0], last_angle, n_last));
    CU(h2d(c, t.q_u8b, obs_pos, n_last));
    CU(upload_state(c, cur_state, cur->n));
    SearchLastParams prm;
    std::memcpy(prm.cur_pose, cur_pose, 7 * sizeof(float));
    prm.th = th; prm.check_orientation = check_orientation; prm.cur_pose_dev = nullptr; prm.flags_dev = nullptr;
    {   // bForward / bBackward, src/ORBmatcher.cc:1686-1693
        float twc[3], r[3];
        h_inverse_translation(cur_pose, twc);
        h_rotate(last_pose, twc, r);
        const float tlc_z = r[2] + last_pose[6];
        prm.forward = (tlc_z > f.mb && !mono) ? 1 : 0;
        prm.backward = (-tlc_z > f.mb && !mono) ? 1 : 0;
    }
    LastFrameDev lf{n_last, t.q_u8a, t.q_f3a, t.q_desc, t.q_i, t.q_f[0], t.q_u8b};
    if (n_last == 0) CU(clear_search_outputs(c, cur->n));
    launch_search_last(c->st, f, t.cell_start.get(), t.csr_idx.get(), lf, prm, scratch(c), t.state.get(), t.match.get(), t.scalars + kDevMatches);
    return finish_search(c, cur->n, match, n_matches);
}

int rgbl_is_in_frustum(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float Rcw[9], const float tcw[3], const float Ow[3], int n,
                       const float* xw, const float* normal, const float* mf_min_dist, const float* mf_max_dist, float cos_limit,
                       uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr, float* track_depth, int32_t* level, float* view_cos) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!cur || !Rcw || !tcw || !Ow || n < 0 || (n > 0 && (!xw || !normal || !mf_min_dist || !mf_max_dist || !in_view || !proj_x || !proj_y || !proj_xr || !track_depth || !level || !view_cos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (n == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    int rc = ensure_queries(c, n); if (rc) return rc;
    TrackBufs& t = c->trk;
    FrameDev f{};
    set_view(f, cur);
    FrustumParams prm;
    std::memcpy(prm.Rcw, Rcw, 9 * sizeof(float)); std::memcpy(prm.tcw, tcw, 3 * sizeof(float)); std::memcpy(prm.Ow, Ow, 3 * sizeof(float));
    prm.cos_limit = cos_limit;
    CU(h2d(c, t.q_f3a, xw, (size_t)n * 3));
    CU(h2d(c, t.q_f3b, normal, (size_t)n * 3));
    CU(h2d(c, t.q_f[4], mf_min_dist, n));
    CU(h2d(c, t.q_f[5], mf_max_dist, n));
    stage_begin(c, ST_MATCH, c->st);
    launch_frustum(c->st, f, prm, n, t.q_f3a, t.q_f3b, t.q_f[4], t.q_f[5], t.q_u8a, t.q_f[0], t.q_f[1], t.q_f[2], t.q_f[3], t.q_i, t.q_f[6]);
    stage_end(c, ST_MATCH, c->st, 1);
    CU(cudaGetLastError());
    CU(d2h(c, in_view, t.q_u8a, n));
    CU(d2h(c, proj_x, t.q_f[0], n));
    CU(d2h(c, proj_y, t.q_f[1], n));
    CU(d2h(c, proj_xr, t.q_f[2], n));
    CU(d2h(c, track_depth, t.q_f[3], n));
    CU(d2h(c, level, t.q_i, n));
    CU(d2h(c, view_cos, t.q_f[6], n));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_search_by_projection_local(rgbl_ctx* ctx, const rgbl_frame_view* cur, int n, const uint8_t* in_view, const float* proj_x,
                                    const float* proj_y, const float* proj_xr, const float* track_depth, const int32_t* level,
                                    const float* view_cos, const uint8_t* mp_desc, const uint8_t* obs_pos, float th, float nn_ratio,
                                    int far_points, float th_far, const uint8_t* cur_state, int32_t* match, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!cur || n < 0 || !match || (n > 0 && (!in_view || !proj_x || !proj_y || !proj_xr || !track_depth || !level || !view_cos || !mp_desc || !obs_pos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (!(nn_ratio > 0.f)) { c->err = "nn_ratio must be > 0"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    CU(h2d(c, t.q_u8a, in_view, n));
    CU(h2d(c, t.q_f[0], proj_x, n));
    CU(h2d(c, t.q_f[1], proj_y, n));
    CU(h2d(c, t.q_f[2], proj_xr, n));
    CU(h2d(c, t.q_f[3], track_depth, n));
    CU(h2d(c, t.q_i, level, n));
    CU(h2d(c, t.q_f[4], view_cos, n));
    CU(h2d(c, t.q_desc, mp_desc, (size_t)n * 32));
    CU(h2d(c, t.q_u8b, obs_pos, n));
    CU(upload_state(c, cur_state, cur->n));
    SearchLocalParams prm;
    prm.th = th; prm.nn_ratio = nn_ratio; prm.th_far = th_far; prm.far_points = far_points;
    prm.use_factor = (th != 1.0) ? 1 : 0;                                         // bFactor, src/ORBmatcher.cc:47
    prm.keep_max = keep_max(100.f, nn_ratio);                                     // TH_HIGH
    LocalPointsDev lp{n, nullptr, t.q_u8a, t.q_f[0], t.q_f[1], t.q_f[2], t.q_f[3], t.q_i, t.q_f[4], t.q_desc, t.q_u8b};
    if (n == 0) CU(clear_search_outputs(c, cur->n));
    launch_search_local(c->st, f, t.cell_start.get(), t.csr_idx.get(), lp, prm, scratch(c), t.state.get(), t.match.get(), t.scalars + kDevMatches);
    return finish_search(c, cur->n, match, n_matches);
}

int rgbl_pose_optimize(rgbl_ctx* ctx, const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2,
                       const uint8_t* stereo, float fx, float fy, float cx, float cy, float bf, float pose_out[7], uint8_t* outlier,
                       int* n_inliers) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!pose_in || !pose_out || n < 0 || !n_inliers || (n > 0 && (!xw || !obs || !inv_sigma2 || !stereo || !outlier))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (const char* why = pose_cluster_unsupported(c->cfg.device)) { c->err = why; return RGBL_E_UNSUPPORTED; }
    CU(cudaSetDevice(c->cfg.device));
    int rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    rc = ensure_frame(c, 1); if (rc) return rc;
    TrackBufs& t = c->trk;
    GROW(t.pose_work, (size_t)std::max(n, 1) * 3);
    CU(h2d(c, t.q_f3a, xw, (size_t)n * 3));
    CU(h2d(c, t.q_f3b, obs, (size_t)n * 3));
    CU(h2d(c, t.q_f[0], inv_sigma2, n));
    CU(h2d(c, t.q_u8a, stereo, n));
    PoseProblemDev p;
    p.n = n; p.xw = t.q_f3a; p.obs = t.q_f3b; p.inv_sigma2 = t.q_f[0]; p.stereo = t.q_u8a;
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = bf; p.n_dev = nullptr; p.pose_in_dev = nullptr;
    std::memcpy(p.pose_in, pose_in, 7 * sizeof(float));
    stage_begin(c, ST_POSE, c->st);
    launch_pose_optimize(c->st, p, t.pose_work.get(), t.q_u8b.get(), t.resolved.get(), t.q_f[1].get(), t.scalars + kDevPoseInliers);
    stage_end(c, ST_POSE, c->st, 1);
    CU(cudaGetLastError());
    CU(d2h(c, pose_out, t.q_f[1], 7));
    if (n >= 3) CU(d2h(c, outlier, t.resolved, n));
    CU(d2h(c, c->h_scalars + kHostPoseInliers, t.scalars + kDevPoseInliers, 1));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    *n_inliers = c->h_scalars[kHostPoseInliers];
    return RGBL_OK;
}

int rgbl_fuse_search(rgbl_ctx* ctx, const rgbl_frame_view* kf, const float Tcw[7], const float Ow[3], int n, const uint8_t* valid, const float* xw,
                     const float* normal, const float* mf_min_dist, const float* mf_max_dist, const uint8_t* mp_desc, float th, int32_t* best_idx,
                     int32_t* best_dist) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!kf || !Tcw || !Ow || n < 0 || (n > 0 && (!valid || !xw || !normal || !mf_min_dist || !mf_max_dist || !mp_desc || !best_idx || !best_dist))) {
        c->err = "null argument"; return RGBL_E_INVALID;
    }
    for (int i = 0; i < n; ++i) { best_idx[i] = -1; best_dist[i] = 256; }
    if (n == 0 || kf->n == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, kf, f); if (rc) return rc;
    rc = ensure_queries(c, n); if (rc) return rc;
    TrackBufs& t = c->trk;
    GROW(t.e_idx, (size_t)2 * n);
    CU(h2d(c, t.q_u8a, valid, n));
    CU(h2d(c, t.q_f3a, xw, (size_t)n * 3));
    CU(h2d(c, t.q_f3b, normal, (size_t)n * 3));
    CU(h2d(c, t.q_f[0], mf_min_dist, n));
    CU(h2d(c, t.q_f[1], mf_max_dist, n));
    CU(h2d(c, t.q_desc, mp_desc, (size_t)n * 32));
    float* hp = reinterpret_cast<float*>(c->h_scalars + kHostFusePose);       // pinned staging (clear of upload_frame's frame-size word): pose + camera centre
    for (int i = 0; i < 7; ++i) hp[i] = Tcw[i];
    for (int i = 0; i < 3; ++i) hp[7 + i] = Ow[i];
    CU(h2d(c, t.q_f[2], hp, 10));
    launch_fuse_search(c->st, f, t.cell_start, t.csr_idx, n, t.q_u8a, t.q_f3a, t.q_f3b, t.q_f[0], t.q_f[1], t.q_desc, t.q_f[2], t.q_f[2] + 7, th,
                       t.e_idx, t.e_idx + n);
    stage_end(c, ST_MATCH, c->st, 2);
    CU(cudaGetLastError());
    CU(d2h(c, best_idx, t.e_idx, n));
    CU(d2h(c, best_dist, t.e_idx + n, n));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_stereo_matches(rgbl_ctx* ctx, int slot_left, int slot_right, float mb, float mbf, float* depth, float* uright, int cap) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!depth || !uright) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (slot_left < 0 || slot_right < 0 || slot_left >= c->last_frames || slot_right >= c->last_frames) { c->err = "frame slot out of range (extract the stereo pair as one batch first)"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    int rc = stereo_matches(c, slot_left, slot_right, 1, mb, mbf); if (rc) return rc;
    CU(d2h(c, c->h_scalars + kHostFrameN, c->d_n_sel + slot_left, 1));
    CU(cudaStreamSynchronize(c->st));
    const int n = c->h_scalars[kHostFrameN];
    if (n > cap) { c->err = "output capacity too small"; return RGBL_E_CAPACITY; }
    CU(d2h(c, depth, c->d_depth + (size_t)slot_left * c->cap_kp, n));
    CU(d2h(c, uright, c->d_uright + (size_t)slot_left * c->cap_kp, n));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_search_by_bow(rgbl_ctx* ctx, int n_kf, const uint8_t* kf_desc, const float* kf_angle, const uint8_t* kf_valid,
                       int n_nodes_kf, const uint32_t* kf_node_ids, const int32_t* kf_node_start, const int32_t* kf_node_feat,
                       int n_f, const uint8_t* f_desc, const float* f_angle,
                       int n_nodes_f, const uint32_t* f_node_ids, const int32_t* f_node_start, const int32_t* f_node_feat,
                       float nn_ratio, int check_orientation, int32_t* match, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (n_kf < 0 || n_f < 0 || n_nodes_kf < 0 || n_nodes_f < 0 || !match || !(nn_ratio > 0.f) ||
        (n_kf > 0 && (!kf_desc || !kf_angle || !kf_valid)) || (n_f > 0 && (!f_desc || !f_angle)) ||
        (n_nodes_kf > 0 && (!kf_node_ids || !kf_node_start || !kf_node_feat)) || (n_nodes_f > 0 && (!f_node_ids || !f_node_start || !f_node_feat))) {
        c->err = "bad argument"; return RGBL_E_INVALID;
    }
    CU(cudaSetDevice(c->cfg.device));
    // merge-join of the two feature vectors (src/ORBmatcher.cc:239-393): queries in the reference's processing order
    std::vector<int> q_feat, q_cbeg, q_cend;
    std::vector<float> q_ang;
    int a = 0, b = 0;
    while (a < n_nodes_kf && b < n_nodes_f) {
        if (kf_node_ids[a] == f_node_ids[b]) {
            for (int ik = kf_node_start[a]; ik < kf_node_start[a + 1]; ++ik) {
                const int ikf = kf_node_feat[ik];
                if (ikf < 0 || ikf >= n_kf) { c->err = "KF feature index out of range"; return RGBL_E_INVALID; }
                if (!kf_valid[ikf]) continue;
                q_feat.push_back(ikf); q_cbeg.push_back(f_node_start[b]); q_cend.push_back(f_node_start[b + 1]); q_ang.push_back(kf_angle[ikf]);
            }
            ++a; ++b;
        } else if (kf_node_ids[a] < f_node_ids[b]) ++a;
        else ++b;
    }
    const int n_q = (int)q_feat.size();
    const int n_fcsr = n_nodes_f > 0 ? f_node_start[n_nodes_f] : 0;
    for (int i = 0; i < n_f; ++i) match[i] = -1;
    if (n_matches) *n_matches = 0;
    if (n_q == 0 || n_f == 0) return RGBL_OK;
    int rc = ensure_frame(c, std::max(n_f, n_fcsr)); if (rc) return rc;
    rc = ensure_queries(c, std::max(n_q, n_kf)); if (rc) return rc;
    TrackBufs& t = c->trk;
    GROW(t.e_idx, (size_t)3 * n_q);
    CU(h2d(c, t.q_desc, kf_desc, (size_t)n_kf * 32));
    CU(h2d(c, t.desc, f_desc, (size_t)n_f * 32));
    CU(h2d(c, t.uright, f_angle, n_f));       // reused as F angles
    CU(h2d(c, t.csr_idx, f_node_feat, n_fcsr));
    CU(h2d(c, t.e_idx, q_feat.data(), n_q));
    CU(h2d(c, t.e_idx + n_q, q_cbeg.data(), n_q));
    CU(h2d(c, t.e_idx + 2 * n_q, q_cend.data(), n_q));
    CU(h2d(c, t.q_f[0], q_ang.data(), n_q));
    CU(cudaMemsetAsync(t.q_u8b, 1, n_q, c->st));                                                              // every assignment blocks
    CU(cudaMemsetAsync(t.state, 0, n_f, c->st));
    c->h_scalars[kHostFrameN] = n_f;
    CU(h2d(c, t.scalars + kDevFrameN, c->h_scalars + kHostFrameN, 1));
    FrameDev f{};
    f.n = t.scalars + kDevFrameN;
    const int km = keep_max(50.f, nn_ratio);                                      // TH_LOW
    stage_begin(c, ST_MATCH, c->st);
    launch_search_bow(c->st, f, n_q, t.e_idx, t.e_idx + n_q, t.e_idx + 2 * n_q, t.q_desc, t.desc, t.q_f[0], t.uright, t.csr_idx, nn_ratio, km,
                      check_orientation, t.q_u8b, scratch(c), t.state, t.match, t.scalars + kDevMatches);
    std::vector<int32_t> mq(n_f);
    rc = finish_search(c, n_f, mq.data(), n_matches); if (rc) return rc;
    for (int i = 0; i < n_f; ++i) match[i] = (mq[i] >= 0) ? q_feat[mq[i]] : -1;       // cleared (-2) -> NULL like the reference
    return RGBL_OK;
}

int rgbl_search_by_projection_reloc(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float cur_pose[7], int n, const uint8_t* valid,
                                    const float* xw, const uint8_t* mp_desc, const float* kf_angle, const float* mf_min_dist,
                                    const float* mf_max_dist, float th, int orb_dist, int check_orientation, const uint8_t* cur_occupied,
                                    int32_t* match, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (!cur || !cur_pose || n < 0 || !match || (n > 0 && (!valid || !xw || !mp_desc || !kf_angle || !mf_min_dist || !mf_max_dist))) { c->err = "null argument"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    if (n) {
        CU(h2d(c, t.q_u8a, valid, n));
        CU(h2d(c, t.q_f3a, xw, (size_t)n * 3));
        CU(h2d(c, t.q_desc, mp_desc, (size_t)n * 32));
        CU(h2d(c, t.q_f[0], kf_angle, n));
        CU(h2d(c, t.q_f[4], mf_min_dist, n));
        CU(h2d(c, t.q_f[5], mf_max_dist, n));
        CU(cudaMemsetAsync(t.q_u8b, 1, n, c->st));
    }
    std::vector<uint8_t> st(std::max(cur->n, 1), 0);
    if (cur_occupied) for (int i = 0; i < cur->n; ++i) st[i] = cur_occupied[i] ? 1 : 0;        // any map point blocks (:1950-1951)
    if (cur->n) CU(h2d(c, t.state, st.data(), cur->n));
    SearchRelocParams prm;
    std::memcpy(prm.cur_pose, cur_pose, 7 * sizeof(float));
    h_inverse_translation(cur_pose, prm.Ow);                       // Ow = Tcw.inverse().translation()
    prm.th = th; prm.orb_dist = orb_dist; prm.check_orientation = check_orientation;
    RelocPointsDev rp{n, t.q_u8a, t.q_f3a, t.q_desc, t.q_f[0], t.q_f[4], t.q_f[5]};
    if (n == 0) CU(clear_search_outputs(c, cur->n));
    launch_search_reloc(c->st, f, t.cell_start, t.csr_idx, rp, prm, t.q_u8b, scratch(c), t.state, t.match, t.scalars + kDevMatches);
    CU(cudaStreamSynchronize(c->st));      // `st` (host vector) must outlive the async copy
    return finish_search(c, cur->n, match, n_matches);
}

#ifdef RGBL_TESTING_EXPORTS        // test hook (csrc/rgbl_testing.h): not in librgbl_b200.so
int rgbl_last_match_rounds(const rgbl_ctx* ctx) { return reinterpret_cast<const Ctx*>(ctx)->last_match_rounds; }
#endif

}  // extern "C" (re-opened below)

/* Resident tracking chain over the frames of the last rgbl_resident_process / rgbl_frame_rgbl_batch call, entirely on the
 * device (no host round trip per frame).  Per frame t (the reference's Tracking::Track for an RGB-L frame, src/Tracking.cc):
 *   TrackWithMotionModel (:2888-2981): SearchByProjection(frame t, frame t-1, th_last) -> PoseOptimization -> discard outliers,
 *     every LiDAR-depth keypoint of frame t-1 acting as a map point (Frame::UnprojectStereo with the final pose of t-1), constant-pose
 *     motion model;
 *   TrackLocalMap (:2983-3050, SearchLocalPoints :3377-3460), when local_map_frames = K > 0: isInFrustum over the local map (the
 *     points of the K frames before t-1), SearchByProjection(frame t, local points, th_local), PoseOptimization on all map points.
 * continue_sequence: frame 0 of the batch is tracked against the last frame of the previous chain of this context (its keypoints,
 * pose and the local map stay on the device), so consecutive batches form ONE sequence.                                        */
// The chain is asynchronous: _begin snapshots the batch's frame outputs into chain-owned buffers (a ~5 MB device copy),
// enqueues the whole per-frame chain on the context's high-priority tracking stream and returns; _end waits for it and
// hands the poses out.  Between the two calls the caller may run rgbl_resident_process on the NEXT batch: its kernels
// fill the SMs the single-CTA chain kernels leave idle (the chain is a latency-bound sequence of small launches).

// Everything that can refuse a chain before any CUDA call (callers see the first failing check's message); fills the plan.
static int check_chain(Ctx* c, const rgbl_chain_params& P, ChainPlan& p) {
    if (c->chain_pending >= 2) { c->err = "two tracking chains are already queued: call rgbl_resident_track_end first"; return RGBL_E_INVALID; }
    if (const char* why = pose_cluster_unsupported(c->cfg.device)) { c->err = why; return RGBL_E_UNSUPPORTED; }
    const int nF = c->last_frames, cap = c->cap_kp, K = std::max(P.local_map_frames, 0);
    if (nF < 1) { c->err = "nothing processed"; return RGBL_E_INVALID; }
    if (K > 16) { c->err = "local_map_frames > 16"; return RGBL_E_INVALID; }
    const bool cont = P.continue_sequence != 0;
    if (cont && !c->chain_has_carry) { c->err = "continue_sequence without a previous chain on this context"; return RGBL_E_INVALID; }
    if (cont && (c->carry_K != K || c->carry_cap != cap)) { c->err = "continue_sequence: local_map_frames / keypoint capacity differ from the previous chain"; return RGBL_E_INVALID; }
    const int S = c->lanes;
    if (nF % S) { c->err = "the batch's frame count is not a multiple of the sequence count (rgbl_set_sequences)"; return RGBL_E_INVALID; }
    if (cont && c->carry_lanes != S) { c->err = "continue_sequence: the sequence count differs from the previous chain's (rgbl_set_sequences)"; return RGBL_E_INVALID; }
    p.nF = nF; p.cap = cap; p.mono = P.mono; p.cont = cont ? 1 : 0; p.K = K; p.prev_valid = (cont && c->carry_prev_valid) ? 1 : 0;
    p.lanes = S; p.m = nF / S;
    p.th = P.th_last; p.th_local = P.th_local; p.nn_local = P.nn_ratio_local;
    p.fx = P.fx; p.fy = P.fy; p.cx = P.cx; p.cy = P.cy; p.bf = P.bf;
    std::memcpy(p.bounds, c->frame_bounds, sizeof(p.bounds));      // ComputeImageBounds of the frames' camera
    return RGBL_OK;
}

// The chain's resources at the plan's sizes: the tracking stream and the events (each one created by the first chain that finds it
// missing), the pinned result staging, every device buffer.
static int ensure_chain_resources(Ctx* c, const ChainPlan& p) {
    const int nF = p.nF, cap = p.cap, K = p.K, n_lq = local_query_cap(p);
    if (!c->st_trk) {
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU(c->st_trk.create(hi));
    }
    auto have = [](Event& e, unsigned flags) { return e ? cudaSuccess : e.create(flags); };
    CU(have(c->ev_snap, cudaEventDisableTiming));
    for (int i = 0; i < 2; ++i) {
        CU(have(c->ev_chain_b[i], 0)); CU(have(c->ev_chain_e[i], 0));
        CU(have(c->ev_chain_done[i], cudaEventDisableTiming));
    }
    // RGBL_CHAIN_TIMING=1: CUDA events between the launches of the middle frame (warm, in-stream kernel times; stderr at _end)
    if (c->chain_timing_on) for (Event& e : c->chain_tev) CU(have(e, 0));
    if (c->h_chain_cap < (size_t)nF) {
        if (c->chain_pending) { c->err = "batch size grew while a chain is in flight"; return RGBL_E_INVALID; }
        const size_t capF = slot_frames(c), nf = 2 * chain_pose_floats(capF), ni = 2 * chain_count_ints(capF, kMaxLanes);
        c->h_chain_cap = 0;
        if (!c->h_chain_f.grow(nf, c->scratch_generation, nf) || !c->h_chain_i.grow(ni, c->scratch_generation, ni)) {
            c->err = "pinned allocation failed (chain result staging)"; return RGBL_E_CUDA;
        }
        c->h_chain_cap = capF;
    }
    // every lane buffer: lanes x its lane stride (ChainLaneStrides)
    const size_t S = (size_t)p.lanes;
    const ChainLaneStrides ls = chain_lane_strides(p);
    TrackBufs& t = c->trk;
    GROW(t.state, S * ls.kp); GROW(t.match, S * ls.kp); GROW(t.minq, S * ls.kp); GROW(t.scalars, S * ls.scalars);
    if (S * ls.inv > t.inv_cnt.size()) {                  // per-feature entry counters + entry total of each lane: zero between launches
        GROW(t.inv_cnt, S * ls.inv);
        CU(cudaMemsetAsync(t.inv_cnt, 0, t.inv_cnt.size() * sizeof(int), c->st));
    }
    int rc = ensure_queries(c, (int)(S * ls.q)); if (rc) return rc;
    GROW(t.pose_work, S * ls.kp * 3);
    GROW(t.ch_poses, (size_t)nF * 7 + S * ls.pose_tmp); GROW(t.ch_counts, chain_count_ints(nF, S));      // poses | per lane: pose after TrackWithMotionModel, predicted pose
    GROW(t.e_xw, S * ls.kp * 3); GROW(t.e_obs, S * ls.kp * 3); GROW(t.e_info, S * ls.kp);
    GROW(t.e_st, S * ls.kp); GROW(t.e_lvl, S * ls.kp); GROW(t.e_out, S * ls.kp); GROW(t.e_idx, S * ls.kp);
    // carried last frame of each lane's sequence + the local map rings (persist across chains of this context)
    GROW(t.c_kps, S * ls.kp); GROW(t.c_desc, S * ls.kp * 32); GROW(t.c_depth, S * ls.kp);
    GROW(t.carry, S);
    if (K > 0) {
        const size_t nr = S * ls.ring;
        if (p.cont && t.r_valid.size() < nr) { c->err = "local map ring missing"; return RGBL_E_INVALID; }
        GROW(t.r_valid, nr); GROW(t.r_xw, nr * 3); GROW(t.r_normal, nr * 3);
        GROW(t.r_min, nr); GROW(t.r_max, nr); GROW(t.r_desc, nr * 32);
        GROW(t.lq_u8, S * kLqU8Planes * ls.lq); GROW(t.lq_f, S * kLqFPlanes * ls.lq); GROW(t.lq_i, S * kLqIPlanes * ls.lq);
        GROW(t.lq_desc, S * ls.lq * 32); GROW(t.match_local, S * ls.kp);
        if (t.lookback.size() < S * ls.lookback) {
            GROW(t.lookback, S * ls.lookback);
            CU(cudaMemsetAsync(t.lookback, 0, t.lookback.size() * sizeof(int), c->st));     // ordered before the chain by ev_snap (snapshot_batch)
        }
        if ((n_lq + 255) / 256 + 1 > 1024) { c->err = "local map too large for the compaction slots (local_map_frames x keypoint capacity > 261 k)"; return RGBL_E_UNSUPPORTED; }
    }
    // per-slot buffers: twice the size, the slot picks its half (chain_slot)
    const size_t nF_full = slot_frames(c), tot_full = nF_full * cap, cs_full = nF_full * (kGridCols * kGridRows + 1);
    if (c->chain_pending && (t.s_kps.size() < 2 * tot_full || t.b_cell_start.size() < 2 * cs_full)) { c->err = "batch size grew while a chain is in flight"; return RGBL_E_INVALID; }
    GROW(t.s_kps, 2 * tot_full); GROW(t.s_desc, 2 * tot_full * 32); GROW(t.s_depth, 2 * tot_full);
    GROW(t.s_uright, 2 * tot_full); GROW(t.s_nsel, 2 * nF_full);
    GROW(t.b_cell_start, 2 * cs_full);
    GROW(t.b_csr_idx, 2 * tot_full); GROW(t.b_kp_cell, 2 * tot_full);
    return RGBL_OK;
}

// Copies the batch's frame outputs into the slot's snapshot on the frame-construction stream (ordered after the batch's kernels, before
// the next batch's) and makes the tracking stream wait for it.
static int snapshot_batch(Ctx* c, const ChainPlan& p, int slot, const ChainSlot& s) {
    const size_t tot = (size_t)p.nF * p.cap;
    // mvKeysUn: the chain reads nothing but undistorted keypoints (grid, projections, edges, UnprojectStereo, ring, carried frame)
    CU(cudaMemcpyAsync(s.s_kps, c->frames_undistorted ? c->d_kps_un : c->d_kps, tot * sizeof(rgbl_keypoint), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s.s_desc, c->d_desc, tot * 32, cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s.s_depth, c->d_depth, tot * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s.s_uright, c->d_uright, tot * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s.s_nsel, c->d_n_sel, (size_t)p.nF * sizeof(int), cudaMemcpyDeviceToDevice, c->st));
    // the frame-construction overflow flags of THIS batch travel with the chain (checked in _end)
    CU(d2h(c, c->h_chain_ovf + 2 * slot, c->d_overflow, 2));
    CU(cudaEventRecord(c->ev_snap, c->st));
    CU(cudaStreamWaitEvent(c->st_aux, c->ev_snap, 0));      // the aux stream writes depth / uright of the next batch
    CU(cudaStreamWaitEvent(c->st_trk, c->ev_snap, 0));
    return RGBL_OK;
}

// Lane s's view of the chain's buffers: the single-sequence chain's buffers, each offset by s times its ChainLaneStrides stride.
struct ChainLane {
    uint8_t *q_u8a, *q_u8b, *state, *e_st, *e_lvl, *e_out, *c_desc;
    float *q_f3a, *q_f0, *e_xw, *e_obs, *e_info, *c_depth, *pose_tmp, *pose_pred;
    int *q_i, *match, *match_local, *e_idx, *scalars, *lookback;
    double* pose_work; rgbl_keypoint* c_kps; ChainCarry* carry;
    MatchScratch ms; ChainCounts cnt; LocalRingDev ring; LocalQueriesDev lq;
    size_t f0;                        // the lane's first frame in the batch (s * m)
};
static ChainLane chain_lane(Ctx* c, const ChainPlan& p, int s) {
    TrackBufs& t = c->trk;
    const ChainLaneStrides st = chain_lane_strides(p);
    const size_t kp = s * st.kp, q = s * st.q, ring = s * st.ring, lq = s * st.lq;
    ChainLane L;
    L.q_u8a = t.q_u8a + q; L.q_u8b = t.q_u8b + q; L.q_f3a = t.q_f3a + 3 * q; L.q_f0 = t.q_f[0] + q; L.q_i = t.q_i + q;
    L.state = t.state + kp; L.match = t.match + kp; L.match_local = p.K > 0 ? t.match_local + kp : nullptr;
    L.e_xw = t.e_xw + 3 * kp; L.e_obs = t.e_obs + 3 * kp; L.e_info = t.e_info + kp; L.e_st = t.e_st + kp; L.e_lvl = t.e_lvl + kp;
    L.e_out = t.e_out + kp; L.e_idx = t.e_idx + kp; L.pose_work = t.pose_work + 3 * kp;
    L.c_kps = t.c_kps + kp; L.c_desc = t.c_desc + 32 * kp; L.c_depth = t.c_depth + kp; L.carry = t.carry + s;
    L.scalars = t.scalars + s * st.scalars;
    L.pose_tmp = t.ch_poses + 7 * (size_t)p.nF + s * st.pose_tmp; L.pose_pred = L.pose_tmp + 7;
    L.cnt = chain_counts(t.ch_counts, p.nF, p.m, s);
    L.f0 = (size_t)s * p.m;
    MatchScratch& m = L.ms;
    m.lists = t.lists + q * kMatchListCap; m.slots = t.list_slots + q * kMatchListCap; m.list_cap = kMatchListCap; m.list_n = t.list_n + q;
    m.dense = t.dense + q * kMatchListCap; m.dense_slot = t.dense_slot + q * kMatchListCap; m.dense_q = t.dense_q + q * kMatchListCap; m.base = t.list_base + q;
    m.inv_cnt = t.inv_cnt + s * st.inv; m.total = m.inv_cnt + p.cap;
    m.minq = t.minq + kp; m.choice = t.choice + q; m.resolved = t.resolved + q; m.overflow = L.cnt.overflow; m.rounds = L.scalars + kDevRounds;
    if (p.K > 0) {
        L.ring = LocalRingDev{p.K, p.cap, t.r_valid + ring, t.r_xw + 3 * ring, t.r_normal + 3 * ring, t.r_min + ring, t.r_max + ring, t.r_desc + 32 * ring,
                              &L.carry->ring_count};
        L.lq = local_queries(t.lq_u8 + kLqU8Planes * lq, t.lq_f + kLqFPlanes * lq, t.lq_i + kLqIPlanes * lq, t.lq_desc + 32 * lq, (int)st.lq, L.cnt.n_queries);
        L.lookback = t.lookback + s * st.lookback;
    } else {
        L.ring = LocalRingDev{p.K, p.cap, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, &L.carry->ring_count};
        L.lq = LocalQueriesDev{}; L.lookback = nullptr;
    }
    return L;
}

// Everything the chain does on the tracking stream.  It is captured ONCE per slot into a CUDA graph and
// replayed: the launch commands then live in device memory, so the dependent-kernel sequence no longer fetches a command
// packet from the host over PCIe per launch (which the concurrent H2D uploads of the next batch were slowing down) and
// _begin costs one graph launch instead of hundreds of kernel launches on the host.
// It reads the plan, the slot's buffers and the context (its scratch, whose addresses scratch_generation stands for, and settings fixed
// at rgbl_create) and nothing else: the graph's key is the plan and that generation.
// Sequence lanes: step k of the loop tracks frame k of every lane (batch frame s * m + k), each launch serving all lanes (Laned arguments
// built from chain_lane(s)), so the launch count per step does not depend on the lane count.
static int enqueue_chain(Ctx* c, const ChainPlan& p, const ChainSlot& s, int& n_launches) {
    struct PdlScope {      // programmatic dependent launches between the chain's kernels (rgbl_device.cuh: pdl_wait)
        explicit PdlScope(bool on) { chain_launch_pdl() = on; }
        ~PdlScope() { chain_launch_pdl() = false; }
    } pdl(c->chain_pdl_on);
    TrackBufs& t = c->trk;
    const cudaStream_t cs = c->st_trk;
    const int nF = p.nF, cap = p.cap, K = p.K, S = p.lanes, m = p.m, n_lq = local_query_cap(p);
    const bool cont = p.cont != 0, chain_timing = c->chain_timing_on;
    const Event* tev = c->chain_tev;
    n_launches = 0;
    std::vector<ChainLane> lanes;
    for (int l = 0; l < S; ++l) lanes.push_back(chain_lane(c, p, l));
    const ChainLane& L0 = lanes[0];
    float* poses = t.ch_poses;                 // batch frame j -> poses + 7 j
    auto pose_of = [&](int l, int k) { return poses + 7 * (lanes[l].f0 + (size_t)k); };
    auto laned = [&](auto make) { return laned_of(S, make); };
    CU(cudaMemsetAsync(t.ch_counts, 0, chain_count_ints(nF, S) * sizeof(int), cs));
    if (!cont) {
        // frame 0 of every lane: its start pose (the slot's pose0 block, one 7-float record per lane)
        CU(cudaMemcpy2DAsync(poses, 7 * sizeof(float) * m, s.h_f, 7 * sizeof(float), 7 * sizeof(float), S, cudaMemcpyHostToDevice, cs));
        if (K > 0) {
            CU(cudaMemsetAsync(t.r_valid, 0, (size_t)S * K * cap, cs));
            for (const ChainLane& L : lanes) CU(cudaMemsetAsync(&L.carry->ring_count, 0, sizeof(int), cs));
        }
    }
    FrameDev f0{};
    set_camera(f0, p.bounds, p.fx, p.fy, p.cx, p.cy, p.bf);
    f0.n_levels = c->tab.nlevels;
    for (int l = 0; l < f0.n_levels; ++l) f0.scale[l] = c->tab.scale[l];
    f0.log_scale_factor = std::log(c->cfg.orb.scale_factor);
    // the 64x48 grids do not depend on the poses: all frames of all lanes in one launch (one CTA per frame)
    {
        FrameDev f = f0;
        f.n = s.s_nsel; f.keys = s.s_kps;
        launch_grid_build_batch(cs, f, nF, cap, s.b_cell_start, s.b_csr_idx, s.b_kp_cell); ++n_launches;
    }
    // unprojection of lane l's frame j (map points of the search in frame j + 1); j == -1: the lane's carried frame
    auto prep_of = [&](int l, int j) {
        const ChainLane& L = lanes[l];
        ChainPrepDev cp{};
        if (j < 0) { cp.kps = L.c_kps; cp.depth = L.c_depth; cp.n_ptr = &L.carry->n_sel; }
        else { cp.kps = s.s_kps + (L.f0 + j) * cap; cp.depth = s.s_depth + (L.f0 + j) * cap; cp.n_ptr = s.s_nsel + L.f0 + j; }
        cp.fx = f0.fx; cp.fy = f0.fy; cp.cx = f0.cx; cp.cy = f0.cy; cp.mb = f0.mb; cp.mono = p.mono; cp.cap = cap;
        cp.valid = L.q_u8a; cp.xw = L.q_f3a; cp.octave = L.q_i; cp.angle = L.q_f0; cp.obs_pos = L.q_u8b; cp.flags = L.cnt.flags; cp.state_clear = L.state;
        // constant-velocity motion model: the pose of the frame before frame j (nullptr at the start of a sequence)
        if (j >= 1) cp.prev_pose = pose_of(l, j - 1);
        else if (j == 0) cp.prev_pose = cont ? L.carry->pose : nullptr;
        else cp.prev_pose = p.prev_valid ? L.carry->prev_pose : nullptr;      // the pose of the frame before the carried one
        cp.pred_pose = L.pose_pred;
        return cp;
    };
    const int k0 = cont ? 0 : 1;
    for (int k = k0; k < m; ++k) {
        const bool tm = chain_timing && k == std::max(1, m / 2);
        const Laned<const float*> last_pose = laned([&](int l) -> const float* { return (k == 0) ? lanes[l].carry->pose : pose_of(l, k - 1); });
        const Laned<const uint8_t*> last_desc = laned([&](int l) -> const uint8_t* {
            return (k == 0) ? lanes[l].c_desc : s.s_desc + (lanes[l].f0 + k - 1) * cap * 32;
        });
        if (tm) cudaEventRecord(tev[0], cs);
        if (k == k0) { launch_chain_prep(cs, laned([&](int l) { return prep_of(l, k - 1); }), last_pose, S); ++n_launches; }   // later frames: prepared by the previous pose kernel
        const Laned<FrameDev> f = laned([&](int l) {
            const size_t cu = (lanes[l].f0 + k) * cap;
            FrameDev fl = f0;
            fl.n = s.s_nsel + lanes[l].f0 + k; fl.keys = s.s_kps + cu; fl.uright = s.s_uright + cu; fl.desc = s.s_desc + cu * 32;
            return fl;
        });
        const Laned<const int*> cell_start = laned([&](int l) -> const int* { return s.b_cell_start + (lanes[l].f0 + k) * (kGridCols * kGridRows + 1); });
        const Laned<const int*> csr_idx = laned([&](int l) -> const int* { return s.b_csr_idx + (lanes[l].f0 + k) * cap; });
        const Laned<MatchScratch> ms = laned([&](int l) { return lanes[l].ms; });
        const Laned<uint8_t*> state = laned([&](int l) { return lanes[l].state; });
        if (tm) cudaEventRecord(tev[1], cs);
        const Laned<SearchLastParams> prm = laned([&](int l) {
            SearchLastParams pr{};
            pr.th = p.th; pr.check_orientation = 1; pr.cur_pose_dev = lanes[l].pose_pred; pr.flags_dev = lanes[l].cnt.flags;      // projected with the motion model's pose (src/Tracking.cc:2904)
            return pr;
        });
        const Laned<LastFrameDev> lf = laned([&](int l) {
            const ChainLane& L = lanes[l];
            return LastFrameDev{cap, L.q_u8a, L.q_f3a, lane_value(last_desc, l), L.q_i, L.q_f0, L.q_u8b};
        });
        const Laned<ChainEdgesOut> eo = laned([&](int l) {
            const ChainLane& L = lanes[l];
            return ChainEdgesOut{L.e_xw, L.e_obs, L.e_info, L.e_st, L.e_idx, L.cnt.n_edges};
        });
        launch_search_last(cs, f, cell_start, csr_idx, lf, prm, ms, state, laned([&](int l) { return lanes[l].match; }),
                           laned([&](int l) { return lanes[l].cnt.n_matches + k; }), &eo, S); n_launches += 2;   // + edges of the matches
        if (tm) cudaEventRecord(tev[2], cs);
        auto pose_problem = [&](int l, bool second) {
            const ChainLane& L = lanes[l];
            PoseProblemDev pp{};
            pp.n = 0; pp.n_dev = second ? L.cnt.n_edges2 : L.cnt.n_edges; pp.pose_in_dev = second ? L.pose_tmp : L.pose_pred;
            pp.xw = L.e_xw; pp.obs = L.e_obs; pp.inv_sigma2 = L.e_info; pp.stereo = L.e_st;
            pp.fx = p.fx; pp.fy = p.fy; pp.cx = p.cx; pp.cy = p.cy; pp.bf = p.bf;
            return pp;
        };
        const Laned<ChainPrepDev> nxt = laned([&](int l) { return prep_of(l, k); });
        const Laned<double*> work = laned([&](int l) { return lanes[l].pose_work; });
        const Laned<uint8_t*> e_lvl = laned([&](int l) { return lanes[l].e_lvl; });
        const Laned<uint8_t*> e_out = laned([&](int l) { return lanes[l].e_out; });
        const Laned<float*> pose_final = laned([&](int l) { return pose_of(l, k); });
        const Laned<int*> n_inliers = laned([&](int l) { return lanes[l].cnt.n_inliers + k; });
        if (K == 0) {
            launch_pose_optimize(cs, laned([&](int l) { return pose_problem(l, false); }), work, e_lvl, e_out, pose_final, n_inliers, (k + 1 < m) ? &nxt : nullptr, S); ++n_launches;
            if (tm) { cudaEventRecord(tev[3], cs); cudaEventRecord(tev[4], cs); cudaEventRecord(tev[5], cs); cudaEventRecord(tev[6], cs); }
        } else {
            const Laned<float*> pose_tmp = laned([&](int l) { return lanes[l].pose_tmp; });
            launch_pose_optimize(cs, laned([&](int l) { return pose_problem(l, false); }), work, e_lvl, e_out, pose_tmp,
                                 laned([&](int l) { return lanes[l].cnt.n_inliers_first + k; }), nullptr, S); ++n_launches;
            if (tm) cudaEventRecord(tev[3], cs);
            // TrackLocalMap: outlier discard + isInFrustum + ordered compaction, local search, edges of all map points, second optimisation
            launch_tlm_prepare(cs, f, laned([&](int l) -> const float* { return lanes[l].pose_tmp; }), laned([&](int l) { return lanes[l].ring; }), 0.5f,
                               laned([&](int l) -> const int* { return lanes[l].cnt.n_edges; }), laned([&](int l) -> const int* { return lanes[l].e_idx; }),
                               laned([&](int l) -> const uint8_t* { return lanes[l].e_out; }), state, laned([&](int l) { return lanes[l].match; }),
                               laned([&](int l) { return lanes[l].lq; }), L0.lookback, laned([&](int l) { return lanes[l].cnt.overflow; }), S); ++n_launches;
            const Laned<LocalPointsDev> lp = laned([&](int l) {
                const LocalQueriesDev& lq = lanes[l].lq;
                return LocalPointsDev{n_lq, lanes[l].cnt.n_queries, lq.in_view, lq.proj_x, lq.proj_y, lq.proj_xr, lq.depth, lq.level, lq.view_cos, lq.desc, lq.obs_pos};
            });
            SearchLocalParams sl{};
            sl.th = p.th_local; sl.nn_ratio = p.nn_local; sl.th_far = 0.f; sl.use_factor = (p.th_local != 1.0f) ? 1 : 0; sl.far_points = 0;
            sl.keep_max = keep_max(100.f, p.nn_local);                                    // TH_HIGH
            // the resolution kernel of the local search also writes the edge list of the second optimisation and hands the last frame's points to the ring
            const Laned<ChainTlmTail> tail = laned([&](int l) {
                const ChainLane& L = lanes[l];
                const ChainEdgesOut eo2{L.e_xw, L.e_obs, L.e_info, L.e_st, L.e_idx, L.cnt.n_edges2};
                return ChainTlmTail{L.match, L.q_f3a, L.lq.xw, L.ring, eo2, L.cnt.n_local_matches + k, cap, L.q_u8a, L.q_i, lane_value(last_desc, l),
                                    lane_value(last_pose, l)};
            });
            launch_search_local(cs, f, cell_start, csr_idx, lp, sl, ms, state, laned([&](int l) { return lanes[l].match_local; }),
                                laned([&](int l) { return lanes[l].scalars + kDevMatches; }), &tail, S); n_launches += 2;
            if (tm) cudaEventRecord(tev[4], cs);
            if (tm) cudaEventRecord(tev[5], cs);
            launch_pose_optimize(cs, laned([&](int l) { return pose_problem(l, true); }), work, e_lvl, e_out, pose_final, n_inliers, (k + 1 < m) ? &nxt : nullptr, S); ++n_launches;
            if (tm) cudaEventRecord(tev[6], cs);
        }
    }
    // carry each lane's last frame (keypoints, depths, descriptors, pose) for a continuing chain: one strided copy per array over the lanes
    const size_t lo = (size_t)(m - 1) * cap, kpb = (size_t)cap * sizeof(rgbl_keypoint), cb = sizeof(ChainCarry), pb = 7 * sizeof(float);
    CU(cudaMemcpy2DAsync(t.c_kps, kpb, s.s_kps + lo, m * kpb, kpb, S, cudaMemcpyDeviceToDevice, cs));
    CU(cudaMemcpy2DAsync(t.c_desc, (size_t)cap * 32, s.s_desc + lo * 32, (size_t)m * cap * 32, (size_t)cap * 32, S, cudaMemcpyDeviceToDevice, cs));
    CU(cudaMemcpy2DAsync(t.c_depth, (size_t)cap * sizeof(float), s.s_depth + lo, (size_t)m * cap * sizeof(float), (size_t)cap * sizeof(float), S, cudaMemcpyDeviceToDevice, cs));
    CU(cudaMemcpy2DAsync(&L0.carry->n_sel, cb, s.s_nsel + (m - 1), m * sizeof(int), sizeof(int), S, cudaMemcpyDeviceToDevice, cs));
    // ... and the pose before it (motion model of the next chain's first frame): frame m - 2, or the previously carried pose for a one-frame lane
    if (m >= 2) CU(cudaMemcpy2DAsync(L0.carry->prev_pose, cb, pose_of(0, m - 2), m * pb, pb, S, cudaMemcpyDeviceToDevice, cs));
    else if (cont) CU(cudaMemcpy2DAsync(L0.carry->prev_pose, cb, L0.carry->pose, cb, pb, S, cudaMemcpyDeviceToDevice, cs));
    CU(cudaMemcpy2DAsync(L0.carry->pose, cb, pose_of(0, m - 1), m * pb, pb, S, cudaMemcpyDeviceToDevice, cs));
    if (chain_timing) c->chain_timing_recorded = true;
    if (lane_layout_broken()) { lane_layout_broken() = false; c->err = "internal error: a sequence lane's chain arguments are not equally spaced"; return RGBL_E_CUDA; }
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(s.h_f + kChainPose0Floats, poses, (size_t)nF * 7 * sizeof(float), cudaMemcpyDeviceToHost, cs));
    CU(cudaMemcpyAsync(s.h_i, t.ch_counts, chain_count_ints(nF, S) * sizeof(int), cudaMemcpyDeviceToHost, cs));
    return RGBL_OK;
}

// Puts the chain on the tracking stream: the slot's graph (captured again when its key changed), or the launches themselves.
static int launch_chain(Ctx* c, const ChainPlan& p, int slot, const ChainSlot& s, int& n_launches) {
    const cudaStream_t cs = c->st_trk;
    if (!c->chain_graphs_on || c->chain_timing_on) return enqueue_chain(c, p, s, n_launches);
    ChainGraphKey key{};
    key.plan = p; key.generation = c->scratch_generation;
    if (!c->chain_exec[slot] || std::memcmp(&key, &c->chain_key[slot], sizeof(key)) != 0) {
        c->chain_exec[slot].reset();
        prepare_match_kernels();
        CU(cudaStreamBeginCapture(cs, cudaStreamCaptureModeRelaxed));
        const int rc_cap = enqueue_chain(c, p, s, n_launches);
        cudaGraph_t graph = nullptr;
        const cudaError_t e_cap = cudaStreamEndCapture(cs, &graph);
        if (rc_cap != RGBL_OK || e_cap != cudaSuccess || !graph) {
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError();
            if (rc_cap == RGBL_OK) c->err = std::string("chain graph capture failed: ") + cudaGetErrorString(e_cap);
            return rc_cap != RGBL_OK ? rc_cap : RGBL_E_CUDA;
        }
        const cudaError_t e_inst = c->chain_exec[slot].instantiate(graph);
        cudaGraphDestroy(graph);
        if (e_inst != cudaSuccess) { c->err = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e_inst); return RGBL_E_CUDA; }
        c->chain_key[slot] = key;
        c->chain_graph_launches[slot] = n_launches;
    }
    n_launches = c->chain_graph_launches[slot];
    CU(cudaGraphLaunch(c->chain_exec[slot], cs));
    return RGBL_OK;
}

static int chain_begin(Ctx* c, const rgbl_chain_params& P) {
    ChainPlan p{};
    int rc = check_chain(c, P, p); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = ensure_chain_resources(c, p); if (rc) return rc;
    const int slot = (c->chain_head + c->chain_pending) & 1;
    const ChainSlot s = chain_slot(c, slot);
    rc = snapshot_batch(c, p, slot, s); if (rc) return rc;
    for (int l = 0; l < p.lanes; ++l)
        for (int i = 0; i < 7; ++i) s.h_f[7 * l + i] = c->lane_pose0_set ? c->lane_pose0[l][i] : P.pose0[i];
    // stage timing events stay outside the graph (events recorded by graph nodes cannot be used for cudaEventElapsedTime)
    if (c->prof_on) CU(cudaEventRecord(c->ev_chain_b[slot], c->st_trk));
    int n_launches = 0;
    rc = launch_chain(c, p, slot, s, n_launches); if (rc) return rc;
    if (c->prof_on) CU(cudaEventRecord(c->ev_chain_e[slot], c->st_trk));
    CU(cudaEventRecord(c->ev_chain_done[slot], c->st_trk));
    c->chain_frames[slot] = p.nF;
    c->chain_lanes[slot] = p.lanes;
    c->chain_first[slot] = p.cont ? 0 : 1;
    c->chain_launches[slot] = n_launches;
    c->chain_pending += 1;
    c->chain_has_carry = true; c->carry_K = p.K; c->carry_cap = p.cap; c->carry_lanes = p.lanes;
    c->carry_prev_valid = (p.m >= 2) || p.cont;
    return RGBL_OK;
}

extern "C" {

int rgbl_resident_track_begin2(rgbl_ctx* ctx, const rgbl_chain_params* prm) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!prm) { c->err = "null argument"; return RGBL_E_INVALID; }
    return chain_begin(c, *prm);
}

int rgbl_resident_track_begin(rgbl_ctx* ctx, const float pose0[7], float fx, float fy, float cx, float cy, float bf, float th, int mono) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!pose0) { c->err = "null argument"; return RGBL_E_INVALID; }
    rgbl_chain_params p{};
    std::memcpy(p.pose0, pose0, 7 * sizeof(float));
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = bf; p.th_last = th; p.mono = mono;
    p.continue_sequence = 0; p.local_map_frames = 0; p.th_local = 3.f; p.nn_ratio_local = 0.8f;
    return chain_begin(c, p);
}

int rgbl_resident_track_end2(rgbl_ctx* ctx, float* poses_out, int* n_matches, int* n_inliers, int* n_local_matches, int* n_inliers_first) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!poses_out || !n_matches || !n_inliers) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (!c->chain_pending) { c->err = "no tracking chain in flight"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    const int slot = c->chain_head;
    c->chain_head ^= 1;
    c->chain_pending -= 1;
    CU(cudaEventSynchronize(c->ev_chain_done[slot]));            // the oldest chain only: a younger one may still be running
    const int nF = c->chain_frames[slot], S = c->chain_lanes[slot];
    const ChainSlot s = chain_slot(c, slot);
    const ChainCounts cnt = chain_counts(s.h_i, nF, nF / S, 0);
    if (c->chain_timing_recorded && c->chain_pending == 0) {
        const Event* e = c->chain_tev;
        const char* names[6] = {"chain_prep (first frame only)", "search_last (collect+resolve+edges)", "pose_optimize #1", "tlm_prepare + search_local (+edges, hand-over)", "-", "pose_optimize #2"};
        for (int i = 0; i < 6; ++i) { float ms = 0; if (cudaEventElapsedTime(&ms, e[i], e[i + 1]) == cudaSuccess) std::fprintf(stderr, "[chain timing] %-36s %8.2f us\n", names[i], ms * 1e3f); }
        cudaGetLastError();
    }
    std::memcpy(poses_out, s.h_f + kChainPose0Floats, (size_t)nF * 7 * sizeof(float));
    std::memcpy(n_matches, cnt.n_matches, (size_t)nF * sizeof(int));
    std::memcpy(n_inliers, cnt.n_inliers, (size_t)nF * sizeof(int));
    if (n_local_matches) std::memcpy(n_local_matches, cnt.n_local_matches, (size_t)nF * sizeof(int));
    if (n_inliers_first) std::memcpy(n_inliers_first, cnt.n_inliers_first, (size_t)nF * sizeof(int));
    c->total_launches += c->chain_launches[slot];
    c->chain_tracked_frames += nF - S * c->chain_first[slot];
    if (c->prof_on) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, c->ev_chain_b[slot], c->ev_chain_e[slot]) == cudaSuccess) {
            c->st_ms[ST_MATCH] += ms; c->st_calls[ST_MATCH] += 1; c->st_launches[ST_MATCH] += c->chain_launches[slot];
        } else {
            cudaGetLastError();
        }
    }
    for (int l = 0; l < S; ++l) {      // the overflow word of each lane
        const int ovf = *chain_counts(s.h_i, nF, nF / S, l).overflow;
        const std::string lane = S > 1 ? " (sequence lane " + std::to_string(l) + ")" : "";
        if (ovf == kTlmWaitFailed) { c->err = "TrackLocalMap compaction: a CTA waited in vain for its predecessors (chain_kernels.cu)" + lane; return RGBL_E_CUDA; }
        if (ovf) { c->err = "matcher candidate list overflow" + lane; return RGBL_E_CAPACITY; }
    }
    // capacity overflow of the frame construction that produced this batch (FAST cell slots, candidate buffer, quad-tree): the chain
    // ran on truncated keypoint sets
    if (c->h_chain_ovf[2 * slot] || c->h_chain_ovf[2 * slot + 1]) { c->err = "frame-construction capacity overflow in the batch this chain tracked"; return RGBL_E_CAPACITY; }
    return RGBL_OK;
}

int rgbl_set_sequences(rgbl_ctx* ctx, int n_sequences, const float* pose0) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (n_sequences < 1 || n_sequences > RGBL_MAX_SEQUENCES) { c->err = "n_sequences must be 1.." + std::to_string(RGBL_MAX_SEQUENCES); return RGBL_E_INVALID; }
    if (pose0)
        for (int i = 0; i < 7 * n_sequences; ++i)
            if (!std::isfinite(pose0[i])) { c->err = "pose0 holds a non-finite value"; return RGBL_E_INVALID; }
    c->lanes = n_sequences;
    c->lane_pose0_set = pose0 != nullptr;
    if (pose0) for (int l = 0; l < n_sequences; ++l) std::memcpy(c->lane_pose0[l], pose0 + 7 * l, 7 * sizeof(float));
    return RGBL_OK;
}

int rgbl_sequence_lanes_resident(rgbl_ctx* ctx, int* n_lanes) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!n_lanes) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (const char* why = pose_cluster_unsupported(c->cfg.device)) { c->err = why; return RGBL_E_UNSUPPORTED; }
    *n_lanes = pose_max_active_clusters(c->cfg.device);
    if (*n_lanes < 1) { c->err = "cudaOccupancyMaxActiveClusters failed"; return RGBL_E_CUDA; }
    return RGBL_OK;
}

int rgbl_resident_track_end(rgbl_ctx* ctx, float* poses_out, int* n_matches, int* n_inliers) {
    return rgbl_resident_track_end2(ctx, poses_out, n_matches, n_inliers, nullptr, nullptr);
}

int rgbl_resident_track(rgbl_ctx* ctx, const float pose0[7], float fx, float fy, float cx, float cy, float bf, float th, int mono,
                        float* poses_out, int* n_matches, int* n_inliers) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!pose0 || !poses_out || !n_matches || !n_inliers) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (const int rc = require_idle(c)) return rc;
    const int rc = rgbl_resident_track_begin(ctx, pose0, fx, fy, cx, cy, bf, th, mono);
    if (rc) return rc;
    return rgbl_resident_track_end(ctx, poses_out, n_matches, n_inliers);
}

}  // extern "C"
