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

// uploads the frame view and builds its 64x48 grid; fills FrameDev
static int upload_frame(Ctx* c, const rgbl_frame_view* v, FrameDev& f) {
    if (!v || v->n < 0 || (v->n > 0 && (!v->keys_un || !v->uright || !v->desc)) || !v->scale_factors || v->n_levels < 1 || v->n_levels > RGBL_MAX_LEVELS) {
        c->err = "bad frame view"; return RGBL_E_INVALID;
    }
    int rc = ensure_frame(c, std::max(v->n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    if (v->n) {
        CU(cudaMemcpyAsync(t.keys, v->keys_un, (size_t)v->n * sizeof(rgbl_keypoint), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.uright, v->uright, (size_t)v->n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.desc, v->desc, (size_t)v->n * 32, cudaMemcpyHostToDevice, c->st));
    }
    c->h_scalars[0] = v->n;
    CU(cudaMemcpyAsync(t.scalars, c->h_scalars, sizeof(int), cudaMemcpyHostToDevice, c->st));
    f.n = t.scalars; f.keys = t.keys; f.uright = t.uright; f.desc = t.desc;
    f.min_x = v->min_x; f.max_x = v->max_x; f.min_y = v->min_y; f.max_y = v->max_y;
    f.inv_w = static_cast<float>(kGridCols) / static_cast<float>(v->max_x - v->min_x);      // src/Frame.cc:351-352
    f.inv_h = static_cast<float>(kGridRows) / static_cast<float>(v->max_y - v->min_y);
    f.n_levels = v->n_levels;
    for (int l = 0; l < v->n_levels; ++l) f.scale[l] = v->scale_factors[l];
    f.fx = v->fx; f.fy = v->fy; f.cx = v->cx; f.cy = v->cy; f.bf = v->bf;
    f.mb = v->bf / v->fx;                                                                     // src/Frame.cc:360
    f.log_scale_factor = v->log_scale_factor;
    stage_begin(c, ST_MATCH, c->st);
    launch_grid_build(c->st, f, t.cell_start, t.csr_idx, t.kp_cell);
    return RGBL_OK;
}

static MatchScratch scratch(Ctx* c) {
    TrackBufs& t = c->trk;
    MatchScratch s;
    s.lists = t.lists; s.list_cap = kMatchListCap; s.list_n = t.list_n; s.minq = t.minq; s.choice = t.choice; s.resolved = t.resolved;
    s.overflow = c->d_overflow; s.rounds = t.scalars + 2; s.slots = t.list_slots; s.inv_cnt = t.inv_cnt; s.total = t.inv_cnt + (t.inv_cnt.size() - 1);
    s.dense = t.dense; s.dense_slot = t.dense_slot; s.dense_q = t.dense_q; s.base = t.list_base;
    return s;
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
    if (n_frame) CU(cudaMemcpyAsync(match, t.match, (size_t)n_frame * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_scalars + 4, t.scalars + 1, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_overflow, c->d_overflow, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    if (*c->h_overflow) {
        cudaMemsetAsync(c->d_overflow, 0, sizeof(int), c->st);
        c->err = "matcher candidate list overflow (> 512 admissible candidates for one map point)";
        return RGBL_E_CAPACITY;
    }
    if (n_matches) *n_matches = c->h_scalars[4];
    c->last_match_rounds = c->h_scalars[5];
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
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!cur || !cur_pose || !last_pose || n_last < 0 || !match || (n_last > 0 && (!valid || !xw || !mp_desc || !last_octave || !last_angle || !obs_pos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n_last, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    if (n_last) {
        CU(cudaMemcpyAsync(t.q_u8a, valid, n_last, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f3a, xw, (size_t)n_last * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_desc, mp_desc, (size_t)n_last * 32, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_i, last_octave, (size_t)n_last * sizeof(int), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[0], last_angle, (size_t)n_last * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_u8b, obs_pos, n_last, cudaMemcpyHostToDevice, c->st));
    }
    if (cur->n) {
        if (cur_state) CU(cudaMemcpyAsync(t.state, cur_state, cur->n, cudaMemcpyHostToDevice, c->st));
        else CU(cudaMemsetAsync(t.state, 0, cur->n, c->st));
    }
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
    if (n_last == 0) { CU(cudaMemsetAsync(t.match, 0xff, (size_t)std::max(cur->n, 1) * sizeof(int), c->st)); CU(cudaMemsetAsync(t.scalars + 1, 0, 2 * sizeof(int), c->st)); }
    launch_search_last(c->st, f, t.cell_start, t.csr_idx, lf, prm, scratch(c), t.state, t.match, t.scalars + 1);
    return finish_search(c, cur->n, match, n_matches);
}

int rgbl_is_in_frustum(rgbl_ctx* ctx, const rgbl_frame_view* cur, const float Rcw[9], const float tcw[3], const float Ow[3], int n,
                       const float* xw, const float* normal, const float* mf_min_dist, const float* mf_max_dist, float cos_limit,
                       uint8_t* in_view, float* proj_x, float* proj_y, float* proj_xr, float* track_depth, int32_t* level, float* view_cos) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!cur || !Rcw || !tcw || !Ow || n < 0 || (n > 0 && (!xw || !normal || !mf_min_dist || !mf_max_dist || !in_view || !proj_x || !proj_y || !proj_xr || !track_depth || !level || !view_cos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (n == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    int rc = ensure_queries(c, n); if (rc) return rc;
    TrackBufs& t = c->trk;
    FrameDev f{};
    f.min_x = cur->min_x; f.max_x = cur->max_x; f.min_y = cur->min_y; f.max_y = cur->max_y;
    f.n_levels = cur->n_levels; f.fx = cur->fx; f.fy = cur->fy; f.cx = cur->cx; f.cy = cur->cy; f.bf = cur->bf;
    f.log_scale_factor = cur->log_scale_factor;
    FrustumParams prm;
    std::memcpy(prm.Rcw, Rcw, 9 * sizeof(float)); std::memcpy(prm.tcw, tcw, 3 * sizeof(float)); std::memcpy(prm.Ow, Ow, 3 * sizeof(float));
    prm.cos_limit = cos_limit;
    CU(cudaMemcpyAsync(t.q_f3a, xw, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f3b, normal, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f[4], mf_min_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f[5], mf_max_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    stage_begin(c, ST_MATCH, c->st);
    launch_frustum(c->st, f, prm, n, t.q_f3a, t.q_f3b, t.q_f[4], t.q_f[5], t.q_u8a, t.q_f[0], t.q_f[1], t.q_f[2], t.q_f[3], t.q_i, t.q_f[6]);
    stage_end(c, ST_MATCH, c->st, 1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(in_view, t.q_u8a, n, cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(proj_x, t.q_f[0], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(proj_y, t.q_f[1], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(proj_xr, t.q_f[2], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(track_depth, t.q_f[3], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(level, t.q_i, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(view_cos, t.q_f[6], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_search_by_projection_local(rgbl_ctx* ctx, const rgbl_frame_view* cur, int n, const uint8_t* in_view, const float* proj_x,
                                    const float* proj_y, const float* proj_xr, const float* track_depth, const int32_t* level,
                                    const float* view_cos, const uint8_t* mp_desc, const uint8_t* obs_pos, float th, float nn_ratio,
                                    int far_points, float th_far, const uint8_t* cur_state, int32_t* match, int* n_matches) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!cur || n < 0 || !match || (n > 0 && (!in_view || !proj_x || !proj_y || !proj_xr || !track_depth || !level || !view_cos || !mp_desc || !obs_pos))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (!(nn_ratio > 0.f)) { c->err = "nn_ratio must be > 0"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    if (n) {
        CU(cudaMemcpyAsync(t.q_u8a, in_view, n, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[0], proj_x, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[1], proj_y, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[2], proj_xr, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[3], track_depth, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_i, level, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[4], view_cos, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_desc, mp_desc, (size_t)n * 32, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_u8b, obs_pos, n, cudaMemcpyHostToDevice, c->st));
    }
    if (cur->n) {
        if (cur_state) CU(cudaMemcpyAsync(t.state, cur_state, cur->n, cudaMemcpyHostToDevice, c->st));
        else CU(cudaMemsetAsync(t.state, 0, cur->n, c->st));
    }
    SearchLocalParams prm;
    prm.th = th; prm.nn_ratio = nn_ratio; prm.th_far = th_far; prm.far_points = far_points;
    prm.use_factor = (th != 1.0) ? 1 : 0;                                         // bFactor, src/ORBmatcher.cc:47
    // a second-best beyond TH_HIGH / nnratio can never reject: best <= TH_HIGH < nnratio * second
    prm.keep_max = std::min(256, (int)std::floor((float)100 / nn_ratio) + 1);
    LocalPointsDev lp{n, nullptr, t.q_u8a, t.q_f[0], t.q_f[1], t.q_f[2], t.q_f[3], t.q_i, t.q_f[4], t.q_desc, t.q_u8b};
    if (n == 0) { CU(cudaMemsetAsync(t.match, 0xff, (size_t)std::max(cur->n, 1) * sizeof(int), c->st)); CU(cudaMemsetAsync(t.scalars + 1, 0, 2 * sizeof(int), c->st)); }
    launch_search_local(c->st, f, t.cell_start, t.csr_idx, lp, prm, scratch(c), t.state, t.match, t.scalars + 1);
    return finish_search(c, cur->n, match, n_matches);
}

int rgbl_pose_optimize(rgbl_ctx* ctx, const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2,
                       const uint8_t* stereo, float fx, float fy, float cx, float cy, float bf, float pose_out[7], uint8_t* outlier,
                       int* n_inliers) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!pose_in || !pose_out || n < 0 || !n_inliers || (n > 0 && (!xw || !obs || !inv_sigma2 || !stereo || !outlier))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (const char* why = pose_cluster_unsupported(c->cfg.device)) { c->err = why; return RGBL_E_UNSUPPORTED; }
    CU(cudaSetDevice(c->cfg.device));
    int rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    rc = ensure_frame(c, 1); if (rc) return rc;
    TrackBufs& t = c->trk;
    GROW(t.pose_work, (size_t)std::max(n, 1) * 3);
    if (n) {
        CU(cudaMemcpyAsync(t.q_f3a, xw, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f3b, obs, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[0], inv_sigma2, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_u8a, stereo, n, cudaMemcpyHostToDevice, c->st));
    }
    PoseProblemDev p;
    p.n = n; p.xw = t.q_f3a; p.obs = t.q_f3b; p.inv_sigma2 = t.q_f[0]; p.stereo = t.q_u8a;
    p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = bf; p.n_dev = nullptr; p.pose_in_dev = nullptr;
    std::memcpy(p.pose_in, pose_in, 7 * sizeof(float));
    stage_begin(c, ST_POSE, c->st);
    launch_pose_optimize(c->st, p, t.pose_work, t.q_u8b, t.resolved, t.q_f[1], reinterpret_cast<int*>(t.scalars + 8));
    stage_end(c, ST_POSE, c->st, 1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(pose_out, t.q_f[1], 7 * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    if (n >= 3) CU(cudaMemcpyAsync(outlier, t.resolved, n, cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_scalars + 8, t.scalars + 8, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    *n_inliers = c->h_scalars[8];
    return RGBL_OK;
}


int rgbl_fuse_search(rgbl_ctx* ctx, const rgbl_frame_view* kf, const float Tcw[7], const float Ow[3], int n, const uint8_t* valid, const float* xw,
                     const float* normal, const float* mf_min_dist, const float* mf_max_dist, const uint8_t* mp_desc, float th, int32_t* best_idx,
                     int32_t* best_dist) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
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
    CU(cudaMemcpyAsync(t.q_u8a, valid, n, cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f3a, xw, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f3b, normal, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f[0], mf_min_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f[1], mf_max_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_desc, mp_desc, (size_t)n * 32, cudaMemcpyHostToDevice, c->st));
    float* hp = reinterpret_cast<float*>(c->h_scalars + 4);       // pinned staging (ints 4..13; [0] carries the frame size): pose + camera centre
    for (int i = 0; i < 7; ++i) hp[i] = Tcw[i];
    for (int i = 0; i < 3; ++i) hp[7 + i] = Ow[i];
    CU(cudaMemcpyAsync(t.q_f[2], hp, 10 * sizeof(float), cudaMemcpyHostToDevice, c->st));
    launch_fuse_search(c->st, f, t.cell_start, t.csr_idx, n, t.q_u8a, t.q_f3a, t.q_f3b, t.q_f[0], t.q_f[1], t.q_desc, t.q_f[2], t.q_f[2] + 7, th,
                       t.e_idx, t.e_idx + n);
    stage_end(c, ST_MATCH, c->st, 2);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(best_idx, t.e_idx, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(best_dist, t.e_idx + n, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_stereo_matches(rgbl_ctx* ctx, int slot_left, int slot_right, float mb, float mbf, float* depth, float* uright, int cap) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!depth || !uright) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (slot_left < 0 || slot_right < 0 || slot_left >= c->last_frames || slot_right >= c->last_frames) { c->err = "frame slot out of range (extract the stereo pair as one batch first)"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    int rc = stereo_matches(c, slot_left, slot_right, 1, mb, mbf); if (rc) return rc;
    float* d_depth = c->d_depth + (size_t)slot_left * c->cap_kp;
    float* d_ur = c->d_uright + (size_t)slot_left * c->cap_kp;
    CU(cudaMemcpyAsync(c->h_scalars, c->d_n_sel + slot_left, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    const int n = c->h_scalars[0];
    if (n > cap) { c->err = "output capacity too small"; return RGBL_E_CAPACITY; }
    if (n) {
        CU(cudaMemcpyAsync(depth, d_depth, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(uright, d_ur, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    }
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
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
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
    CU(cudaMemcpyAsync(t.q_desc, kf_desc, (size_t)n_kf * 32, cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.desc, f_desc, (size_t)n_f * 32, cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.uright, f_angle, (size_t)n_f * sizeof(float), cudaMemcpyHostToDevice, c->st));       // reused as F angles
    CU(cudaMemcpyAsync(t.csr_idx, f_node_feat, (size_t)n_fcsr * sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.e_idx, q_feat.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.e_idx + n_q, q_cbeg.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.e_idx + 2 * n_q, q_cend.data(), (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(t.q_f[0], q_ang.data(), (size_t)n_q * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemsetAsync(t.q_u8b, 1, n_q, c->st));                                                              // every assignment blocks
    CU(cudaMemsetAsync(t.state, 0, n_f, c->st));
    c->h_scalars[0] = n_f;
    CU(cudaMemcpyAsync(t.scalars, c->h_scalars, sizeof(int), cudaMemcpyHostToDevice, c->st));
    FrameDev f{};
    f.n = t.scalars;
    // a second-best beyond TH_LOW / nnratio can never reject: best <= TH_LOW < nnratio * second
    const int keep_max = std::min(256, (int)std::floor(50.0f / nn_ratio) + 1);
    stage_begin(c, ST_MATCH, c->st);
    launch_search_bow(c->st, f, n_q, t.e_idx, t.e_idx + n_q, t.e_idx + 2 * n_q, t.q_desc, t.desc, t.q_f[0], t.uright, t.csr_idx, nn_ratio, keep_max,
                      check_orientation, t.q_u8b, scratch(c), t.state, t.match, t.scalars + 1);
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
    if (!c) return RGBL_E_INVALID;
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    if (!cur || !cur_pose || n < 0 || !match || (n > 0 && (!valid || !xw || !mp_desc || !kf_angle || !mf_min_dist || !mf_max_dist))) { c->err = "null argument"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    FrameDev f;
    int rc = upload_frame(c, cur, f); if (rc) return rc;
    rc = ensure_queries(c, std::max(n, 1)); if (rc) return rc;
    TrackBufs& t = c->trk;
    if (n) {
        CU(cudaMemcpyAsync(t.q_u8a, valid, n, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f3a, xw, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_desc, mp_desc, (size_t)n * 32, cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[0], kf_angle, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[4], mf_min_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(t.q_f[5], mf_max_dist, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemsetAsync(t.q_u8b, 1, n, c->st));
    }
    std::vector<uint8_t> st(std::max(cur->n, 1), 0);
    if (cur_occupied) for (int i = 0; i < cur->n; ++i) st[i] = cur_occupied[i] ? 1 : 0;        // any map point blocks (:1950-1951)
    if (cur->n) CU(cudaMemcpyAsync(t.state, st.data(), cur->n, cudaMemcpyHostToDevice, c->st));
    SearchRelocParams prm;
    std::memcpy(prm.cur_pose, cur_pose, 7 * sizeof(float));
    {   // Ow = Tcw.inverse().translation()
        h_inverse_translation(cur_pose, prm.Ow);
    }
    prm.th = th; prm.orb_dist = orb_dist; prm.check_orientation = check_orientation;
    RelocPointsDev rp{n, t.q_u8a, t.q_f3a, t.q_desc, t.q_f[0], t.q_f[4], t.q_f[5]};
    if (n == 0) { CU(cudaMemsetAsync(t.match, 0xff, (size_t)std::max(cur->n, 1) * sizeof(int), c->st)); CU(cudaMemsetAsync(t.scalars + 1, 0, 2 * sizeof(int), c->st)); }
    launch_search_reloc(c->st, f, t.cell_start, t.csr_idx, rp, prm, t.q_u8b, scratch(c), t.state, t.match, t.scalars + 1);
    CU(cudaStreamSynchronize(c->st));      // `st` (host vector) must outlive the async copy
    return finish_search(c, cur->n, match, n_matches);
}

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
static int chain_begin(Ctx* c, const rgbl_chain_params& cp_) {
    const rgbl_chain_params P = cp_;
    const float fx = P.fx, fy = P.fy, cx = P.cx, cy = P.cy, bf = P.bf, th = P.th_last;
    const int mono = P.mono, K = std::max(P.local_map_frames, 0);
    if (c->chain_pending >= 2) { c->err = "two tracking chains are already queued: call rgbl_resident_track_end first"; return RGBL_E_INVALID; }
    if (const char* why = pose_cluster_unsupported(c->cfg.device)) { c->err = why; return RGBL_E_UNSUPPORTED; }
    const int nF = c->last_frames, cap = c->cap_kp;
    const int slot = (c->chain_head + c->chain_pending) & 1;
    if (nF < 1) { c->err = "nothing processed"; return RGBL_E_INVALID; }
    if (K > 16) { c->err = "local_map_frames > 16"; return RGBL_E_INVALID; }
    const bool cont = P.continue_sequence != 0;
    if (cont && !c->chain_has_carry) { c->err = "continue_sequence without a previous chain on this context"; return RGBL_E_INVALID; }
    if (cont && (c->carry_K != K || c->carry_cap != cap)) { c->err = "continue_sequence: local_map_frames / keypoint capacity differ from the previous chain"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    // the tracking stream and the chain's events: each one created by the first chain that finds it missing
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
    const size_t n_counts = (size_t)4 * nF + 8;          // n_matches | n_inliers | n_local_matches | n_inliers_first | ne, ne2, flags[2], overflow, nq
    if (c->h_chain_cap < (size_t)nF) {
        if (c->chain_pending) { c->err = "batch size grew while a chain is in flight"; return RGBL_E_INVALID; }
        const size_t capF = (size_t)std::max(nF, c->cfg.max_batch), nf = 2 * (7 + capF * 7), ni = 2 * (4 * capF + 8);
        c->h_chain_cap = 0;
        if (!c->h_chain_f.grow(nf, c->scratch_generation, nf) || !c->h_chain_i.grow(ni, c->scratch_generation, ni)) {
            c->err = "pinned allocation failed (chain result staging)"; return RGBL_E_CUDA;
        }
        c->h_chain_cap = capF;
    }
    int rc = ensure_frame(c, cap); if (rc) return rc;
    const int n_lq = std::max(K * cap, 1);                // local-search queries (compacted, at most every ring point)
    rc = ensure_queries(c, std::max(cap, n_lq)); if (rc) return rc;
    TrackBufs& t = c->trk;
    const size_t tot = (size_t)nF * cap;
    GROW(t.pose_work, (size_t)cap * 3);
    GROW(t.ch_poses, (size_t)nF * 7 + 14); GROW(t.ch_counts, n_counts);      // poses | pose after TrackWithMotionModel | predicted pose
    GROW(t.e_xw, (size_t)cap * 3); GROW(t.e_obs, (size_t)cap * 3); GROW(t.e_info, cap);
    GROW(t.e_st, cap); GROW(t.e_lvl, cap); GROW(t.e_out, cap); GROW(t.e_idx, cap);
    // carried last frame of the sequence + the local map ring (persist across chains of this context)
    GROW(t.c_kps, cap); GROW(t.c_desc, (size_t)cap * 32); GROW(t.c_depth, cap);
    GROW(t.c_misc, 16);                     // int n_sel | float pose[7] (as raw 32-bit words) | ring count | float prev_pose[7]
    if (K > 0) {
        const size_t nr = (size_t)K * cap;
        if (cont && t.r_valid.size() < nr) { c->err = "local map ring missing"; return RGBL_E_INVALID; }
        GROW(t.r_valid, nr); GROW(t.r_xw, nr * 3); GROW(t.r_normal, nr * 3);
        GROW(t.r_min, nr); GROW(t.r_max, nr); GROW(t.r_desc, nr * 32);
        GROW(t.lq_u8, 2 * (size_t)n_lq); GROW(t.lq_f, 8 * (size_t)n_lq); GROW(t.lq_i, 2 * (size_t)n_lq);
        GROW(t.lq_desc, (size_t)n_lq * 32); GROW(t.match_local, cap);
        if (!t.lookback) {
            GROW(t.lookback, tlm_lookback_ints());
            CU(cudaMemsetAsync(t.lookback, 0, t.lookback.size() * sizeof(int), c->st));     // ordered before the chain by ev_snap below
        }
        if ((n_lq + 255) / 256 + 1 > 1024) { c->err = "local map too large for the compaction slots (local_map_frames x keypoint capacity > 261 k)"; return RGBL_E_UNSUPPORTED; }
    }
    // per-slot buffers: twice the size, the slot picks its half (sizes are those of the context's full batch so that the halves
    // never move while a chain is in flight)
    const size_t tot_full = (size_t)std::max(nF, c->cfg.max_batch) * cap, nF_full = (size_t)std::max(nF, c->cfg.max_batch);
    const size_t cs_full = nF_full * (kGridCols * kGridRows + 1);
    if (c->chain_pending && (t.s_kps.size() < 2 * tot_full || t.b_cell_start.size() < 2 * cs_full)) { c->err = "batch size grew while a chain is in flight"; return RGBL_E_INVALID; }
    GROW(t.s_kps, 2 * tot_full); GROW(t.s_desc, 2 * tot_full * 32); GROW(t.s_depth, 2 * tot_full);
    GROW(t.s_uright, 2 * tot_full); GROW(t.s_nsel, 2 * nF_full);
    GROW(t.b_cell_start, 2 * cs_full);
    GROW(t.b_csr_idx, 2 * tot_full); GROW(t.b_kp_cell, 2 * tot_full);
    rgbl_keypoint* s_kps = t.s_kps + slot * tot_full; uint8_t* s_desc = t.s_desc + slot * tot_full * 32;
    float* s_depth = t.s_depth + slot * tot_full; float* s_uright = t.s_uright + slot * tot_full; int* s_nsel = t.s_nsel + slot * nF_full;
    int* b_cell_start = t.b_cell_start + slot * cs_full; int* b_csr_idx = t.b_csr_idx + slot * tot_full; int* b_kp_cell = t.b_kp_cell + slot * tot_full;
    float* h_f = c->h_chain_f + (size_t)slot * (7 + c->h_chain_cap * 7);
    int* h_i = c->h_chain_i + (size_t)slot * (4 * c->h_chain_cap + 8);

    // snapshot on the frame-construction stream (ordered after the batch's kernels, before the next batch's)
    // mvKeysUn: the chain reads nothing but undistorted keypoints (grid, projections, edges, UnprojectStereo, ring, carried frame)
    CU(cudaMemcpyAsync(s_kps, c->frames_undistorted ? c->d_kps_un : c->d_kps, tot * sizeof(rgbl_keypoint), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s_desc, c->d_desc, tot * 32, cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s_depth, c->d_depth, tot * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s_uright, c->d_uright, tot * sizeof(float), cudaMemcpyDeviceToDevice, c->st));
    CU(cudaMemcpyAsync(s_nsel, c->d_n_sel, (size_t)nF * sizeof(int), cudaMemcpyDeviceToDevice, c->st));
    // the frame-construction overflow flags of THIS batch travel with the chain (checked in _end)
    CU(cudaMemcpyAsync(c->h_chain_ovf + 2 * slot, c->d_overflow, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaEventRecord(c->ev_snap, c->st));
    CU(cudaStreamWaitEvent(c->st_aux, c->ev_snap, 0));      // the aux stream writes depth / uright of the next batch
    cudaStream_t cs = c->st_trk;
    CU(cudaStreamWaitEvent(cs, c->ev_snap, 0));

    for (int i = 0; i < 7; ++i) h_f[i] = P.pose0[i];
    const bool chain_timing = c->chain_timing_on;
    const bool chain_graphs = c->chain_graphs_on;
    const Event* tev = c->chain_tev;
    int* c_nsel = reinterpret_cast<int*>(t.c_misc.get());
    float* c_pose = reinterpret_cast<float*>(t.c_misc.get()) + 1;
    int* r_count = reinterpret_cast<int*>(t.c_misc.get()) + 8;
    float* c_prev = reinterpret_cast<float*>(t.c_misc.get()) + 9;      // pose of the frame before the carried one (valid: c->carry_prev_valid)
    const bool prev_valid = cont && c->carry_prev_valid;
    int n_launches = 0;
    const float* bounds = c->frame_bounds;
    // Everything the chain does on the tracking stream.  It is captured ONCE per slot into a CUDA graph and
    // replayed: the launch commands then live in device memory, so the dependent-kernel sequence no longer fetches a command
    // packet from the host over PCIe per launch (which the concurrent H2D uploads of the next batch were slowing down) and
    // _begin costs one graph launch instead of hundreds of kernel launches on the host.
    auto enqueue_chain = [&]() -> int {
        n_launches = 0;
        float* poses = t.ch_poses;                 // frame k -> poses + 7 k
        float* pose_tmp = t.ch_poses + 7 * (size_t)nF;      // pose after TrackWithMotionModel (input of the second PoseOptimization)
        float* pose_pred = pose_tmp + 7;                    // the motion model's pose of the frame being tracked (written when the previous frame's pose is final)
        CU(cudaMemsetAsync(t.ch_counts, 0, n_counts * sizeof(int), cs));
        if (!cont) {
            CU(cudaMemcpyAsync(poses, h_f, 7 * sizeof(float), cudaMemcpyHostToDevice, cs));
            if (K > 0) { CU(cudaMemsetAsync(t.r_valid, 0, (size_t)K * cap, cs)); CU(cudaMemsetAsync(r_count, 0, sizeof(int), cs)); }
        }
        int* d_nm = t.ch_counts; int* d_ni = t.ch_counts + nF; int* d_nml = t.ch_counts + 2 * nF; int* d_ni1 = t.ch_counts + 3 * nF;
        int* d_ne = t.ch_counts + 4 * nF; int* d_ne2 = d_ne + 1; int* d_flags = d_ne + 2; int* d_ovf = d_ne + 4; int* d_nq = d_ne + 5;
        FrameDev f{};
        f.min_x = bounds[0]; f.max_x = bounds[1]; f.min_y = bounds[2]; f.max_y = bounds[3];      // ComputeImageBounds of the frames' camera
        f.inv_w = static_cast<float>(kGridCols) / static_cast<float>(f.max_x - f.min_x);
        f.inv_h = static_cast<float>(kGridRows) / static_cast<float>(f.max_y - f.min_y);
        f.n_levels = c->tab.nlevels;
        for (int l = 0; l < f.n_levels; ++l) f.scale[l] = c->tab.scale[l];
        f.fx = fx; f.fy = fy; f.cx = cx; f.cy = cy; f.bf = bf; f.mb = bf / fx;
        f.log_scale_factor = std::log(c->cfg.orb.scale_factor);
        MatchScratch ms = scratch(c);
        ms.overflow = d_ovf;
        // the 64x48 grids do not depend on the poses: all frames in one launch (one CTA per frame)
        f.n = s_nsel; f.keys = s_kps;
        launch_grid_build_batch(cs, f, nF, cap, b_cell_start, b_csr_idx, b_kp_cell); ++n_launches;
        // unprojection of frame j's keypoints (map points of the search in frame j + 1); j == -1: the carried frame
        auto prep_of = [&](int j) {
            ChainPrepDev cp{};
            if (j < 0) { cp.kps = t.c_kps; cp.depth = t.c_depth; cp.n_ptr = c_nsel; }
            else { cp.kps = s_kps + (size_t)j * cap; cp.depth = s_depth + (size_t)j * cap; cp.n_ptr = s_nsel + j; }
            cp.fx = f.fx; cp.fy = f.fy; cp.cx = f.cx; cp.cy = f.cy; cp.mb = f.mb; cp.mono = mono; cp.cap = cap;
            cp.valid = t.q_u8a; cp.xw = t.q_f3a; cp.octave = t.q_i; cp.angle = t.q_f[0]; cp.obs_pos = t.q_u8b; cp.flags = d_flags; cp.state_clear = t.state;
            // constant-velocity motion model: the pose of the frame before frame j (nullptr at the start of a sequence)
            if (j >= 1) cp.prev_pose = poses + 7 * (size_t)(j - 1);
            else if (j == 0) cp.prev_pose = cont ? c_pose : nullptr;
            else cp.prev_pose = prev_valid ? c_prev : nullptr;
            cp.pred_pose = pose_pred;
            return cp;
        };
        LocalRingDev ring{K, cap, t.r_valid, t.r_xw, t.r_normal, t.r_min, t.r_max, t.r_desc, r_count};
        LocalQueriesDev lq{};
        if (K > 0) {
            lq.cap = n_lq; lq.n = d_nq; lq.in_view = t.lq_u8; lq.obs_pos = t.lq_u8 + n_lq;
            lq.proj_x = t.lq_f; lq.proj_y = t.lq_f + n_lq; lq.proj_xr = t.lq_f + 2 * (size_t)n_lq; lq.depth = t.lq_f + 3 * (size_t)n_lq;
            lq.view_cos = t.lq_f + 4 * (size_t)n_lq; lq.xw = t.lq_f + 5 * (size_t)n_lq; lq.level = t.lq_i; lq.src = t.lq_i + n_lq; lq.desc = t.lq_desc;
        }
        const int k0 = cont ? 0 : 1;
        for (int k = k0; k < nF; ++k) {
            const bool tm = chain_timing && k == std::max(1, nF / 2);
            const size_t cu = (size_t)k * cap;
            const float* last_pose = (k == 0) ? c_pose : poses + 7 * (size_t)(k - 1);
            const uint8_t* last_desc = (k == 0) ? t.c_desc : s_desc + (size_t)(k - 1) * cap * 32;
            if (tm) cudaEventRecord(tev[0], cs);
            if (k == k0) { launch_chain_prep(cs, prep_of(k - 1), last_pose); ++n_launches; }   // later frames: prepared by the previous pose kernel
            f.n = s_nsel + k; f.keys = s_kps + cu; f.uright = s_uright + cu; f.desc = s_desc + cu * 32;
            const int* cell_start = b_cell_start + (size_t)k * (kGridCols * kGridRows + 1);
            const int* csr_idx = b_csr_idx + cu;
            if (tm) cudaEventRecord(tev[1], cs);
            SearchLastParams prm{};
            prm.th = th; prm.check_orientation = 1; prm.cur_pose_dev = pose_pred; prm.flags_dev = d_flags;      // projected with the motion model's pose (src/Tracking.cc:2904)
            LastFrameDev lf{cap, t.q_u8a, t.q_f3a, last_desc, t.q_i, t.q_f[0], t.q_u8b};
            const ChainEdgesOut eo{t.e_xw, t.e_obs, t.e_info, t.e_st, t.e_idx, d_ne};
            launch_search_last(cs, f, cell_start, csr_idx, lf, prm, ms, t.state, t.match, d_nm + k, &eo); n_launches += 2;   // + edges of the matches
            if (tm) cudaEventRecord(tev[2], cs);
            PoseProblemDev p{};
            p.n = 0; p.n_dev = d_ne; p.pose_in_dev = pose_pred;
            p.xw = t.e_xw; p.obs = t.e_obs; p.inv_sigma2 = t.e_info; p.stereo = t.e_st;
            p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = bf;
            const ChainPrepDev nxt = prep_of(k);
            if (K == 0) {
                launch_pose_optimize(cs, p, t.pose_work, t.e_lvl, t.e_out, poses + 7 * (size_t)k, d_ni + k, (k + 1 < nF) ? &nxt : nullptr); ++n_launches;
                if (tm) { cudaEventRecord(tev[3], cs); cudaEventRecord(tev[4], cs); cudaEventRecord(tev[5], cs); cudaEventRecord(tev[6], cs); }
            } else {
                launch_pose_optimize(cs, p, t.pose_work, t.e_lvl, t.e_out, pose_tmp, d_ni1 + k, nullptr); ++n_launches;
                if (tm) cudaEventRecord(tev[3], cs);
                // TrackLocalMap: outlier discard + isInFrustum + ordered compaction, local search, edges of all map points, second optimisation
                launch_tlm_prepare(cs, f, pose_tmp, ring, 0.5f, d_ne, t.e_idx, t.e_out, t.state, t.match, lq, t.lookback, d_ovf); ++n_launches;
                LocalPointsDev lp{n_lq, d_nq, lq.in_view, lq.proj_x, lq.proj_y, lq.proj_xr, lq.depth, lq.level, lq.view_cos, lq.desc, lq.obs_pos};
                SearchLocalParams sl{};
                sl.th = P.th_local; sl.nn_ratio = P.nn_ratio_local; sl.th_far = 0.f; sl.use_factor = (P.th_local != 1.0f) ? 1 : 0; sl.far_points = 0; sl.keep_max = std::min(256, (int)std::floor((float)100 / P.nn_ratio_local) + 1);
                // the resolution kernel of the local search also writes the edge list of the second optimisation and hands the last frame's points to the ring
                const ChainEdgesOut eo2{t.e_xw, t.e_obs, t.e_info, t.e_st, t.e_idx, d_ne2};
                const ChainTlmTail tail{t.match, t.q_f3a, lq.xw, ring, eo2, d_nml + k, cap, t.q_u8a, t.q_i, last_desc, last_pose};
                launch_search_local(cs, f, cell_start, csr_idx, lp, sl, ms, t.state, t.match_local, t.scalars + 1, &tail); n_launches += 2;
                if (tm) cudaEventRecord(tev[4], cs);
                if (tm) cudaEventRecord(tev[5], cs);
                PoseProblemDev p2 = p;
                p2.n_dev = d_ne2; p2.pose_in_dev = pose_tmp;
                launch_pose_optimize(cs, p2, t.pose_work, t.e_lvl, t.e_out, poses + 7 * (size_t)k, d_ni + k, (k + 1 < nF) ? &nxt : nullptr); ++n_launches;
                if (tm) cudaEventRecord(tev[6], cs);
            }
        }
        // carry the last frame of this batch (keypoints, depths, descriptors, pose) for a continuing chain
        const size_t lo = (size_t)(nF - 1) * cap;
        CU(cudaMemcpyAsync(t.c_kps, s_kps + lo, (size_t)cap * sizeof(rgbl_keypoint), cudaMemcpyDeviceToDevice, cs));
        CU(cudaMemcpyAsync(t.c_desc, s_desc + lo * 32, (size_t)cap * 32, cudaMemcpyDeviceToDevice, cs));
        CU(cudaMemcpyAsync(t.c_depth, s_depth + lo, (size_t)cap * sizeof(float), cudaMemcpyDeviceToDevice, cs));
        CU(cudaMemcpyAsync(c_nsel, s_nsel + (nF - 1), sizeof(int), cudaMemcpyDeviceToDevice, cs));
        // ... and the pose before it (motion model of the next chain's first frame): frame nF - 2, or the previously carried pose for a one-frame batch
        if (nF >= 2) CU(cudaMemcpyAsync(c_prev, poses + 7 * (size_t)(nF - 2), 7 * sizeof(float), cudaMemcpyDeviceToDevice, cs));
        else if (cont) CU(cudaMemcpyAsync(c_prev, c_pose, 7 * sizeof(float), cudaMemcpyDeviceToDevice, cs));
        CU(cudaMemcpyAsync(c_pose, poses + 7 * (size_t)(nF - 1), 7 * sizeof(float), cudaMemcpyDeviceToDevice, cs));
        if (chain_timing) c->chain_timing_recorded = true;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(h_f + 7, poses, (size_t)nF * 7 * sizeof(float), cudaMemcpyDeviceToHost, cs));
        CU(cudaMemcpyAsync(h_i, t.ch_counts, n_counts * sizeof(int), cudaMemcpyDeviceToHost, cs));
        return RGBL_OK;
    };
    // stage timing events stay outside the graph (events recorded by graph nodes cannot be used for cudaEventElapsedTime)
    if (c->prof_on) CU(cudaEventRecord(c->ev_chain_b[slot], cs));
    if (chain_graphs && !chain_timing) {
        Ctx::ChainGraphKey key{};
        key.nF = nF; key.cap = cap; key.mono = mono; key.cont = cont ? 1 : 0; key.K = K; key.prev_valid = prev_valid ? 1 : 0; key.th = th; key.th_local = P.th_local; key.nn_local = P.nn_ratio_local;
        key.fx = fx; key.fy = fy; key.cx = cx; key.cy = cy; key.bf = bf; std::memcpy(key.bounds, bounds, sizeof(key.bounds)); key.generation = c->scratch_generation;
        if (!c->chain_exec[slot] || std::memcmp(&key, &c->chain_key[slot], sizeof(key)) != 0) {
            c->chain_exec[slot].reset();
            prepare_match_kernels();
            CU(cudaStreamBeginCapture(cs, cudaStreamCaptureModeRelaxed));
            chain_launch_pdl() = c->chain_pdl_on;           // programmatic dependent launches between the chain's kernels (rgbl_device.cuh: pdl_wait)
            const int rc_cap = enqueue_chain();
            chain_launch_pdl() = false;
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
    } else {
        chain_launch_pdl() = c->chain_pdl_on;
        const int rc_q = enqueue_chain();
        chain_launch_pdl() = false;
        if (rc_q) return rc_q;
    }
    if (c->prof_on) CU(cudaEventRecord(c->ev_chain_e[slot], cs));
    CU(cudaEventRecord(c->ev_chain_done[slot], cs));
    c->chain_frames[slot] = nF;
    c->chain_first[slot] = cont ? 0 : 1;
    c->chain_launches[slot] = n_launches;
    c->chain_pending += 1;
    c->chain_has_carry = true; c->carry_K = K; c->carry_cap = cap;
    c->carry_prev_valid = (nF >= 2) || cont;
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
    const int nF = c->chain_frames[slot];
    const float* h_f = c->h_chain_f + (size_t)slot * (7 + c->h_chain_cap * 7);
    const int* h_i = c->h_chain_i + (size_t)slot * (4 * c->h_chain_cap + 8);
    if (c->chain_timing_recorded && c->chain_pending == 0) {
        const Event* e = c->chain_tev;
        const char* names[6] = {"chain_prep (first frame only)", "search_last (collect+resolve+edges)", "pose_optimize #1", "tlm_prepare + search_local (+edges, hand-over)", "-", "pose_optimize #2"};
        for (int i = 0; i < 6; ++i) { float ms = 0; if (cudaEventElapsedTime(&ms, e[i], e[i + 1]) == cudaSuccess) std::fprintf(stderr, "[chain timing] %-36s %8.2f us\n", names[i], ms * 1e3f); }
        cudaGetLastError();
    }
    std::memcpy(poses_out, h_f + 7, (size_t)nF * 7 * sizeof(float));
    std::memcpy(n_matches, h_i, (size_t)nF * sizeof(int));
    std::memcpy(n_inliers, h_i + nF, (size_t)nF * sizeof(int));
    if (n_local_matches) std::memcpy(n_local_matches, h_i + 2 * nF, (size_t)nF * sizeof(int));
    if (n_inliers_first) std::memcpy(n_inliers_first, h_i + 3 * nF, (size_t)nF * sizeof(int));
    c->total_launches += c->chain_launches[slot];
    c->chain_tracked_frames += nF - c->chain_first[slot];
    if (c->prof_on) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, c->ev_chain_b[slot], c->ev_chain_e[slot]) == cudaSuccess) {
            c->st_ms[ST_MATCH] += ms; c->st_calls[ST_MATCH] += 1; c->st_launches[ST_MATCH] += c->chain_launches[slot];
        } else {
            cudaGetLastError();
        }
    }
    if (h_i[4 * nF + 4] == 9) { c->err = "TrackLocalMap compaction: a CTA waited in vain for its predecessors (chain_kernels.cu)"; return RGBL_E_CUDA; }
    if (h_i[4 * nF + 4]) { c->err = "matcher candidate list overflow"; return RGBL_E_CAPACITY; }
    // capacity overflow of the frame construction that produced this batch (FAST cell slots, candidate buffer, quad-tree): the chain
    // ran on truncated keypoint sets
    if (c->h_chain_ovf[2 * slot] || c->h_chain_ovf[2 * slot + 1]) { c->err = "frame-construction capacity overflow in the batch this chain tracked"; return RGBL_E_CAPACITY; }
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
    if (c->chain_pending) { c->err = "a tracking chain is in flight (rgbl_resident_track_end not called)"; return RGBL_E_INVALID; }
    const int rc = rgbl_resident_track_begin(ctx, pose0, fx, fy, cx, cy, bf, th, mono);
    if (rc) return rc;
    return rgbl_resident_track_end(ctx, poses_out, n_matches, n_inliers);
}

}  // extern "C"
