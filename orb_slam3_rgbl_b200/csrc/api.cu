// Context, memory plan and the C ABI entry points of librgbl_b200.so (see include/rgbl_b200.h).
// There is no CPU fallback anywhere in this file: every compute entry point needs the CUDA device
// the context was created on and reports RGBL_E_CUDA otherwise.
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
#include <vector>

#include "rgbl_ctx.h"
#include "rgbl_device.cuh"

namespace rgbl {

static thread_local std::string g_create_error;

// The members of Ctx own every resource of the context; their destructors release them once no stream has work left.
static void release(Ctx* c) {
    if (!c) return;
    cudaSetDevice(c->cfg.device);
    for (cudaStream_t s : {c->st.get(), c->st_aux.get(), c->st_trk.get()}) if (s) cudaStreamSynchronize(s);      // st_trk: a chain may be in flight
    delete c;
}

// a lazily allocated array of at least n elements: allocated by the first call that needs it, reallocated (contents not kept) by a call
// that needs more (the input planes after a larger rgbl_set_input_resize), and retried by the next call if that allocation failed
template <class A>
static bool ensure(A& a, size_t n) { return a.size() >= n || a.alloc(n) == cudaSuccess; }

// the row pitch of an input-size image of ch bytes per pixel (64-byte rows)
static int input_pitch(const Ctx* c, int ch) { return (c->input.w * ch + 63) & ~63; }

// After a change of the camera-input setting: writes its derived values and drops the resident batch, which was loaded for the previous
// setting (stereo_only: the change concerns stereo pairs only, and a batch of another kind is kept)
static void input_changed(Ctx* c, bool stereo_only = false) {
    InputSetting& in = c->input;
    const int W = c->cfg.width, H = c->cfg.height;
    in.pitch = input_pitch(c, in.ch);
    in.depth_pitch = ((size_t)in.w * sizeof(uint16_t) + 63) / 64 * 32;
    in.kx = in.w % W == 0 ? in.w / W : 0; in.ky = in.h % H == 0 ? in.h / H : 0;
    if (!stereo_only || c->resident_kind == InputKind::stereo) c->resident_frames = 0;
}

static int create(const rgbl_config* cfg, Ctx** out) {
    Ctx* c = new Ctx();
    c->cfg = *cfg;
    auto fail = [&](int rc) { g_create_error = c->err; release(c); return rc; };
    if (cfg->width < 1 || cfg->height < 1 || cfg->max_batch < 1 || cfg->max_points < 0) { c->err = "invalid configuration"; return fail(RGBL_E_INVALID); }
    if (cfg->max_points >= (1 << 22) - 1) { c->err = "max_points must be < 4194303"; return fail(RGBL_E_UNSUPPORTED); }
    int rc = compute_orb_tables(cfg->orb, c->tab);
    if (rc) { c->err = "invalid ORB parameters"; return fail(rc); }
    rc = build_geometry(cfg->width, cfg->height, c->tab, c->levels, c->cells, c->coefs, c->frame_bytes, c->err);
    if (rc) return fail(rc);
    c->n_cells = (int)c->cells.size();
    c->input.w = cfg->width; c->input.h = cfg->height; input_changed(c);      // gray images of the context's size
    // DistributeOctTree returns at most max(quota + 2, 4 * nIni) keypoints per level (SURVEY App. C: the very
    // first subdivision pass is unguarded, later ones stop within +3 of the budget).
    c->cap_kp = 0;
    for (const LevelGeom& g : c->levels) {
        const int n_ini = (int)std::round(static_cast<float>(g.max_bx - g.min_bx) / (g.max_by - g.min_by));
        c->cap_kp += std::max(g.quota + 3, 4 * n_ini);
    }
    const int B = cfg->max_batch;
    const int per_frame_cand = cfg->max_candidates > 0 ? cfg->max_candidates : std::max(32768, cfg->width * cfg->height / 8);
    c->dense_cap = per_frame_cand * B;

    cudaError_t e = cudaSetDevice(cfg->device);
    if (e != cudaSuccess) { c->err = std::string("cudaSetDevice: ") + cudaGetErrorString(e) + " (librgbl_b200 has no CPU fallback)"; return fail(RGBL_E_CUDA); }
    const int nl = c->tab.nlevels;
    const size_t WH = (size_t)cfg->width * cfg->height;
#define CUF(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { c->err = std::string(#call) + ": " + cudaGetErrorString(e_); return fail(RGBL_E_CUDA); } } while (0)
    CUF(c->st.create());
    CUF(c->st_aux.create());
    CUF(c->ev_t0.create());
    CUF(c->ev_t1.create());
    CUF(c->ev_pyr.create(cudaEventDisableTiming));
    CUF(c->ev_blur.create(cudaEventDisableTiming));
    for (int i = 0; i < kNumStages; ++i) { CUF(c->ev_b[i].create()); CUF(c->ev_e[i].create()); }
    CUF(c->d_levels.alloc(nl));
    CUF(c->d_cells.alloc(c->cells.size()));
    CUF(c->d_coefs.alloc(std::max<size_t>(c->coefs.size(), 1)));
    CUF(cudaMemcpy(c->d_levels, c->levels.data(), nl * sizeof(LevelGeom), cudaMemcpyHostToDevice));
    CUF(cudaMemcpy(c->d_cells, c->cells.data(), c->cells.size() * sizeof(CellInfo), cudaMemcpyHostToDevice));
    if (!c->coefs.empty()) CUF(cudaMemcpy(c->d_coefs, c->coefs.data(), c->coefs.size() * sizeof(LinCoef), cudaMemcpyHostToDevice));
    CUF(c->d_pyr.alloc(c->frame_bytes * B));
    CUF(c->d_blur.alloc(c->frame_bytes * B));
    CUF(cudaMemset(c->d_pyr, 0, c->frame_bytes * B));
    CUF(cudaMemset(c->d_blur, 0, c->frame_bytes * B));
    CUF(c->d_slots.alloc((size_t)B * c->n_cells * kCellCap));
    CUF(c->d_counts.alloc((size_t)B * c->n_cells));
    CUF(c->d_cell_off.alloc((size_t)B * c->n_cells));
    CUF(c->d_level_cnt.alloc((size_t)B * RGBL_MAX_LEVELS));
    CUF(c->d_frame_total.alloc((size_t)B));
    CUF(c->d_overflow.alloc(4));
    CUF(cudaMemset(c->d_overflow, 0, 4 * sizeof(int)));
    CUF(c->d_dense.alloc((size_t)c->dense_cap));
    {   // device quad-tree: per-level survivor regions + scratch mirroring the dense candidate buffer
        std::vector<int> region(nl + 1, 0);
        bool fits = true;
        for (int l = 0; l < nl; ++l) {
            const LevelGeom& g = c->levels[l];
            const int n_ini = (int)std::round(static_cast<float>(g.max_bx - g.min_bx) / (g.max_by - g.min_by));
            region[l + 1] = region[l] + std::max(g.quota + 3, 4 * n_ini);
            if (g.quota + 3 > 1024 || 4 * n_ini > 1024 || n_ini < 1 || n_ini > 64) fits = false;
            c->qt_max_nodes = std::max(c->qt_max_nodes, std::max(g.quota + 3, 4 * n_ini));
        }
        int dev_smem = 0;
        cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device);
        c->qt_device_ok = fits && dev_smem >= quadtree_smem_bytes();
        c->device_quadtree = c->qt_device_ok;
        CUF(c->d_lvl_region.alloc(nl + 1));
        CUF(cudaMemcpy(c->d_lvl_region, region.data(), (nl + 1) * sizeof(int), cudaMemcpyHostToDevice));
        CUF(c->d_sel_lvl.alloc((size_t)B * c->cap_kp));
        CUF(c->d_n_sel_lvl.alloc((size_t)B * RGBL_MAX_LEVELS));
        CUF(c->qt_perm_a.alloc(c->dense_cap)); CUF(c->qt_perm_b.alloc(c->dense_cap));
        CUF(c->qt_node_a.alloc(c->dense_cap)); CUF(c->qt_node_b.alloc(c->dense_cap));
        CUF(c->qt_scan.alloc((size_t)c->dense_cap + (size_t)B * nl + 8));
        CUF(c->qt_quad.alloc(c->dense_cap));
        c->qt_scr = QtScratchDev{c->qt_perm_a, c->qt_perm_b, c->qt_node_a, c->qt_node_b, c->qt_scan, c->qt_quad};
    }
    {   // fused TMA level kernel unless RGBL_LEVEL_TMA=0 or its tensor maps cannot be made; the cell strips of the FAST kernel
        const char* envt = getenv("RGBL_LEVEL_TMA");
        c->level_tma = !(envt && envt[0] == '0') && make_level_tensor_maps(c->d_pyr, c->frame_bytes, B, c->levels.data(), nl, &c->level_tms) == 0;
        build_fast_strips(c->cells, 8, 264, c->strips, c->strip_rows_cap, c->strip_list_cap);
        CUF(c->d_strips.alloc(c->strips.size()));
        CUF(cudaMemcpy(c->d_strips, c->strips.data(), c->strips.size() * sizeof(StripInfo), cudaMemcpyHostToDevice));
    }
    CUF(c->d_sel.alloc((size_t)B * c->cap_kp));
    CUF(c->d_n_sel.alloc((size_t)B));
    CUF(c->d_kps.alloc((size_t)B * c->cap_kp));
    CUF(c->d_kps_un.alloc((size_t)B * c->cap_kp));      // mvKeysUn of batched frame construction with a distorted camera
    CUF(c->d_kps_in.alloc(2 * (size_t)c->cap_kp));      // the two-call forms' mvKeys | mvKeysUn uploads
    c->cam_bounds[0] = c->frame_bounds[0] = 0.f; c->cam_bounds[1] = c->frame_bounds[1] = (float)cfg->width;
    c->cam_bounds[2] = c->frame_bounds[2] = 0.f; c->cam_bounds[3] = c->frame_bounds[3] = (float)cfg->height;
    CUF(c->d_n_kp_in.alloc(1));
    CUF(c->d_desc.alloc((size_t)B * c->cap_kp * 32));
    CUF(c->d_depth.alloc((size_t)B * c->cap_kp));
    CUF(c->d_uright.alloc((size_t)B * c->cap_kp));
    if (cfg->max_points > 0) {
        CUF(c->d_pts.alloc((size_t)B * 4 * cfg->max_points));
        CUF(c->d_n_pts.alloc((size_t)B));
        CUF(c->d_idx_map.alloc((size_t)B * WH));
        CUF(cudaMemset(c->d_idx_map, 0, (size_t)B * WH * sizeof(uint32_t)));
        CUF(c->d_raw.alloc((size_t)B * WH));
        CUF(c->d_processed.alloc((size_t)B * WH));
        CUF(c->h_n_pts.alloc((size_t)B));
    }
    c->scratch_bytes = (size_t)(cfg->width + 2 * kEdgeThreshold + 64) * (cfg->height + 2 * kEdgeThreshold);
    CUF(c->d_scratch.alloc(c->scratch_bytes));
    CUF(c->h_scalars.alloc(16));
    CUF(c->h_chain_ovf.alloc(4));
    for (int i = 0; i < 4; ++i) c->h_chain_ovf[i] = 0;
    c->chain_timing_on = std::getenv("RGBL_CHAIN_TIMING") != nullptr;
    c->chain_graphs_on = !(std::getenv("RGBL_CHAIN_GRAPH") && std::getenv("RGBL_CHAIN_GRAPH")[0] == '0');
    c->chain_pdl_on = !(std::getenv("RGBL_CHAIN_PDL") && std::getenv("RGBL_CHAIN_PDL")[0] == '0');
    CUF(c->h_level_cnt.alloc((size_t)B * RGBL_MAX_LEVELS));
    CUF(c->h_frame_total.alloc((size_t)B));
    CUF(c->h_overflow.alloc(4));
    CUF(c->h_n_sel.alloc((size_t)B));
    CUF(c->h_dense.alloc((size_t)c->dense_cap));
    CUF(c->h_sel.alloc((size_t)B * c->cap_kp));
#undef CUF
    *out = c;
    return RGBL_OK;
}

// ---- profiling helpers -----------------------------------------------------------------------------
void stage_begin(Ctx* c, int stage, cudaStream_t st) {
    if (c->prof_on) { cudaEventRecord(c->ev_b[stage], st); c->st_used[stage] = true; }
}
void stage_end(Ctx* c, int stage, cudaStream_t st, int launches) {
    c->total_launches += launches;
    c->st_pending_launches[stage] += launches;
    if (c->prof_on) cudaEventRecord(c->ev_e[stage], st);
}
// call after both streams are idle
void prof_collect(Ctx* c) {
    for (int i = 0; i < kNumStages; ++i) {
        if (c->prof_on && c->st_used[i]) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, c->ev_b[i], c->ev_e[i]) == cudaSuccess) { c->st_ms[i] += ms; c->st_calls[i] += 1; c->st_launches[i] += c->st_pending_launches[i]; }
        }
        c->st_used[i] = false;
        c->st_pending_launches[i] = 0;
    }
    float ms = 0.f;
    if (c->prof_on && c->rsd_used && cudaEventElapsedTime(&ms, c->ev_rsd_b, c->ev_rsd_e) == cudaSuccess) c->st_ms[ST_DEPTH_GATHER] += ms;
    c->rsd_used = false;
}

// ---- extraction pipeline -----------------------------------------------------------------------
// Stage 0 (copy):   images -> level 0 of each frame slot (upload_planes).
// Stage 1 (device): pyramid, FAST + compaction on the main stream; blur on the aux stream.
// Stage 2 (host):   quad-tree per (frame, level) on worker threads -> SelKp lists.
// Stage 3 (device): describe.  Results stay in d_kps / d_desc (copied out by the callers).

// The image planes of a batch: plane f at base + f * stride + off, rows pitch bytes apart, w x h pixels of ch bytes
struct Planes {
    uint8_t* base; size_t stride, off; int pitch; int w, h; int ch = 1;
    uint8_t* at(int f) const { return base + (size_t)f * stride + off; }
};

static Planes level0_planes(const Ctx* c) {
    return {c->d_pyr, c->frame_bytes, (size_t)c->levels[0].off, c->levels[0].pitch, c->cfg.width, c->cfg.height};
}

// H2D of n host images into planes [first, first + n) of dst, on stream st
static int upload_planes(Ctx* c, const Planes& dst, int first, int n, const uint8_t* const* img, int stride, cudaStream_t st) {
    for (int f = 0; f < n; ++f)
        CU(cudaMemcpy2DAsync(dst.at(first + f), dst.pitch, img[f], stride, (size_t)dst.w * dst.ch, dst.h, cudaMemcpyHostToDevice, st));
    return RGBL_OK;
}

// level0: if set, enqueues the kernels that write level 0 on the main stream (rectification of stereo pairs, the input resize) and returns
// their count; billed to the pyramid stage.
static int run_extract(Ctx* c, int n_frames, const std::function<void()>& aux_work = nullptr, const std::function<int()>& level0 = nullptr) {
    const int nl = c->tab.nlevels;
    // new frames: mvKeysUn == mvKeys and image bounds until undistort_keypoints says otherwise
    c->frames_undistorted = false;
    c->frame_bounds[0] = 0.f; c->frame_bounds[1] = (float)c->cfg.width; c->frame_bounds[2] = 0.f; c->frame_bounds[3] = (float)c->cfg.height;
    stage_begin(c, ST_PYRAMID, c->st);
    const int level0_launches = level0 ? level0() : 0;
    // fused TMA tile kernel: level l's launch writes blur(l) and level l+1 (the separate blur stage below is then empty)
    const bool fused_levels = c->level_tma && launch_level_tiles(c->st, c->level_tms, c->d_pyr, c->d_blur, c->frame_bytes, c->levels.data(), nl, c->d_coefs, n_frames) == 0;
    if (!fused_levels) launch_pyramid(c->st, c->d_pyr, c->frame_bytes, c->levels.data(), nl, c->d_coefs, n_frames);
    stage_end(c, ST_PYRAMID, c->st, level0_launches + (fused_levels ? nl : nl - 1));
    stage_begin(c, ST_FAST, c->st);
    if (launch_fast_strips(c->st, c->d_pyr, c->frame_bytes, c->d_levels, c->d_cells, c->n_cells, c->d_strips, (int)c->strips.size(),
                           c->strip_rows_cap, c->strip_list_cap, c->cfg.orb.ini_th_fast, c->cfg.orb.min_th_fast, c->d_slots,
                           c->d_counts, c->d_overflow, n_frames) != 0) {
        c->err = "strip FAST kernel needs more shared memory than this device allows"; return RGBL_E_CUDA;
    }
    stage_end(c, ST_FAST, c->st, 1);
    stage_begin(c, ST_COMPACT, c->st);
    launch_compact(c->st, c->d_levels, nl, c->n_cells, c->d_slots, c->d_counts, c->d_cell_off, c->d_level_cnt,
                   c->d_frame_total, c->d_dense, c->dense_cap, c->d_overflow, n_frames);
    stage_end(c, ST_COMPACT, c->st, 2);
    // The aux stream starts once FAST + compaction are done, i.e. it runs the blur (and, for RGB-L frames, the
    // depth maps queued by the caller via `aux_work`) while the host is busy with the quad-tree.
    CU(cudaEventRecord(c->ev_pyr, c->st));
    CU(cudaStreamWaitEvent(c->st_aux, c->ev_pyr, 0));
    stage_begin(c, ST_BLUR, c->st_aux);
    if (!fused_levels) launch_blur(c->st_aux, c->d_pyr, c->d_blur, c->frame_bytes, c->levels.data(), nl, n_frames);
    stage_end(c, ST_BLUR, c->st_aux, fused_levels ? 0 : nl);
    if (aux_work) aux_work();
    CU(cudaEventRecord(c->ev_blur, c->st_aux));
    if (c->prof_serial) CU(cudaStreamWaitEvent(c->st, c->ev_blur, 0));      // rgbl_profile_enable(ctx, 2): no kernel of this context overlaps another
    if (c->device_quadtree) {
        // Fully on-device keypoint distribution: no host round trip between FAST and describe.
        stage_begin(c, ST_QUADTREE, c->st);
        if (launch_quadtree(c->st, c->d_dense, c->d_level_cnt, c->d_frame_total, c->d_levels, nl, c->qt_scr, c->d_sel_lvl, c->d_n_sel_lvl,
                            c->d_lvl_region, c->cap_kp, c->d_overflow + 1, c->d_sel, c->d_n_sel, n_frames, c->qt_max_nodes, c->dense_cap) != 0) {
            c->err = "quad-tree kernel needs more shared memory than this device allows"; return RGBL_E_CUDA;
        }
        stage_end(c, ST_QUADTREE, c->st, 2);
        CU(cudaStreamWaitEvent(c->st, c->ev_blur, 0));
        stage_begin(c, ST_DESCRIBE, c->st);
        launch_describe_staged(c->st, c->d_pyr, c->d_blur, c->frame_bytes, c->d_levels, c->d_sel, c->d_n_sel, c->cap_kp, c->cap_kp, c->tab.umax,
                               c->d_kps, c->d_desc, n_frames);
        stage_end(c, ST_DESCRIBE, c->st, 1);
        CU(cudaGetLastError());
        c->last_frames = n_frames;
        c->blur_valid = true;
        c->host_counts_valid = false;
        return c->cap_kp;        // upper bound of keypoints per frame (exact counts are in d_n_sel)
    }
    CU(cudaMemcpyAsync(c->h_level_cnt, c->d_level_cnt, (size_t)n_frames * RGBL_MAX_LEVELS * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_frame_total, c->d_frame_total, (size_t)n_frames * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_overflow, c->d_overflow, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    if (*c->h_overflow) {
        cudaMemsetAsync(c->d_overflow, 0, sizeof(int), c->st);
        c->err = (*c->h_overflow == 1) ? "FAST cell slot overflow (>256 survivors in one cell)" : "candidate buffer overflow: raise max_candidates";
        return RGBL_E_CAPACITY;
    }
    size_t total = 0;
    std::vector<size_t> fbase(n_frames + 1, 0);
    for (int f = 0; f < n_frames; ++f) { total += c->h_frame_total[f]; fbase[f + 1] = total; }
    if (total > (size_t)c->dense_cap) { c->err = "candidate buffer overflow: raise max_candidates"; return RGBL_E_CAPACITY; }
    if (total) CU(cudaMemcpyAsync(c->h_dense, c->d_dense, total * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));

    // host quad-tree: tasks = (frame, level)
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::vector<SelKp>> sel_lists((size_t)n_frames * nl);
    std::atomic<int> next{0};
    std::atomic<int> status{0};
    const int n_tasks = n_frames * nl;
    auto worker = [&]() {
        std::vector<int32_t> xys, idx;
        for (;;) {
            const int t = next.fetch_add(1);
            if (t >= n_tasks) break;
            const int f = t / nl, l = t % nl;
            size_t off = fbase[f];
            for (int k = 0; k < l; ++k) off += c->h_level_cnt[f * RGBL_MAX_LEVELS + k];
            const int n = c->h_level_cnt[f * RGBL_MAX_LEVELS + l];
            const LevelGeom& lg = c->levels[l];
            xys.resize((size_t)n * 3);
            for (int k = 0; k < n; ++k) {
                const uint32_t p = c->h_dense[off + k];
                xys[3 * k] = (int)(p & 0xfff); xys[3 * k + 1] = (int)((p >> 12) & 0xfff); xys[3 * k + 2] = (int)(p >> 24);
            }
            idx.resize((size_t)c->cap_kp);
            int m = quadtree_select(xys.data(), n, lg.min_bx, lg.max_bx, lg.min_by, lg.max_by, lg.quota, idx.data(), (int)idx.size());
            if (m < 0) { status.store(m); continue; }
            std::vector<SelKp>& out = sel_lists[t];
            out.resize(m);
            for (int k = 0; k < m; ++k) {
                const int q = idx[k];
                out[k].x = (uint16_t)(xys[3 * q] + lg.min_bx);
                out[k].y = (uint16_t)(xys[3 * q + 1] + lg.min_by);
                out[k].level = (uint8_t)l; out[k].score = (uint8_t)xys[3 * q + 2]; out[k].pad = 0;
            }
        }
    };
    int n_threads = (int)std::thread::hardware_concurrency();
    n_threads = std::max(1, std::min(std::min(n_threads, 32), n_tasks));
    if (n_threads == 1) worker();
    else {
        std::vector<std::thread> pool;
        for (int i = 0; i < n_threads; ++i) pool.emplace_back(worker);
        for (auto& th : pool) th.join();
    }
    if (status.load()) { c->err = "quad-tree selection failed"; return status.load(); }
    int max_n = 0;
    for (int f = 0; f < n_frames; ++f) {
        int n = 0;
        for (int l = 0; l < nl; ++l) {
            const std::vector<SelKp>& sl = sel_lists[(size_t)f * nl + l];
            if (n + (int)sl.size() > c->cap_kp) { c->err = "keypoint capacity exceeded"; return RGBL_E_CAPACITY; }
            if (!sl.empty()) std::memcpy(c->h_sel + (size_t)f * c->cap_kp + n, sl.data(), sl.size() * sizeof(SelKp));
            n += (int)sl.size();
        }
        c->h_n_sel[f] = n;
        max_n = std::max(max_n, n);
    }
    c->host_quadtree_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    CU(cudaMemcpyAsync(c->d_sel, c->h_sel, (size_t)n_frames * c->cap_kp * sizeof(SelKp), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_n_sel, c->h_n_sel, (size_t)n_frames * sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaStreamWaitEvent(c->st, c->ev_blur, 0));
    stage_begin(c, ST_DESCRIBE, c->st);
    launch_describe_staged(c->st, c->d_pyr, c->d_blur, c->frame_bytes, c->d_levels, c->d_sel, c->d_n_sel, c->cap_kp, max_n, c->tab.umax,
                           c->d_kps, c->d_desc, n_frames);
    stage_end(c, ST_DESCRIBE, c->st, max_n > 0 ? 1 : 0);
    CU(cudaGetLastError());
    c->last_frames = n_frames;
    c->blur_valid = true;
    c->host_counts_valid = true;
    return max_n;
}

// Device-quad-tree mode: bring the per-frame keypoint counts and the status flags to the host (one small sync).
static int fetch_counts(Ctx* c, int n_frames) {
    if (c->host_counts_valid) return RGBL_OK;
    CU(cudaMemcpyAsync(c->h_n_sel, c->d_n_sel, (size_t)n_frames * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(c->h_overflow, c->d_overflow, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    if (c->h_overflow[0] || c->h_overflow[1]) {
        const int a = c->h_overflow[0], b = c->h_overflow[1];
        cudaMemsetAsync(c->d_overflow, 0, 2 * sizeof(int), c->st);
        c->err = b ? "device quad-tree capacity exceeded (select the host quad-tree: rgbl_set_host_quadtree)" : (a == 1 ? "FAST cell slot overflow (>256 survivors in one cell)" : "candidate buffer overflow: raise max_candidates");
        return RGBL_E_CAPACITY;
    }
    return RGBL_OK;
}

// Depth maps for n_frames resident point clouds (d_pts / d_n_pts) on stream st.
static void run_depth_maps(Ctx* c, const DepthDev& dd, int n_frames, int max_pts, float* raw, cudaStream_t st) {
    const int W = c->cfg.width, H = c->cfg.height;
    stage_begin(c, ST_DEPTH_PROJECT, st);
    launch_depth_project(st, c->d_pts, 4 * c->cfg.max_points, c->d_n_pts, max_pts, dd, W, H, c->d_idx_map, c->stamp, n_frames);
    stage_end(c, ST_DEPTH_PROJECT, st, max_pts > 0 ? 1 : 0);
    stage_begin(c, ST_DEPTH_DILATE, st);
    const bool need_raw = dd.method == RGBL_DEPTH_AVERAGE_FILTERING || dd.method == RGBL_DEPTH_NEAREST_NEIGHBOR_PIXEL;
    float* raw_out = need_raw ? c->d_raw : raw;
    launch_depth_resolve_dilate_v2(st, c->d_pts, 4 * c->cfg.max_points, c->d_n_pts, dd, W, H, c->d_idx_map, c->stamp, raw_out, c->d_processed,
                                   n_frames);
    int launches = 1;
    if (dd.method == RGBL_DEPTH_AVERAGE_FILTERING) { launch_depth_average_filter(st, c->d_raw, W, H, dd.avg_kernel, c->d_processed, n_frames); ++launches; }
    stage_end(c, ST_DEPTH_DILATE, st, launches);
}

// Frame::UndistortKeyPoints (src/Frame.cc:837-869) of the batch just extracted, between describe (the last writer of d_kps) and the depth
// association, on stream st; the caller bills it to its depth-gather stage.  k1 == 0 (the default): the reference's early return
// mvKeysUn = mvKeys, nothing is launched.  -> mvKeysUn; *launches counts the kernel.
static const rgbl_keypoint* undistort_keypoints(Ctx* c, int max_n, int n_frames, cudaStream_t st, int* launches) {
    if (!c->undistort) return c->d_kps;
    launch_undistort_keypoints(st, c->cam_un, c->d_kps, c->d_n_sel, c->cap_kp, max_n, c->d_kps_un, n_frames);
    if (max_n > 0) ++*launches;
    c->frames_undistorted = true;
    std::memcpy(c->frame_bounds, c->cam_bounds, sizeof(c->frame_bounds));
    return c->d_kps_un;
}

// GetFeatureDepthFromDepthMap / the per-keypoint part of Upsample_NearestNeighbor_Pixel.  undistort: batched frame construction, kps_un
// is computed from kps first (undistort_keypoints).
static void run_depth_keypoints(Ctx* c, const DepthDev& dd, const rgbl_keypoint* kps, const rgbl_keypoint* kps_un, const int* n_kp, int max_n,
                                int n_frames, cudaStream_t st, bool undistort = false) {
    const int W = c->cfg.width, H = c->cfg.height;
    int launches = max_n > 0 ? 1 : 0;
    stage_begin(c, ST_DEPTH_GATHER, st);
    if (undistort) kps_un = undistort_keypoints(c, max_n, n_frames, st, &launches);
    if (dd.method == RGBL_DEPTH_NEAREST_NEIGHBOR_PIXEL)
        launch_depth_nn_pixel(st, c->d_raw, W, H, kps, kps_un, n_kp, c->cap_kp, max_n, dd.bf, dd.nn_radius, c->d_depth, c->d_uright, n_frames);
    else
        launch_depth_gather(st, c->d_processed, W, H, kps, kps_un, n_kp, c->cap_kp, max_n, dd.method == RGBL_DEPTH_NONE ? -1.f : dd.bf,
                            c->d_depth, c->d_uright, n_frames);
    stage_end(c, ST_DEPTH_GATHER, st, launches);
}

static int setup_depth(Ctx* c, const float P[12], const rgbl_depth_params* prm, DepthDev& dd) {
    if (!c->d_pts) { c->err = "context was created with max_points == 0"; return RGBL_E_INVALID; }
    std::memcpy(dd.P, P, sizeof(float) * 12);
    dd.min_dist = prm->min_dist; dd.max_dist = prm->max_dist; dd.bf = prm->bf;
    dd.inv_scale_m = prm->max_dist * prm->inv_dilation_scale;
    dd.method = prm->method; dd.avg_kernel = prm->avg_kernel; dd.nn_radius = prm->nn_search_radius;
    switch (prm->method) {
        case RGBL_DEPTH_INVERSE_DILATION:
            if (prm->ku < 1 || prm->kv < 1 || prm->ku > 9 || prm->kv > 9) { c->err = "structuring element must be 1..9"; return RGBL_E_INVALID; }
            dd.ku = prm->ku; dd.kv = prm->kv;
            std::memcpy(dd.mask, prm->mask, 81);
            break;
        case RGBL_DEPTH_AVERAGE_FILTERING:
            if (prm->avg_kernel < 1 || prm->avg_kernel > 9) { c->err = "AverageFiltering kernel size must be 1..9"; return RGBL_E_INVALID; }
            dd.ku = dd.kv = 1; std::memset(dd.mask, 0, 81); dd.mask[0] = 1;          // resolve only: Raw is the filter input
            break;
        case RGBL_DEPTH_NEAREST_NEIGHBOR_PIXEL:
            if (!(prm->nn_search_radius >= 1.f) || prm->nn_search_radius > 30.f) { c->err = "NearestNeighborPixel search distance must be 1..30"; return RGBL_E_INVALID; }
            dd.ku = dd.kv = 1; std::memset(dd.mask, 0, 81); dd.mask[0] = 1;
            break;
        case RGBL_DEPTH_NONE:
            dd.ku = dd.kv = 1; std::memset(dd.mask, 0, 81); dd.mask[0] = 1;
            break;
        default:
            c->err = "LiDAR.Method not implemented (IPBasic has no definition in the reference either, src/DepthModule.cc:62-77)";
            return RGBL_E_UNSUPPORTED;
    }
    if (++c->stamp >= 1023u) {
        // stamp wrap: clear the index map once every 1022 calls (both streams idle first)
        cudaStreamSynchronize(c->st); cudaStreamSynchronize(c->st_aux);
        if (cudaMemset(c->d_idx_map, 0, (size_t)c->cfg.max_batch * c->cfg.width * c->cfg.height * sizeof(uint32_t)) != cudaSuccess) {
            c->err = "cudaMemset(idx_map) failed"; return RGBL_E_CUDA;
        }
        c->stamp = 1;
    }
    return RGBL_OK;
}

int stereo_matches(Ctx* c, int l0, int r0, int n_pairs, float mb, float mbf) {
    if (c->cap_kp > 65535) { c->err = "more than 65535 keypoints per frame"; return RGBL_E_UNSUPPORTED; }      // the match key holds 16 index bits
    const int H = c->cfg.height;
    const size_t pairs = (size_t)std::max(1, c->cfg.max_batch / 2);
    c->stereo_idx_cap = stereo_row_index_cap(c->cap_kp, c->tab.scale, c->tab.nlevels, H);
    if (!ensure(c->d_stereo_row_start, pairs * (H + 1)) || !ensure(c->d_stereo_row_idx, pairs * c->stereo_idx_cap) || !ensure(c->d_stereo_sad, pairs * c->cap_kp)) {
        c->err = "device allocation failed (stereo row index)"; return RGBL_E_CUDA;
    }
    StereoBatchDev s{};
    s.pyr = c->d_pyr; s.frame_stride = c->frame_bytes; s.levels = c->d_levels;
    s.kps = c->d_kps; s.desc = c->d_desc; s.n_sel = c->d_n_sel; s.cap = c->cap_kp;
    s.l0 = l0; s.r0 = r0; s.n_rows = H;
    for (int l = 0; l < c->tab.nlevels; ++l) { s.scale[l] = c->tab.scale[l]; s.inv_scale[l] = c->tab.inv_scale[l]; }
    s.mb = mb; s.mbf = mbf;
    s.depth = c->d_depth; s.uright = c->d_uright;
    s.row_start = c->d_stereo_row_start; s.row_idx = c->d_stereo_row_idx; s.idx_cap = c->stereo_idx_cap; s.sad = c->d_stereo_sad;
    stage_begin(c, ST_MATCH, c->st);
    launch_stereo_matches(c->st, s, n_pairs);
    stage_end(c, ST_MATCH, c->st, 5);
    CU(cudaGetLastError());
    return RGBL_OK;
}

}  // namespace rgbl

using namespace rgbl;

extern "C" {

int rgbl_create(const rgbl_config* cfg, rgbl_ctx** out) {
    if (!cfg || !out) return RGBL_E_INVALID;
    *out = nullptr;
    Ctx* c = nullptr;
    int rc = create(cfg, &c);
    if (rc) return rc;
    *out = reinterpret_cast<rgbl_ctx*>(c);
    return RGBL_OK;
}

void rgbl_destroy(rgbl_ctx* ctx) { release(reinterpret_cast<Ctx*>(ctx)); }

int rgbl_keypoint_capacity(const rgbl_ctx* ctx) { return ctx ? reinterpret_cast<const Ctx*>(ctx)->cap_kp : RGBL_E_INVALID; }

const char* rgbl_last_error(const rgbl_ctx* ctx) {
    if (!ctx) return g_create_error.c_str();
    return reinterpret_cast<const Ctx*>(ctx)->err.c_str();
}

int rgbl_orb_extract_batch(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                           int lap0, int lap1, rgbl_keypoint* kps, uint8_t* desc, int cap, int* n_out, int* mono_index) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || n_frames < 1 || !kps || !desc || !n_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (width <= 0 || height <= 0) { c->err = "empty image"; return RGBL_E_EMPTY; }
    for (int f = 0; f < n_frames; ++f) if (!gray[f]) { c->err = "empty image"; return RGBL_E_EMPTY; }
    if (width != c->cfg.width || height != c->cfg.height || stride < width) { c->err = "image size does not match the context"; return RGBL_E_INVALID; }
    if (n_frames > c->cfg.max_batch) { c->err = "n_frames exceeds max_batch"; return RGBL_E_CAPACITY; }
    CU(cudaSetDevice(c->cfg.device));
    int rc = upload_planes(c, level0_planes(c), 0, n_frames, gray, stride, c->st);
    if (rc) return rc;
    rc = run_extract(c, n_frames);
    if (rc < 0) return rc;
    rc = fetch_counts(c, n_frames); if (rc) return rc;
    for (int f = 0; f < n_frames; ++f) {
        const int n = c->h_n_sel[f];
        n_out[f] = n;
        if (n > cap) { c->err = "output capacity too small"; return RGBL_E_CAPACITY; }
        if (n) {
            CU(cudaMemcpyAsync(kps + (size_t)f * cap, c->d_kps + (size_t)f * c->cap_kp, (size_t)n * sizeof(rgbl_keypoint), cudaMemcpyDeviceToHost, c->st));
            CU(cudaMemcpyAsync(desc + (size_t)f * cap * 32, c->d_desc + (size_t)f * c->cap_kp * 32, (size_t)n * 32, cudaMemcpyDeviceToHost, c->st));
        }
    }
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    prof_collect(c);
    // vLappingArea placement (src/ORBextractor.cc:1153-1162): lapping keypoints fill the back.
    for (int f = 0; f < n_frames; ++f) {
        const int n = n_out[f];
        int mono = n;
        if (!(lap0 == 0 && lap1 == 0)) {
            rgbl_keypoint* k = kps + (size_t)f * cap;
            uint8_t* d = desc + (size_t)f * cap * 32;
            std::vector<rgbl_keypoint> k2(n);
            std::vector<uint8_t> d2((size_t)n * 32);
            int mi = 0, si = n - 1;
            for (int i = 0; i < n; ++i) {
                const bool lapping = k[i].x >= (float)lap0 && k[i].x <= (float)lap1;
                const int slot = lapping ? si-- : mi++;
                k2[slot] = k[i];
                std::memcpy(&d2[(size_t)slot * 32], d + (size_t)i * 32, 32);
            }
            std::memcpy(k, k2.data(), (size_t)n * sizeof(rgbl_keypoint));
            std::memcpy(d, d2.data(), (size_t)n * 32);
            mono = mi;
        }
        if (mono_index) mono_index[f] = mono;
    }
    return RGBL_OK;
}

int rgbl_orb_extract(rgbl_ctx* ctx, const uint8_t* gray, int width, int height, int stride, int lap0, int lap1,
                     rgbl_keypoint* kps, uint8_t* desc, int cap, int* n_out, int* mono_index) {
    const uint8_t* g[1] = {gray};
    return rgbl_orb_extract_batch(ctx, 1, g, width, height, stride, lap0, lap1, kps, desc, cap, n_out, mono_index);
}

static int check_frame_level(Ctx* c, int frame, int level) {
    if (frame < 0 || frame >= c->last_frames || level < 0 || level >= c->tab.nlevels) { c->err = "frame/level out of range (no extraction yet?)"; return RGBL_E_INVALID; }
    return RGBL_OK;
}

int rgbl_orb_get_pyramid(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride, int* w_out, int* h_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !dst) return RGBL_E_INVALID;
    int rc = check_frame_level(c, frame, level); if (rc) return rc;
    const LevelGeom& lg = c->levels[level];
    const int W = lg.w + 2 * kEdgeThreshold, H = lg.h + 2 * kEdgeThreshold;
    if (dst_stride < W) { c->err = "dst_stride too small"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    const int pitch = (W + 63) & ~63;
    launch_padded_level(c->st, c->d_pyr, c->frame_bytes, frame, lg, c->d_scratch, pitch);
    CU(cudaMemcpy2DAsync(dst, dst_stride, c->d_scratch, pitch, W, H, cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    if (w_out) *w_out = lg.w;
    if (h_out) *h_out = lg.h;
    return RGBL_OK;
}

static int get_plane(Ctx* c, const uint8_t* base, int frame, int level, uint8_t* dst, int dst_stride, int* w_out, int* h_out) {
    int rc = check_frame_level(c, frame, level); if (rc) return rc;
    const LevelGeom& lg = c->levels[level];
    if (dst_stride < lg.w) { c->err = "dst_stride too small"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    CU(cudaMemcpy2DAsync(dst, dst_stride, base + (size_t)frame * c->frame_bytes + lg.off, lg.pitch, lg.w, lg.h, cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    if (w_out) *w_out = lg.w;
    if (h_out) *h_out = lg.h;
    return RGBL_OK;
}

int rgbl_orb_get_level(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride, int* w_out, int* h_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !dst) return RGBL_E_INVALID;
    return get_plane(c, c->d_pyr, frame, level, dst, dst_stride, w_out, h_out);
}

int rgbl_orb_get_blurred_level(rgbl_ctx* ctx, int frame, int level, uint8_t* dst, int dst_stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !dst) return RGBL_E_INVALID;
    if (!c->blur_valid) { c->err = "no extraction yet"; return RGBL_E_INVALID; }
    CU(cudaStreamSynchronize(c->st_aux));
    return get_plane(c, c->d_blur, frame, level, dst, dst_stride, nullptr, nullptr);
}

int rgbl_orb_get_candidates(rgbl_ctx* ctx, int frame, int level, int32_t* xys, int cap, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !xys || !n_out) return RGBL_E_INVALID;
    int rc = check_frame_level(c, frame, level); if (rc) return rc;
    if (!c->host_counts_valid) {
        CU(cudaSetDevice(c->cfg.device));
        CU(cudaMemcpyAsync(c->h_level_cnt, c->d_level_cnt, (size_t)c->last_frames * RGBL_MAX_LEVELS * sizeof(int), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(c->h_frame_total, c->d_frame_total, (size_t)c->last_frames * sizeof(int), cudaMemcpyDeviceToHost, c->st));
        CU(cudaStreamSynchronize(c->st));
        size_t tot = 0;
        for (int f = 0; f < c->last_frames; ++f) tot += c->h_frame_total[f];
        if (tot > (size_t)c->dense_cap) { c->err = "candidate buffer overflow"; return RGBL_E_CAPACITY; }
        if (tot) CU(cudaMemcpyAsync(c->h_dense, c->d_dense, tot * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->st));
        CU(cudaStreamSynchronize(c->st));
    }
    size_t off = 0;
    for (int f = 0; f < frame; ++f) off += c->h_frame_total[f];
    for (int l = 0; l < level; ++l) off += c->h_level_cnt[frame * RGBL_MAX_LEVELS + l];
    const int n = c->h_level_cnt[frame * RGBL_MAX_LEVELS + level];
    *n_out = n;
    if (n > cap) { c->err = "capacity too small"; return RGBL_E_CAPACITY; }
    for (int k = 0; k < n; ++k) {
        const uint32_t p = c->h_dense[off + k];
        xys[3 * k] = (int)(p & 0xfff); xys[3 * k + 1] = (int)((p >> 12) & 0xfff); xys[3 * k + 2] = (int)(p >> 24);
    }
    return RGBL_OK;
}

int rgbl_depth_from_pcd(rgbl_ctx* ctx, const float* pts4xn, int n_pts, const float P[12], int width, int height,
                        const rgbl_depth_params* prm, const rgbl_keypoint* kps, const rgbl_keypoint* kps_un, int n_kp,
                        float* depth, float* uright, float* raw_map, float* processed_map) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!pts4xn || !P || !prm || n_pts < 0 || n_kp < 0 || (n_kp > 0 && (!kps || !kps_un || !depth || !uright))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (width != c->cfg.width || height != c->cfg.height) { c->err = "image size does not match the context"; return RGBL_E_INVALID; }
    if (n_pts > c->cfg.max_points) { c->err = "n_pts exceeds max_points"; return RGBL_E_CAPACITY; }
    if (n_kp > c->cap_kp) { c->err = "n_kp exceeds keypoint capacity"; return RGBL_E_CAPACITY; }
    CU(cudaSetDevice(c->cfg.device));
    DepthDev dd;
    int rc = setup_depth(c, P, prm, dd); if (rc) return rc;
    const size_t WH = (size_t)width * height;
    c->h_n_pts[0] = n_pts;
    int* h_nkp = c->h_overflow;          // 1-int pinned scratch (overflow flag is re-read on every extract)
    *h_nkp = n_kp;
    if (n_pts) CU(cudaMemcpyAsync(c->d_pts, pts4xn, (size_t)4 * n_pts * sizeof(float), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_n_pts, c->h_n_pts, sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_n_kp_in, h_nkp, sizeof(int), cudaMemcpyHostToDevice, c->st));
    if (n_kp) {
        CU(cudaMemcpyAsync(c->d_kps_in, kps, (size_t)n_kp * sizeof(rgbl_keypoint), cudaMemcpyHostToDevice, c->st));
        CU(cudaMemcpyAsync(c->d_kps_in + c->cap_kp, kps_un, (size_t)n_kp * sizeof(rgbl_keypoint), cudaMemcpyHostToDevice, c->st));
    }
    run_depth_maps(c, dd, 1, n_pts, c->d_raw, c->st);
    run_depth_keypoints(c, dd, c->d_kps_in, c->d_kps_in + c->cap_kp, c->d_n_kp_in, n_kp, 1, c->st);
    CU(cudaGetLastError());
    if (n_kp) {
        CU(cudaMemcpyAsync(depth, c->d_depth, (size_t)n_kp * sizeof(float), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(uright, c->d_uright, (size_t)n_kp * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    }
    if (raw_map) CU(cudaMemcpyAsync(raw_map, c->d_raw, WH * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    if (processed_map) CU(cudaMemcpyAsync(processed_map, c->d_processed, WH * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

/* Frame::ComputeStereoFromRGBD (src/Frame.cc:1074-1095), the depth association of System::TrackRGBD: d = imDepth(kp.y, kp.x) at the
 * DISTORTED keypoint (C-style truncation of the float coordinates), mvDepth = d and mvuRight = kpUn.x - mbf / d where d > 0, else -1.
 * The gather runs on the device: the depth image (H x W float32, already scaled by DepthMapFactor, src/Tracking.cc:1538-1539) is uploaded
 * into the context's processed-depth plane and read by the same kernel that serves DepthModule::GetFeatureDepthFromDepthMap.        */
int rgbl_depth_from_map(rgbl_ctx* ctx, const float* depth_map, int width, int height, int stride_floats, float bf, const rgbl_keypoint* kps,
                        const rgbl_keypoint* kps_un, int n_kp, float* depth, float* uright) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!depth_map || n_kp < 0 || (n_kp > 0 && (!kps || !kps_un || !depth || !uright))) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (width != c->cfg.width || height != c->cfg.height || stride_floats < width) { c->err = "image size does not match the context"; return RGBL_E_INVALID; }
    if (!c->d_processed) { c->err = "context was created with max_points == 0 (no depth planes)"; return RGBL_E_INVALID; }
    if (n_kp > c->cap_kp) { c->err = "n_kp exceeds keypoint capacity"; return RGBL_E_CAPACITY; }
    if (n_kp == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    int* h_nkp = c->h_overflow;
    *h_nkp = n_kp;
    CU(cudaMemcpy2DAsync(c->d_processed, (size_t)width * sizeof(float), depth_map, (size_t)stride_floats * sizeof(float), (size_t)width * sizeof(float), height,
                         cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_n_kp_in, h_nkp, sizeof(int), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_kps_in, kps, (size_t)n_kp * sizeof(rgbl_keypoint), cudaMemcpyHostToDevice, c->st));
    CU(cudaMemcpyAsync(c->d_kps_in + c->cap_kp, kps_un, (size_t)n_kp * sizeof(rgbl_keypoint), cudaMemcpyHostToDevice, c->st));
    stage_begin(c, ST_DEPTH_GATHER, c->st);
    launch_depth_gather(c->st, c->d_processed, width, height, c->d_kps_in, c->d_kps_in + c->cap_kp, c->d_n_kp_in, c->cap_kp, n_kp, bf, c->d_depth, c->d_uright, 1);
    stage_end(c, ST_DEPTH_GATHER, c->st, 1);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(depth, c->d_depth, (size_t)n_kp * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaMemcpyAsync(uright, c->d_uright, (size_t)n_kp * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    prof_collect(c);
    return RGBL_OK;
}

// n_frames images (or pairs) in one batch
static int check_batch(Ctx* c, int n_frames) {
    if (n_frames < 1) { c->err = "n_frames < 1"; return RGBL_E_INVALID; }
    if (n_frames > c->cfg.max_batch) { c->err = "n_frames exceeds max_batch"; return RGBL_E_CAPACITY; }
    return RGBL_OK;
}

// A batch of n_frames images of width x height pixels, rows stride bytes apart, that an entry point takes as `images` has them: camera
// input (c->input), or gray images of the context's size (gray_images)
static int check_images(Ctx* c, const InputSetting& images, int n_frames, int width, int height, int stride) {
    if (width <= 0 || height <= 0) { c->err = "empty image"; return RGBL_E_EMPTY; }
    if (images.ch > 1 && stride < width * images.ch) { c->err = "stride < width * channels (rgbl_set_input_channels)"; return RGBL_E_INVALID; }
    if (width != images.w || height != images.h || stride < width) {
        c->err = images.resize ? "image size does not match the input size (rgbl_set_input_resize)" : "image size does not match the context"; return RGBL_E_INVALID;
    }
    return check_batch(c, n_frames);
}
static InputSetting gray_images(const Ctx* c) { return InputSetting{c->cfg.width, c->cfg.height}; }

// what each input kind is called, and the process call and sequence runner that take it (indexed by InputKind)
struct KindNames { const char* what; const char* process; const char* runner; };
static const KindNames kKindNames[] = {
    {"RGB-L frames", "rgbl_resident_process", "rgbl_track_sequence"},
    {"RGB-D frames", "rgbl_resident_process_rgbd", "rgbl_track_sequence_rgbd"},
    {"stereo pairs", "rgbl_resident_process_stereo", "rgbl_track_sequence_stereo"},
};
static const KindNames& kind_names(InputKind k) { return kKindNames[(int)k]; }

// the working buffers hold n frames of `kind` (stereo: n pairs in slots [0, 2n)), whose largest cloud has max_pts points
static void set_resident(Ctx* c, InputKind kind, int n, int max_pts) {
    c->resident_frames = n; c->resident_max_pts = max_pts; c->resident_kind = kind;
}

// one batch of host inputs of one kind: n frames (RGB-L, RGB-D) or n pairs (stereo, the right images in `right`).  RGB-L clouds:
// layout 0 planar 4 x N rows (x, y, z, 1) as LoadPointcloudBinaryMat builds them; layout 1 the raw KITTI .bin records (x, y, z,
// reflectance) x N, de-interleaved on the device (the 4th row becomes 1, Examples/RGB-L/rgbl_kitti.cc:168-177).  gray == nullptr: the
// images are already on the device (PNG decode).  ch: bytes per pixel of the images (camera(): the context's colour input setting).
struct HostInputs {
    InputKind kind;
    int n;
    const uint8_t* const* gray; const uint8_t* const* right; int stride;
    const float* const* pts; const int* n_pts; int layout;
    const uint16_t* const* depth; int depth_stride;
    int ch = 1;

    static HostInputs rgbl(int n, const uint8_t* const* gray, int stride, const float* const* pts, const int* n_pts, int layout = 0) {
        return {InputKind::rgbl, n, gray, nullptr, stride, pts, n_pts, layout, nullptr, 0};
    }
    static HostInputs rgbd(int n, const uint8_t* const* gray, int stride, const uint16_t* const* depth, int depth_stride) {
        return {InputKind::rgbd, n, gray, nullptr, stride, nullptr, nullptr, 0, depth, depth_stride};
    }
    static HostInputs stereo(int n, const uint8_t* const* left, const uint8_t* const* right, int stride) {
        return {InputKind::stereo, n, left, right, stride, nullptr, nullptr, 0, nullptr, 0};
    }
    // the images are camera input, of the context's channel count (rgbl_set_input_channels)
    HostInputs camera(const Ctx* c) const { HostInputs r = *this; r.ch = c->input.ch; return r; }
    // batch b of consecutive batches of n
    HostInputs batch(int b) const {
        const size_t o = (size_t)b * n;
        HostInputs r = *this;
        if (gray) r.gray += o;
        if (right) r.right += o;
        if (pts) r.pts += o;
        if (n_pts) r.n_pts += o;
        if (depth) r.depth += o;
        return r;
    }
};

// A missing image or depth image is RGBL_E_EMPTY, a bad point cloud RGBL_E_CAPACITY -> *max_pts: the largest cloud.
static int check_inputs(Ctx* c, const HostInputs& in, int* max_pts) {
    *max_pts = 0;
    if (in.kind == InputKind::rgbl) {
        if (!c->d_pts) { c->err = "context was created with max_points == 0"; return RGBL_E_INVALID; }
        for (int f = 0; f < in.n; ++f) {
            if (in.gray && !in.gray[f]) { c->err = "empty image"; return RGBL_E_EMPTY; }
            if (in.n_pts[f] < 0 || in.n_pts[f] > c->cfg.max_points || (in.n_pts[f] && !in.pts[f])) { c->err = "bad point cloud"; return RGBL_E_CAPACITY; }
            *max_pts = std::max(*max_pts, in.n_pts[f]);
        }
        return RGBL_OK;
    }
    for (int f = 0; f < in.n; ++f)
        if (!in.gray[f] || (in.right && !in.right[f])) { c->err = "empty image"; return RGBL_E_EMPTY; }
    if (in.kind == InputKind::rgbd) {
        if (!in.depth || in.depth_stride < c->input.w) { c->err = !in.depth ? "null argument" : "depth_stride < width"; return RGBL_E_INVALID; }
        for (int f = 0; f < in.n; ++f) if (!in.depth[f]) { c->err = "empty depth image"; return RGBL_E_EMPTY; }
    }
    return RGBL_OK;
}

// cv::imread(PNG, IMREAD_UNCHANGED) + cvtColor to gray (Examples/RGB-L/rgbl_kitti.cc:87, src/Tracking.cc:1567-1580) into the image planes
// of the batch: host inflate into pinned staging, H2D of the filtered scanlines, reconstruction + gray on the device.
static int ensure_png_staging(Ctx* c, int width, int height) {
    const size_t w = width, B = c->cfg.max_batch;
    c->png_raw_stride = ((w * 4 + 1) * height + 255) & ~(size_t)255;
    if (!c->d_png_status) {          // allocated and zeroed, or not at all
        if (c->d_png_status.alloc(1) != cudaSuccess) { c->err = "allocation of the PNG staging buffers failed"; return RGBL_E_CUDA; }
        if (cudaMemset(c->d_png_status, 0, sizeof(int)) != cudaSuccess) { c->d_png_status.reset(); c->err = "cudaMemset failed (PNG status word)"; return RGBL_E_CUDA; }
    }
    if (!ensure(c->d_png_raw, c->png_raw_stride * B) || !ensure(c->h_png_raw, c->png_raw_stride * B) || !ensure(c->d_png_band, B * w) ||
        !ensure(c->h_png_status, 1)) {
        c->err = "allocation of the PNG staging buffers failed"; return RGBL_E_CUDA;
    }
    return RGBL_OK;
}

// host inflate of n PNG streams of w x h pixels into the pinned staging buffer + H2D of the filtered scanlines -> bytes per pixel (or < 0).
// gray_only: if given, a colour stream is RGBL_E_UNSUPPORTED with this message, refused before anything is copied.
static int inflate_png_batch(Ctx* c, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int w, int h, bool depth16, cudaStream_t st,
                             const char* gray_only = nullptr) {
    int rc = ensure_png_staging(c, w, h); if (rc) return rc;
    for (int f = 0; f < n_frames; ++f) if (!png[f] || !png_bytes[f]) { c->err = "empty image"; return RGBL_E_EMPTY; }
    int ch = 0;
    std::string perr;
    const int prc = png_inflate_batch(n_frames, png, png_bytes, w, h, c->h_png_raw, c->png_raw_stride, &ch, perr, depth16);
    if (prc) { c->err = perr; return prc == -2 ? RGBL_E_UNSUPPORTED : RGBL_E_INVALID; }
    if (gray_only && ch != 1) { c->err = gray_only; return RGBL_E_UNSUPPORTED; }
    const size_t used = ((size_t)w * ch + 1) * h;
    for (int f = 0; f < n_frames; ++f)
        CU(cudaMemcpyAsync(c->d_png_raw + (size_t)f * c->png_raw_stride, c->h_png_raw + (size_t)f * c->png_raw_stride, used, cudaMemcpyHostToDevice, st));
    return ch;
}

// after the reconstruction kernel: wait for it and report a bad scanline filter byte
static int png_status(Ctx* c, cudaStream_t st) {
    CU(cudaMemcpyAsync(c->h_png_status, c->d_png_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));          // the staging buffer is free again, and a bad scanline filter byte is an error of THIS call
    if (*c->h_png_status) {
        CU(cudaMemsetAsync(c->d_png_status, 0, sizeof(int), st));
        c->err = "corrupt PNG: scanline filter type above 4"; return RGBL_E_INVALID;
    }
    return RGBL_OK;
}

// The kernel that writes level 0 from a batch of `kind` with ch bytes per pixel: System::TrackStereo's remap (rectification on), else
// TrackRGBD's / TrackStereo's resize (input resize on; RGB-D depth images too), else GrabImage*'s cvtColor of colour images, which the
// remap and the resize also apply; direct: the upload writes level 0.  All but direct read the batch's raw planes (LoadedInput).
enum class Level0 { direct, gray, resize, remap };
static Level0 level0_writer(const Ctx* c, InputKind kind, int ch) {
    if (kind == InputKind::stereo && c->input.rectify) return Level0::remap;
    if (kind != InputKind::rgbl && c->input.resize) return Level0::resize;
    return ch > 1 ? Level0::gray : Level0::direct;
}
static bool depth_resized(const Ctx* c) { return level0_writer(c, InputKind::rgbd, 1) == Level0::resize; }

// Where the image planes (ch bytes per pixel) of the batch being loaded go: into stage slot `slot` if given, else level 0 of the frame
// slots.  With a level-0 writer (level0_writer), the raw planes it reads, recorded in `loaded` with the context's gray weight: the
// planes of the slot `staged` that already holds them (base == nullptr: nothing to copy), or else d_raw_img.
static int image_planes(Ctx* c, InputKind kind, int ch, Ctx::StageSlot* slot, const Ctx::StageSlot* staged, Planes* p) {
    const InputSetting& in = c->input;
    if (slot) { *p = {slot->img, in.plane_bytes(), 0, in.pitch, in.w, in.h, ch}; return RGBL_OK; }
    if (level0_writer(c, kind, ch) == Level0::direct) { *p = level0_planes(c); c->loaded.ch = 0; return RGBL_OK; }
    const int pitch = staged ? in.pitch : input_pitch(c, ch);
    if (staged) *p = {};
    else if (!ensure(c->d_raw_img, (size_t)c->cfg.max_batch * pitch * in.h)) { c->err = "device allocation failed (raw image planes)"; return RGBL_E_CUDA; }
    else *p = {c->d_raw_img, (size_t)pitch * in.h, 0, pitch, in.w, in.h, ch};
    c->loaded = {staged ? staged->img.get() : c->d_raw_img.get(), ch, in.w0, pitch, c->loaded.depth};
    return RGBL_OK;
}

// n PNG streams into the image planes of the batch being loaded (image_planes).  Without a level-0 writer the unfilter kernel converts to
// gray and writes level 0.  With the remap or the resize, the reference converts the image imread returned to gray after it, which differs
// for colour images: the raw planes then take the reconstructed pixels as they are, colour streams on a colour context only (a gray
// context refuses them).  The file's samples are in R, G, B order, imread's in B, G, R: channel 0 gets the red weight when camera_rgb is 0.
static int decode_png_gray(Ctx* c, InputKind kind, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb, cudaStream_t st) {
    const Level0 writer = level0_writer(c, kind, 1);
    const bool raw = writer != Level0::direct;
    const char* gray_only = !raw || c->input.ch > 1 ? nullptr
                          : writer == Level0::remap ? "rectified stereo takes 8-bit gray PNGs only on a gray context (the reference remaps colour images before their conversion to gray; rgbl_set_input_channels)"
                                                    : "with the input resize on, image PNGs must be 8-bit gray on a gray context (the reference resizes colour images before their conversion to gray; rgbl_set_input_channels)";
    const int ch = inflate_png_batch(c, n_frames, png, png_bytes, raw ? c->input.w : c->cfg.width, raw ? c->input.h : c->cfg.height, false, st, gray_only);
    if (ch < 0) return ch;
    Planes p;
    int rc = image_planes(c, kind, raw ? ch : 1, nullptr, nullptr, &p); if (rc) return rc;
    if (p.ch > 1) {
        launch_png_unfilter_pixels(st, c->d_png_raw, c->png_raw_stride, p.w, p.h, ch, p.base, p.stride, p.pitch, c->d_png_band, c->d_png_status, n_frames);
        c->loaded.w0 = camera_rgb ? 3735 : 9798;
    } else {
        LevelGeom g = c->levels[0];
        g.off = p.off; g.pitch = p.pitch;
        launch_png_unfilter_gray(st, c->d_png_raw, c->png_raw_stride, p.w, p.h, ch, raw ? 0 : camera_rgb, p.base, p.stride, g,
                                 c->d_png_band, c->d_png_status, n_frames);
    }
    return png_status(c, st);
}

static size_t depth16_frame_elems(const Ctx* c) { return c->depth16_pitch * c->cfg.height; }

static int ensure_depth16(Ctx* c) {
    c->depth16_pitch = ((size_t)c->cfg.width * sizeof(uint16_t) + 63) / 64 * 32;
    if (!ensure(c->d_depth16, c->depth16_pitch * c->cfg.height * c->cfg.max_batch)) { c->err = "device allocation failed (RGB-D depth planes)"; return RGBL_E_CUDA; }
    if (depth_resized(c) && !ensure(c->d_depth16_raw, c->input.depth_elems() * c->cfg.max_batch)) { c->err = "device allocation failed (RGB-D input-size depth planes)"; return RGBL_E_CUDA; }
    return RGBL_OK;
}

// Where the input-size depth images of the RGB-D batch being loaded go: into stage slot `slot` if given, else d_depth16, or with the depth
// resize into its source, recorded in `loaded`: the slot `staged` that already holds them (nullptr: nothing to copy), or else d_depth16_raw.
static uint16_t* depth_planes(Ctx* c, Ctx::StageSlot* slot, const Ctx::StageSlot* staged) {
    if (slot) return slot->depth;
    if (!depth_resized(c)) return c->d_depth16;
    c->loaded.depth = staged ? staged->depth.get() : c->d_depth16_raw.get();
    return staged ? nullptr : c->d_depth16_raw.get();
}

// cv::imread(depth PNG, IMREAD_UNCHANGED) of Examples/RGB-D/rgbd_kitti.cc into the uint16 depth planes of frame slots 0..n_frames-1
// (16-bit gray only); shares the staging buffer with the image decode, one after the other.  camera: the streams are camera input,
// decoded at the input size into the depth planes of the batch being loaded (depth_planes); else at the context's size into d_depth16.
static int decode_png_to_depth16(Ctx* c, int n_frames, const uint8_t* const* png, const size_t* png_bytes, cudaStream_t st, bool camera) {
    int rc = ensure_depth16(c); if (rc) return rc;
    const int w = camera ? c->input.w : c->cfg.width, h = camera ? c->input.h : c->cfg.height;
    const int ch = inflate_png_batch(c, n_frames, png, png_bytes, w, h, true, st);
    if (ch < 0) return ch;
    uint16_t* dst = camera ? depth_planes(c, nullptr, nullptr) : c->d_depth16.get();
    launch_png_unfilter_depth16(st, c->d_png_raw, c->png_raw_stride, w, h, dst, camera ? c->input.depth_elems() : depth16_frame_elems(c),
                                camera ? c->input.depth_pitch : c->depth16_pitch, c->d_png_band, c->d_png_status, n_frames);
    return png_status(c, st);
}

// device buffers of a stage slot (allocated on first use, grown for a larger input size; a slot can hold batches of each kind in turn)
static int stage_slot_alloc(Ctx* c, Ctx::StageSlot& sl, InputKind kind) {
    const size_t B = c->cfg.max_batch;
    bool ok = ensure(sl.img, B * c->input.plane_bytes());     // stereo: the left and the right planes, 2 n_pairs <= max_batch
    if (ok && kind == InputKind::rgbd) ok = ensure(sl.depth, B * c->input.depth_elems());
    if (ok && kind == InputKind::rgbl) ok = ensure(sl.pts, B * 4 * c->cfg.max_points) && ensure(sl.n_pts, B);
    if (!ok) { c->err = "device allocation failed (stage slot)"; return RGBL_E_CUDA; }
    return RGBL_OK;
}

// H2D of a checked host batch into stage slot `slot`, or (nullptr) into the working buffers: the image planes (image_planes), d_pts (or
// d_pts_raw, de-interleaved into d_pts) and d_n_pts, d_depth16.  Clouds and depth images go on the aux stream, images on the main one.
static int copy_inputs(Ctx* c, const HostInputs& in, int max_pts, Ctx::StageSlot* slot) {
    const bool kitti = in.kind == InputKind::rgbl && in.layout == 1;
    if (in.kind == InputKind::rgbd) { int rc = ensure_depth16(c); if (rc) return rc; }
    if (kitti && !ensure(c->d_pts_raw, (size_t)c->cfg.max_batch * 4 * c->cfg.max_points)) { c->err = "device allocation failed (raw point records)"; return RGBL_E_CUDA; }
    if (slot) { int rc = stage_slot_alloc(c, *slot, in.kind); if (rc) return rc; }
    if (in.kind == InputKind::rgbl) {
        float* pts = slot ? slot->pts.get() : kitti ? c->d_pts_raw.get() : c->d_pts.get();
        for (int f = 0; f < in.n; ++f) {
            c->h_n_pts[f] = in.n_pts[f];
            if (in.n_pts[f]) CU(cudaMemcpyAsync(pts + (size_t)f * 4 * c->cfg.max_points, in.pts[f], (size_t)4 * in.n_pts[f] * sizeof(float), cudaMemcpyHostToDevice, c->st_aux));
        }
        CU(cudaMemcpyAsync(slot ? slot->n_pts.get() : c->d_n_pts.get(), c->h_n_pts, (size_t)in.n * sizeof(int), cudaMemcpyHostToDevice, c->st_aux));
        if (kitti && max_pts > 0) launch_deinterleave_xyzr(c->st_aux, c->d_pts_raw, c->d_pts, 4 * c->cfg.max_points, c->d_n_pts, max_pts, in.n);
    } else if (in.kind == InputKind::rgbd) {
        uint16_t* depth = depth_planes(c, slot, nullptr);
        for (int f = 0; f < in.n; ++f)
            CU(cudaMemcpy2DAsync(depth + (size_t)f * c->input.depth_elems(), c->input.depth_pitch * sizeof(uint16_t), in.depth[f],
                                 (size_t)in.depth_stride * sizeof(uint16_t), (size_t)c->input.w * sizeof(uint16_t), c->input.h, cudaMemcpyHostToDevice, c->st_aux));
    }
    if (!in.gray) return RGBL_OK;          // level 0 was written by a PNG decode
    Planes p;
    int rc = image_planes(c, in.kind, in.ch, slot, nullptr, &p); if (rc) return rc;
    rc = upload_planes(c, p, 0, in.n, in.gray, in.stride, c->st); if (rc) return rc;
    return in.right ? upload_planes(c, p, in.n, in.n, in.right, in.stride, c->st) : RGBL_OK;
}

// a host batch -> the working buffers, which then hold the resident batch
static int upload_inputs(Ctx* c, const HostInputs& in) {
    int max_pts = 0;
    int rc = check_inputs(c, in, &max_pts); if (rc) return rc;
    rc = copy_inputs(c, in, max_pts, nullptr); if (rc) return rc;
    set_resident(c, in.kind, in.n, max_pts);
    return RGBL_OK;
}

// upload_inputs, then wait for both streams (the host buffers are free again)
static int upload_inputs_sync(Ctx* c, const HostInputs& in) {
    int rc = upload_inputs(c, in); if (rc) return rc;
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    return RGBL_OK;
}

// a host batch -> stage slot `slot`, for a later restage
static int stage_inputs(Ctx* c, int slot, const HostInputs& in) {
    int max_pts = 0;
    int rc = check_inputs(c, in, &max_pts); if (rc) return rc;
    Ctx::StageSlot& sl = c->stage[slot];
    rc = copy_inputs(c, in, max_pts, &sl); if (rc) return rc;
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    sl.n_frames = in.n; sl.max_pts = max_pts; sl.kind = in.kind; sl.input = c->input;
    return RGBL_OK;
}

// The level0 step of run_extract for the n images of the loaded batch (stereo: n / 2 pairs, left then right): its level-0 writer on the
// main stream (nullptr: direct).  With both the rectification and the resize on, the remap reads the input-size planes: its maps have the
// context's size and index the input-size images (Settings builds them with initUndistortRectifyMap(..., newImSize_, ...)).
static int level0_step(Ctx* c, InputKind kind, int n, std::function<int()>* step) {
    const Level0 writer = level0_writer(c, kind, c->loaded.ch);
    *step = nullptr;
    if (writer == Level0::direct) return RGBL_OK;
    if (!c->loaded.img || !c->loaded.ch) { c->err = writer == Level0::remap ? "no raw stereo planes to rectify" : "no input-size planes to resize"; return RGBL_E_INVALID; }
    *step = [c, n, writer]() {
        const LoadedInput& ld = c->loaded;
        const size_t stride = (size_t)ld.pitch * c->input.h;
        LevelGeom src{};
        src.w = c->input.w; src.h = c->input.h; src.pitch = ld.pitch;
        if (writer == Level0::remap) {
            const LevelGeom& l0 = c->levels[0];
            RectifyDev r{};
            r.xy = c->d_rect_xy; r.a = c->d_rect_a; r.map_pitch = c->rect_pitch;
            r.W = c->cfg.width; r.H = c->cfg.height; r.src_W = c->input.w; r.src_H = c->input.h;
            r.src = ld.img; r.src_stride = stride; r.src_pitch = ld.pitch; r.ch = ld.ch; r.w0 = ld.w0;
            r.dst = c->d_pyr; r.dst_stride = c->frame_bytes; r.dst_off = l0.off; r.dst_pitch = l0.pitch;
            launch_rectify(c->st, r, n / 2);
        } else if (writer == Level0::resize) {
            launch_resize_planes(c->st, ld.img, stride, src, c->d_pyr, c->frame_bytes, c->levels[0], c->d_resize_coefs,
                                 c->d_resize_coefs + c->cfg.width, n, ld.ch, ld.w0);
        } else {
            launch_gray_planes(c->st, ld.img, stride, src, c->d_pyr, c->frame_bytes, c->levels[0], ld.ch, ld.w0, n);
        }
        return 1;
    };
    return RGBL_OK;
}

// Everything of Frame::Frame (RGB-L) after the inputs are in HBM: (colour input: the gray conversion into level 0, level0_step), depth
// maps (aux stream) || extraction, then gather.
static int process_rgbl(Ctx* c, int n_frames, int max_pts, const float P[12], const rgbl_depth_params* prm) {
    DepthDev dd;
    int rc = setup_depth(c, P, prm, dd); if (rc) return rc;
    std::function<int()> level0;
    rc = level0_step(c, InputKind::rgbl, n_frames, &level0); if (rc) return rc;
    // depth maps run on the aux stream behind the blur, overlapping the host quad-tree; describe waits for both
    int max_n = run_extract(c, n_frames, [&]() { run_depth_maps(c, dd, n_frames, max_pts, nullptr, c->st_aux); }, level0);
    if (max_n < 0) return max_n;
    run_depth_keypoints(c, dd, c->d_kps, c->d_kps, c->d_n_sel, max_n, n_frames, c->st, true);
    CU(cudaGetLastError());
    return max_n;
}

// Everything of the RGB-D Frame constructor (src/Frame.cc:200-237) after the inputs are in HBM: extraction, UndistortKeyPoints (context's
// camera, rgbl_set_camera_distortion), then ComputeStereoFromRGBD as the gather of the uint16 depth plane, scaled per pixel like
// GrabImageRGBD's convertTo.  With the input resize on, System::TrackRGBD's cv::resize of the depth images (src/System.cc) writes d_depth16
// on the aux stream, behind the blur and overlapping the quad-tree (billed to depth_gather); the gather waits for it through ev_blur.
static int process_rgbd(Ctx* c, int n_frames, float depth_scale, float bf) {
    std::function<int()> level0;
    std::function<void()> depth_resize;
    int rc = level0_step(c, InputKind::rgbd, n_frames, &level0); if (rc) return rc;
    if (depth_resized(c)) {
        if (!c->loaded.depth) { c->err = "no input-size planes to resize"; return RGBL_E_INVALID; }
        depth_resize = [&]() {
            if (c->prof_on) cudaEventRecord(c->ev_rsd_b, c->st_aux);
            launch_resize_depth16(c->st_aux, c->loaded.depth, c->input.depth_elems(), c->input.depth_pitch, c->input.kx, c->input.ky, c->d_depth16,
                                  depth16_frame_elems(c), c->depth16_pitch, c->cfg.width, c->cfg.height, n_frames);
            if (c->prof_on) { cudaEventRecord(c->ev_rsd_e, c->st_aux); c->rsd_used = true; }
            c->total_launches += 1;
            c->st_pending_launches[ST_DEPTH_GATHER] += 1;
        };
    }
    const int max_n = run_extract(c, n_frames, depth_resize, level0);
    if (max_n < 0) return max_n;
    int launches = max_n > 0 ? 1 : 0;
    stage_begin(c, ST_DEPTH_GATHER, c->st);
    const rgbl_keypoint* kps_un = undistort_keypoints(c, max_n, n_frames, c->st, &launches);
    launch_depth_gather_u16(c->st, c->d_depth16, depth16_frame_elems(c), c->depth16_pitch, depth_scale, c->d_kps, kps_un, c->d_n_sel, c->cap_kp, max_n, bf,
                            c->d_depth, c->d_uright, n_frames);
    stage_end(c, ST_DEPTH_GATHER, c->st, launches);
    CU(cudaGetLastError());
    return max_n;
}

static int check_rgbd_params(Ctx* c, float depth_scale, float bf) {
    if (!std::isfinite(depth_scale) || !(bf > 0.f) || !std::isfinite(bf)) { c->err = "depth_scale must be finite and bf > 0"; return RGBL_E_INVALID; }
    return RGBL_OK;
}

// The stereo Frame constructor (src/Frame.cc:101-197) after the n_pairs left images are in slots [0, n) and the right ones in [n, 2n):
// both extracted as one batch of 2n frames (the reference's two ORBextractor threads), then ComputeStereoMatches.  The left frames are
// then the batch (last_frames = n) for download, ComputeBoW and the tracking chain.  The capacity-overflow flags cover all 2n frames,
// so an overflow in a right frame, which changes the left frame's depths, fails the chain's _end2 like a left-frame overflow.
// The pairs' level-0 writer (TrackStereo's cv::remap or cv::resize, src/System.cc:251 ff.) runs first, billed to the pyramid stage.
static int process_stereo(Ctx* c, int n_pairs, float mb, float mbf) {
    std::function<int()> level0;
    int rc = level0_step(c, InputKind::stereo, 2 * n_pairs, &level0); if (rc) return rc;
    const int max_n = run_extract(c, 2 * n_pairs, nullptr, level0);
    if (max_n < 0) return max_n;
    rc = stereo_matches(c, 0, n_pairs, n_pairs, mb, mbf); if (rc) return rc;
    c->last_frames = n_pairs;
    return max_n;
}

// what every stereo entry point requires: 2 n_pairs <= max_batch, and a rectified camera (mvKeys of the rectified images are matched;
// the stereo Frame constructor undistorts nothing before ComputeStereoMatches)
static int check_stereo(Ctx* c, int n_pairs) {
    if (2 * n_pairs > c->cfg.max_batch) { c->err = "a stereo batch of n pairs takes 2 n frame slots: 2 n_pairs exceeds max_batch"; return RGBL_E_INVALID; }
    if (c->undistort) { c->err = "stereo needs rectified images: this context's camera has k1 != 0 (rgbl_set_camera_distortion)"; return RGBL_E_UNSUPPORTED; }
    return RGBL_OK;
}

// RGB-L input is never resized: the reference's Settings do not handle RGB-L (System::TrackRGBL's resize branch never runs), and the LiDAR
// projection P describes the original image
static int check_rgbl_input(Ctx* c) {
    if (c->input.resize) { c->err = "RGB-L input is never resized: clear the input resize (rgbl_set_input_resize(ctx, 0, 0))"; return RGBL_E_UNSUPPORTED; }
    return RGBL_OK;
}

// RGB-D input with the resize on: the depth resize restates OpenCV's 16-bit INTER_LINEAR at integer factors only
static int check_rgbd_input(Ctx* c) {
    if (depth_resized(c) && !(c->input.kx && c->input.ky)) { c->err = "RGB-D input resize needs integer factors (input width / width and input height / height)"; return RGBL_E_UNSUPPORTED; }
    return RGBL_OK;
}

static int check_stereo_params(Ctx* c, float mb, float mbf) {
    if (!(mb > 0.f) || !std::isfinite(mb) || !(mbf > 0.f) || !std::isfinite(mbf)) { c->err = "mb and mbf must be finite and > 0"; return RGBL_E_INVALID; }
    return RGBL_OK;
}

// the uploaded frames must be of `kind`; else the message names the process call that takes them
static int check_resident_kind(Ctx* c, InputKind kind) {
    if (c->resident_frames < 1) { c->err = "nothing uploaded"; return RGBL_E_INVALID; }
    if (c->resident_kind == kind) return RGBL_OK;
    const KindNames& k = kind_names(c->resident_kind);
    c->err = std::string("the uploaded frames are ") + k.what + " (" + k.process + ")";
    return RGBL_E_INVALID;
}

// the end of every process call: both streams idle, the profile collected, the keypoint counts in n_out (if given)
static int finish_process(Ctx* c, int* n_out) {
    if (n_out) { int rc = fetch_counts(c, c->resident_frames); if (rc) return rc; }
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    prof_collect(c);
    if (n_out) for (int f = 0; f < c->resident_frames; ++f) n_out[f] = c->h_n_sel[f];
    return RGBL_OK;
}

static int download_rgbl(Ctx* c, int n_frames, rgbl_keypoint* kps, uint8_t* desc, float* depth, float* uright, int cap, int* n_out) {
    { int rc = fetch_counts(c, n_frames); if (rc) return rc; }
    for (int f = 0; f < n_frames; ++f) {
        const int n = c->h_n_sel[f];
        n_out[f] = n;
        if (n > cap) { c->err = "output capacity too small"; return RGBL_E_CAPACITY; }
        if (!n) continue;
        CU(cudaMemcpyAsync(kps + (size_t)f * cap, c->d_kps + (size_t)f * c->cap_kp, (size_t)n * sizeof(rgbl_keypoint), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(desc + (size_t)f * cap * 32, c->d_desc + (size_t)f * c->cap_kp * 32, (size_t)n * 32, cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(depth + (size_t)f * cap, c->d_depth + (size_t)f * c->cap_kp, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
        CU(cudaMemcpyAsync(uright + (size_t)f * cap, c->d_uright + (size_t)f * c->cap_kp, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    }
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    prof_collect(c);
    return RGBL_OK;
}

int rgbl_frame_rgbl_batch(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                          const float* const* pts4xn, const int* n_pts, const float P[12], const rgbl_depth_params* prm,
                          rgbl_keypoint* kps, uint8_t* desc, float* depth, float* uright, int cap, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !pts4xn || !n_pts || !P || !prm || !kps || !desc || !depth || !uright || !n_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_images(c, gray_images(c), n_frames, width, height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = upload_inputs(c, HostInputs::rgbl(n_frames, gray, stride, pts4xn, n_pts)); if (rc) return rc;
    rc = process_rgbl(c, n_frames, c->resident_max_pts, P, prm); if (rc < 0) return rc;
    return download_rgbl(c, n_frames, kps, desc, depth, uright, cap, n_out);
}

/* Resident form used to measure device throughput: inputs are uploaded once, processing can then be
 * repeated without any host->device input traffic; results stay in HBM until rgbl_resident_download. */
int rgbl_resident_upload(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                         const float* const* pts4xn, const int* n_pts) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !pts4xn || !n_pts) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_images(c, c->input, n_frames, width, height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return upload_inputs_sync(c, HostInputs::rgbl(n_frames, gray, stride, pts4xn, n_pts).camera(c));
}

int rgbl_resident_upload_kitti(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                               const float* const* xyzr, const int* n_pts) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !xyzr || !n_pts) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_images(c, c->input, n_frames, width, height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return upload_inputs_sync(c, HostInputs::rgbl(n_frames, gray, stride, xyzr, n_pts, 1).camera(c));
}

int rgbl_resident_upload_kitti_png(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb,
                                   const float* const* xyzr, const int* n_pts) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!png || !png_bytes || !xyzr || !n_pts) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_batch(c, n_frames); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = decode_png_gray(c, InputKind::rgbl, n_frames, png, png_bytes, camera_rgb, c->st); if (rc) return rc;
    return upload_inputs_sync(c, HostInputs::rgbl(n_frames, nullptr, 0, xyzr, n_pts, 1));
}

int rgbl_decode_png_gray(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb, uint8_t* const* gray_out,
                         int stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!png || !png_bytes || !gray_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_images(c, gray_images(c), n_frames, c->cfg.width, c->cfg.height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = decode_png_gray(c, InputKind::rgbl, n_frames, png, png_bytes, camera_rgb, c->st); if (rc) return rc;
    const Planes l0 = level0_planes(c);
    for (int f = 0; f < n_frames; ++f) {
        if (!gray_out[f]) { c->err = "null output image"; return RGBL_E_INVALID; }
        CU(cudaMemcpy2DAsync(gray_out[f], stride, l0.at(f), l0.pitch, c->cfg.width, c->cfg.height, cudaMemcpyDeviceToHost, c->st));
    }
    CU(cudaStreamSynchronize(c->st));
    return RGBL_OK;
}

int rgbl_resident_process(rgbl_ctx* ctx, const float P[12], const rgbl_depth_params* prm, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!P || !prm) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_resident_kind(c, InputKind::rgbl); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = process_rgbl(c, c->resident_frames, c->resident_max_pts, P, prm); if (rc < 0) return rc;
    return finish_process(c, n_out);
}

/* ---- sequence runner: many consecutive batches of ONE sequence per host call ------------------------------------------------------
 * The per-batch calls above return to the caller between batches; with a slow caller (Python, several ranks on one host) the device
 * waits for the host.  rgbl_track_sequence keeps the whole loop native: per batch  inputs (host buffers, or a staged device slot) ->
 * frame construction -> tracking chain (queued two deep on the tracking stream, continue_sequence from the second batch on) -> poses
 * (and, if asked for, the frame-construction outputs) back to the host.  Nothing synchronises with the device until a chain's results
 * are collected, one batch behind.                                                                                                   */
int rgbl_resident_stage(rgbl_ctx* ctx, int slot, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                        const float* const* pts4xn, const int* n_pts) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !pts4xn || !n_pts) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (slot < 0 || slot >= Ctx::kMaxStageSlots) { c->err = "stage slot out of range"; return RGBL_E_INVALID; }
    if (!c->d_pts) { c->err = "context was created with max_points == 0"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_images(c, c->input, n_frames, width, height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return stage_inputs(c, slot, HostInputs::rgbl(n_frames, gray, stride, pts4xn, n_pts).camera(c));
}

int rgbl_resident_stage_rgbd(rgbl_ctx* ctx, int slot, int n_frames, const uint8_t* const* gray, int width, int height, int stride,
                             const uint16_t* const* depth, int depth_stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !depth) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (slot < 0 || slot >= Ctx::kMaxStageSlots) { c->err = "stage slot out of range"; return RGBL_E_INVALID; }
    int rc = check_rgbd_input(c); if (rc) return rc;
    rc = check_images(c, c->input, n_frames, width, height, stride); if (rc) return rc;
    if (depth_stride < width) { c->err = "depth_stride < width"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    return stage_inputs(c, slot, HostInputs::rgbd(n_frames, gray, stride, depth, depth_stride).camera(c));
}

int rgbl_resident_stage_stereo(rgbl_ctx* ctx, int slot, int n_pairs, const uint8_t* const* left, const uint8_t* const* right, int width, int height,
                               int stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!left || !right) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (slot < 0 || slot >= Ctx::kMaxStageSlots) { c->err = "stage slot out of range"; return RGBL_E_INVALID; }
    int rc = check_images(c, c->input, n_pairs, width, height, stride); if (rc) return rc;
    rc = check_stereo(c, n_pairs); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return stage_inputs(c, slot, HostInputs::stereo(n_pairs, left, right, stride).camera(c));
}

// staged slot -> the context's working input buffers (device-to-device, ~76 MB per 32 KITTI frames: tens of microseconds); the slot must hold
// frames of the kind the caller processes
static int restage(Ctx* c, int slot, InputKind kind) {
    const Ctx::StageSlot& sl = c->stage[slot];
    if (!sl.img || sl.n_frames < 1) { c->err = "stage slot is empty"; return RGBL_E_INVALID; }
    if (sl.kind != kind) {
        const KindNames& k = kind_names(sl.kind);
        c->err = std::string("stage slot holds ") + k.what + " (" + k.runner + ")";
        return RGBL_E_INVALID;
    }
    if (sl.input.w != c->input.w || sl.input.h != c->input.h) { c->err = "stage slot was staged at another input size (rgbl_set_input_resize)"; return RGBL_E_INVALID; }
    if (sl.input.ch != c->input.ch) { c->err = "stage slot was staged with another channel count (rgbl_set_input_channels)"; return RGBL_E_INVALID; }
    Planes dst;
    int rc = image_planes(c, kind, sl.input.ch, nullptr, &sl, &dst); if (rc) return rc;
    const size_t img_bytes = sl.input.plane_bytes();
    const int n_img = kind == InputKind::stereo ? 2 * sl.n_frames : sl.n_frames;
    if (dst.base)
        for (int f = 0; f < n_img; ++f) CU(cudaMemcpyAsync(dst.at(f), sl.img + (size_t)f * img_bytes, img_bytes, cudaMemcpyDeviceToDevice, c->st));
    if (kind == InputKind::rgbd) {
        uint16_t* depth = depth_planes(c, nullptr, &sl);
        if (depth) CU(cudaMemcpyAsync(depth, sl.depth, (size_t)sl.n_frames * sl.input.depth_elems() * sizeof(uint16_t), cudaMemcpyDeviceToDevice, c->st_aux));
    } else if (kind == InputKind::rgbl) {
        CU(cudaMemcpyAsync(c->d_pts, sl.pts, (size_t)sl.n_frames * 4 * c->cfg.max_points * sizeof(float), cudaMemcpyDeviceToDevice, c->st_aux));
        CU(cudaMemcpyAsync(c->d_n_pts, sl.n_pts, (size_t)sl.n_frames * sizeof(int), cudaMemcpyDeviceToDevice, c->st_aux));
    }
    set_resident(c, kind, sl.n_frames, sl.max_pts);
    return RGBL_OK;
}

// Argument checks both sequence runners share (batch geometry, no chain in flight, staged-slot count, frame outputs).
static int check_sequence_io(Ctx* c, const rgbl_chain_params* chain, const rgbl_sequence_io* io) {
    if (!chain || !io || !io->poses || !io->n_matches || !io->n_inliers) { c->err = "null argument"; return RGBL_E_INVALID; }
    const int T = io->frames_per_batch, nb = io->n_batches;
    if (T < 1 || T > c->cfg.max_batch || nb < 1) { c->err = "bad batch geometry"; return RGBL_E_INVALID; }
    if (const int rc = require_idle(c)) return rc;
    if (T % c->lanes) { c->err = "frames_per_batch is not a multiple of the sequence count (rgbl_set_sequences)"; return RGBL_E_INVALID; }
    if (io->gray) {
        int rc = check_images(c, c->input, T, io->width, io->height, io->stride); if (rc) return rc;
    } else if (io->n_slots < 1 || io->n_slots > Ctx::kMaxStageSlots) { c->err = "resident mode needs 1..8 staged slots"; return RGBL_E_INVALID; }
    if (io->kps && (!io->desc || !io->depth || !io->uright || !io->n_kp || io->cap != c->cap_kp)) {
        c->err = "frame outputs need kps, desc, depth, uright, n_kp and cap == rgbl_keypoint_capacity()"; return RGBL_E_INVALID;
    }
    return RGBL_OK;
}

// The per-batch load of the sequence runners: batch b's staged slot (resident mode), or batch b of the host inputs `in`.
static std::function<int(int)> batch_loader(Ctx* c, const rgbl_sequence_io* io, const HostInputs& in) {
    return [=](int b) { return io->gray ? upload_inputs(c, in.batch(b)) : restage(c, (io->first_slot + b) % io->n_slots, in.kind); };
}

// The batch loop of both sequence runners: per batch  load(b) -> construct() -> (frame outputs D2H) -> tracking chain queued two deep
// (continue_sequence from the second batch on), results collected one batch behind; on an error the queued chains are drained first.
// load(b) puts batch b's inputs into the working buffers (host upload or staged slot); construct() runs the frame construction and
// returns < 0 on error.
static int run_sequence(Ctx* c, const rgbl_chain_params* chain, const rgbl_sequence_io* io, const std::function<int(int)>& load,
                        const std::function<int()>& construct) {
    rgbl_ctx* ctx = reinterpret_cast<rgbl_ctx*>(c);
    const int T = io->frames_per_batch, nb = io->n_batches;
    const bool want_frames = io->kps != nullptr;
    rgbl_chain_params cp = *chain;
    int collected = 0;
    auto collect = [&]() -> int {
        const size_t o = (size_t)collected * T;
        const int rc = rgbl_resident_track_end2(ctx, io->poses + o * 7, io->n_matches + o, io->n_inliers + o,
                                                io->n_local_matches ? io->n_local_matches + o : nullptr, nullptr);
        ++collected;
        return rc;
    };
    for (int b = 0; b < nb; ++b) {
        int rc = load(b);
        if (!rc && c->resident_frames != T) { c->err = "staged slot holds a different number of frames"; rc = RGBL_E_INVALID; }
        if (rc) { while (c->chain_pending) collect(); return rc; }
        rc = construct();
        if (rc < 0) { while (c->chain_pending) collect(); return rc; }
        if (want_frames) {        // whole [T][cap] arrays + counts, asynchronously behind the batch's kernels
            const size_t o = (size_t)b * T, n = (size_t)T * c->cap_kp;
            CU(cudaMemcpyAsync(io->kps + o * io->cap, c->d_kps, n * sizeof(rgbl_keypoint), cudaMemcpyDeviceToHost, c->st));
            CU(cudaMemcpyAsync(io->desc + o * io->cap * 32, c->d_desc, n * 32, cudaMemcpyDeviceToHost, c->st));
            CU(cudaMemcpyAsync(io->depth + o * io->cap, c->d_depth, n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
            CU(cudaMemcpyAsync(io->uright + o * io->cap, c->d_uright, n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
            CU(cudaMemcpyAsync(io->n_kp + o, c->d_n_sel, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost, c->st));
        }
        cp.continue_sequence = (b > 0 || chain->continue_sequence) ? 1 : 0;
        rc = rgbl_resident_track_begin2(ctx, &cp);
        if (rc) { while (c->chain_pending) collect(); return rc; }
        if (c->chain_pending == 2) { rc = collect(); if (rc) { while (c->chain_pending) collect(); return rc; } }
    }
    int rc_all = RGBL_OK;
    while (c->chain_pending) { const int rc = collect(); if (rc && !rc_all) rc_all = rc; }
    CU(cudaStreamSynchronize(c->st));
    CU(cudaStreamSynchronize(c->st_aux));
    prof_collect(c);
    return rc_all;
}

int rgbl_track_sequence(rgbl_ctx* ctx, const float P[12], const rgbl_depth_params* prm, const rgbl_chain_params* chain, const rgbl_sequence_io* io) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!P || !prm) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbl_input(c); if (rc) return rc;
    rc = check_sequence_io(c, chain, io); if (rc) return rc;
    if (io->gray && (!io->pts4xn || !io->n_pts)) { c->err = "null argument"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    const int T = io->frames_per_batch;
    const auto load = batch_loader(c, io, HostInputs::rgbl(T, io->gray, io->stride, io->pts4xn, io->n_pts).camera(c));
    return run_sequence(c, chain, io, load, [&]() { return process_rgbl(c, T, c->resident_max_pts, P, prm); });
}

int rgbl_track_sequence_rgbd(rgbl_ctx* ctx, float depth_scale, float bf, const rgbl_chain_params* chain, const rgbl_sequence_io* io,
                             const uint16_t* const* depth, int depth_stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    int rc = check_sequence_io(c, chain, io); if (rc) return rc;
    rc = check_rgbd_params(c, depth_scale, bf); if (rc) return rc;
    rc = check_rgbd_input(c); if (rc) return rc;
    if (io->pts4xn || io->n_pts) { c->err = "RGB-D sequences take depth images, not point clouds (pts4xn / n_pts must be NULL)"; return RGBL_E_INVALID; }
    if (io->gray && (!depth || depth_stride < io->width)) { c->err = "host mode needs one depth image per frame and depth_stride >= width"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    const int T = io->frames_per_batch;
    const auto load = batch_loader(c, io, HostInputs::rgbd(T, io->gray, io->stride, depth, depth_stride).camera(c));
    return run_sequence(c, chain, io, load, [&]() { return process_rgbd(c, T, depth_scale, bf); });
}

int rgbl_track_sequence_stereo(rgbl_ctx* ctx, float mb, float mbf, const rgbl_chain_params* chain, const rgbl_sequence_io* io, const uint8_t* const* right) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    int rc = check_sequence_io(c, chain, io); if (rc) return rc;
    rc = check_stereo_params(c, mb, mbf); if (rc) return rc;
    rc = check_stereo(c, io->frames_per_batch); if (rc) return rc;
    if (io->pts4xn || io->n_pts) { c->err = "stereo sequences take right images, not point clouds (pts4xn / n_pts must be NULL)"; return RGBL_E_INVALID; }
    if (io->gray && !right) { c->err = "host mode needs one right image per frame"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    const int T = io->frames_per_batch;
    const auto load = batch_loader(c, io, HostInputs::stereo(T, io->gray, right, io->stride).camera(c));
    return run_sequence(c, chain, io, load, [&]() { return process_stereo(c, T, mb, mbf); });
}

// ---- RGB-D frame construction (resident form) ----
int rgbl_resident_upload_rgbd(rgbl_ctx* ctx, int n_frames, const uint8_t* const* gray, int width, int height, int stride, const uint16_t* const* depth,
                              int depth_stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!gray || !depth) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbd_input(c); if (rc) return rc;
    rc = check_images(c, c->input, n_frames, width, height, stride); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return upload_inputs_sync(c, HostInputs::rgbd(n_frames, gray, stride, depth, depth_stride).camera(c));
}

int rgbl_resident_upload_rgbd_png(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, int camera_rgb,
                                  const uint8_t* const* depth_png, const size_t* depth_png_bytes) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!png || !png_bytes || !depth_png || !depth_png_bytes) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_rgbd_input(c); if (rc) return rc;
    rc = check_batch(c, n_frames); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = decode_png_gray(c, InputKind::rgbd, n_frames, png, png_bytes, camera_rgb, c->st); if (rc) return rc;
    rc = decode_png_to_depth16(c, n_frames, depth_png, depth_png_bytes, c->st, true); if (rc) return rc;
    set_resident(c, InputKind::rgbd, n_frames, 0);
    return RGBL_OK;
}

int rgbl_decode_png_depth16(rgbl_ctx* ctx, int n_frames, const uint8_t* const* png, const size_t* png_bytes, uint16_t* const* depth_out, int stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!png || !png_bytes || !depth_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_images(c, gray_images(c), n_frames, c->cfg.width, c->cfg.height, stride); if (rc) return rc;
    for (int f = 0; f < n_frames; ++f) if (!depth_out[f]) { c->err = "null output image"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    rc = decode_png_to_depth16(c, n_frames, png, png_bytes, c->st, false); if (rc) return rc;
    for (int f = 0; f < n_frames; ++f)
        CU(cudaMemcpy2DAsync(depth_out[f], (size_t)stride * sizeof(uint16_t), c->d_depth16 + (size_t)f * depth16_frame_elems(c), c->depth16_pitch * sizeof(uint16_t),
                             (size_t)c->cfg.width * sizeof(uint16_t), c->cfg.height, cudaMemcpyDeviceToHost, c->st));
    CU(cudaStreamSynchronize(c->st));
    return RGBL_OK;
}

int rgbl_resident_process_rgbd(rgbl_ctx* ctx, float depth_scale, float bf, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    int rc = check_resident_kind(c, InputKind::rgbd); if (rc) return rc;
    rc = check_rgbd_params(c, depth_scale, bf); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = process_rgbd(c, c->resident_frames, depth_scale, bf); if (rc < 0) return rc;
    return finish_process(c, n_out);
}

// ---- stereo frame construction (resident form): n pairs = one batch of 2n frames, left images in slots [0, n), right ones in [n, 2n) ----
int rgbl_resident_upload_stereo(rgbl_ctx* ctx, int n_pairs, const uint8_t* const* left, const uint8_t* const* right, int width, int height, int stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!left || !right) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_images(c, c->input, n_pairs, width, height, stride); if (rc) return rc;
    rc = check_stereo(c, n_pairs); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    return upload_inputs_sync(c, HostInputs::stereo(n_pairs, left, right, stride).camera(c));
}

int rgbl_resident_upload_stereo_png(rgbl_ctx* ctx, int n_pairs, const uint8_t* const* left_png, const size_t* left_bytes, const uint8_t* const* right_png,
                                    const size_t* right_bytes, int camera_rgb) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!left_png || !left_bytes || !right_png || !right_bytes) { c->err = "null argument"; return RGBL_E_INVALID; }
    int rc = check_batch(c, n_pairs); if (rc) return rc;
    rc = check_stereo(c, n_pairs); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    // one decode of 2n streams: every stream must have the input size, so left and right sizes that differ are an error
    std::vector<const uint8_t*> png(left_png, left_png + n_pairs);
    std::vector<size_t> bytes(left_bytes, left_bytes + n_pairs);
    png.insert(png.end(), right_png, right_png + n_pairs);
    bytes.insert(bytes.end(), right_bytes, right_bytes + n_pairs);
    rc = decode_png_gray(c, InputKind::stereo, 2 * n_pairs, png.data(), bytes.data(), camera_rgb, c->st); if (rc) return rc;
    set_resident(c, InputKind::stereo, n_pairs, 0);
    return RGBL_OK;
}

int rgbl_resident_process_stereo(rgbl_ctx* ctx, float mb, float mbf, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    int rc = check_resident_kind(c, InputKind::stereo); if (rc) return rc;
    rc = check_stereo_params(c, mb, mbf); if (rc) return rc;
    rc = check_stereo(c, c->resident_frames); if (rc) return rc;
    CU(cudaSetDevice(c->cfg.device));
    rc = process_stereo(c, c->resident_frames, mb, mbf); if (rc < 0) return rc;
    return finish_process(c, n_out);
}

// Settings::precomputeRectificationMaps' M1l / M2l / M1r / M2r (cv::initUndistortRectifyMap, CV_32F) -> OpenCV's fixed-point form on the
// device.  Every check runs before anything is written, so a refused setting leaves the previous one in place.
int rgbl_set_stereo_rectification(rgbl_ctx* ctx, const float* m1l, const float* m2l, const float* m1r, const float* m2r, int map_stride) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    const float* maps[4] = {m1l, m2l, m1r, m2r};
    int n_null = 0;
    for (const float* m : maps) n_null += m == nullptr;
    if (n_null == 4) { c->input.rectify = false; input_changed(c, true); return RGBL_OK; }
    if (n_null) { c->err = "the four rectification maps are all given or all NULL"; return RGBL_E_INVALID; }
    const int W = c->cfg.width, H = c->cfg.height;
    if (map_stride < W) { c->err = "map_stride < width"; return RGBL_E_INVALID; }
    for (const float* m : maps)
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                if (!std::isfinite(m[(size_t)y * map_stride + x])) { c->err = "a rectification map holds a value that is not finite"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    c->rect_pitch = (W + 3) & ~3;
    const size_t entries = (size_t)2 * H * c->rect_pitch;
    if (!ensure(c->d_rect_xy, entries) || !ensure(c->d_rect_a, entries)) { c->err = "device allocation failed (rectification maps)"; return RGBL_E_CUDA; }
    DeviceArray<float> staged;       // the float maps, for the conversion only
    if (staged.alloc((size_t)4 * H * W) != cudaSuccess) { c->err = "device allocation failed (rectification map staging)"; return RGBL_E_CUDA; }
    for (int i = 0; i < 4; ++i)
        CU(cudaMemcpy2DAsync(staged + (size_t)i * H * W, (size_t)W * sizeof(float), maps[i], (size_t)map_stride * sizeof(float), (size_t)W * sizeof(float), H,
                             cudaMemcpyHostToDevice, c->st));
    launch_rectify_maps(c->st, staged, W, H, c->d_rect_xy, c->d_rect_a, c->rect_pitch);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->st));
    c->input.rectify = true; input_changed(c, true);
    return RGBL_OK;
}

// Settings::needToResize(): camera images of src_width x src_height resized to the context's size before frame construction (System::TrackRGBD,
// System::TrackStereo).  Every check runs before anything is changed, so a refused setting leaves the previous one in place.
int rgbl_set_input_resize(rgbl_ctx* ctx, int src_width, int src_height) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (src_width < 0 || src_height < 0 || (src_width == 0) != (src_height == 0)) {
        c->err = "the input size is (0, 0) (no resize) or two positive sizes"; return RGBL_E_INVALID;
    }
    const int W = c->cfg.width, H = c->cfg.height;
    const bool on = src_width != 0 && (src_width != W || src_height != H);
    if (on && (src_width < W || src_height < H)) {
        c->err = "the input resize only downscales (input size >= the context's size in both axes)"; return RGBL_E_UNSUPPORTED;
    }
    if (on && (src_width > 32767 || src_height > 32767)) { c->err = "input sizes above 32767 px are not supported"; return RGBL_E_UNSUPPORTED; }
    if (on) {
        CU(cudaSetDevice(c->cfg.device));
        std::vector<LinCoef> tab((size_t)W + H);
        linear_coefs(src_width, W, tab.data());
        linear_coefs(src_height, H, tab.data() + W);
        if (!ensure(c->d_resize_coefs, tab.size())) { c->err = "device allocation failed (input resize tables)"; return RGBL_E_CUDA; }
        if (!c->ev_rsd_b) CU(c->ev_rsd_b.create());
        if (!c->ev_rsd_e) CU(c->ev_rsd_e.create());
        CU(cudaStreamSynchronize(c->st));         // a batch in flight may still read the previous tables
        CU(cudaMemcpy(c->d_resize_coefs, tab.data(), tab.size() * sizeof(LinCoef), cudaMemcpyHostToDevice));
    }
    c->input.resize = on; c->input.w = on ? src_width : W; c->input.h = on ? src_height : H;
    input_changed(c);
    return RGBL_OK;
}

// Tracking::GrabImageRGBL / GrabImageRGBD / GrabImageStereo's cvtColor of 3- and 4-channel camera images (src/Tracking.cc:1518 ff., 1567-1580).
// Every check runs before anything is changed, so a refused setting leaves the previous one in place.
int rgbl_set_input_channels(rgbl_ctx* ctx, int channels, int camera_rgb) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if ((channels != 1 && channels != 3 && channels != 4) || (camera_rgb != 0 && camera_rgb != 1)) {
        c->err = "channels must be 1, 3 or 4 and camera_rgb 0 or 1"; return RGBL_E_INVALID;
    }
    c->input.ch = channels; c->input.w0 = camera_rgb ? 9798 : 3735;      // mbRGB: COLOR_RGB2GRAY weights channel 0 as red, COLOR_BGR2GRAY as blue
    input_changed(c);
    return RGBL_OK;
}

int rgbl_resident_download(rgbl_ctx* ctx, rgbl_keypoint* kps, uint8_t* desc, float* depth, float* uright, int cap, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!kps || !desc || !depth || !uright || !n_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (c->last_frames < 1) { c->err = "nothing processed"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    return download_rgbl(c, c->last_frames, kps, desc, depth, uright, cap, n_out);
}

// ---- camera model of Frame::UndistortKeyPoints / Frame::ComputeImageBounds (src/Frame.cc:837-899) ----
int rgbl_set_camera_distortion(rgbl_ctx* ctx, float fx, float fy, float cx, float cy, const float* dist, int n_dist, float bounds_out[4]) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!dist) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (n_dist != 4 && n_dist != 5) { c->err = "the distortion has 4 or 5 coefficients (k1, k2, p1, p2[, k3])"; return RGBL_E_INVALID; }
    bool finite = std::isfinite(fx) && std::isfinite(fy) && std::isfinite(cx) && std::isfinite(cy);
    for (int i = 0; i < n_dist; ++i) finite = finite && std::isfinite(dist[i]);
    if (!finite || !(fx > 0.f) || !(fy > 0.f)) { c->err = "the camera needs finite values and fx, fy > 0"; return RGBL_E_INVALID; }
    if (const int rc = require_idle(c)) return rc;
    const UndistortDev m = make_undistort_dev(fx, fy, cx, cy, dist, n_dist);
    float b[4];
    image_bounds(m, dist[0], c->cfg.width, c->cfg.height, b);      // once per setting, with the kernel's arithmetic
    c->undistort = dist[0] != 0.f;           // mDistCoef.at<float>(0) == 0: mvKeysUn = mvKeys, even if k2, p1, p2 or k3 are not
    c->cam_un = m;
    std::memcpy(c->cam_bounds, b, sizeof(b));
    if (bounds_out) std::memcpy(bounds_out, b, sizeof(b));
    return RGBL_OK;
}

int rgbl_resident_download_keys_un(rgbl_ctx* ctx, rgbl_keypoint* kps_un, int cap, int* n_out) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!kps_un || !n_out) { c->err = "null argument"; return RGBL_E_INVALID; }
    if (c->last_frames < 1) { c->err = "nothing processed"; return RGBL_E_INVALID; }
    CU(cudaSetDevice(c->cfg.device));
    { int rc = fetch_counts(c, c->last_frames); if (rc) return rc; }
    const rgbl_keypoint* src = c->frames_undistorted ? c->d_kps_un : c->d_kps;
    for (int f = 0; f < c->last_frames; ++f) {
        const int n = c->h_n_sel[f];
        n_out[f] = n;
        if (n > cap) { c->err = "output capacity too small"; return RGBL_E_CAPACITY; }
        if (n) CU(cudaMemcpyAsync(kps_un + (size_t)f * cap, src + (size_t)f * c->cap_kp, (size_t)n * sizeof(rgbl_keypoint), cudaMemcpyDeviceToHost, c->st));
    }
    CU(cudaStreamSynchronize(c->st));
    return RGBL_OK;
}

int rgbl_set_host_quadtree(rgbl_ctx* ctx, int on) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (!on && !c->qt_device_ok) {       // the same test rgbl_create made: node capacity, root count and shared memory of every level
        c->err = "this context's level geometry does not fit the device quad-tree (quota + 3 <= 1024, 1 <= nIni <= 64 per level)"; return RGBL_E_UNSUPPORTED;
    }
    c->device_quadtree = !on;
    return RGBL_OK;
}

/* ---- device-side stopwatch on the context's main stream ---- */
int rgbl_timer_mark(rgbl_ctx* ctx, int which) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || (which != 0 && which != 1)) return RGBL_E_INVALID;
    CU(cudaSetDevice(c->cfg.device));
    CU(cudaEventRecord(which == 0 ? c->ev_t0 : c->ev_t1, c->st));
    return RGBL_OK;
}
int rgbl_timer_elapsed_ms(rgbl_ctx* ctx, double* ms) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c || !ms) return RGBL_E_INVALID;
    CU(cudaSetDevice(c->cfg.device));
    CU(cudaEventSynchronize(c->ev_t1));
    float f = 0.f;
    CU(cudaEventElapsedTime(&f, c->ev_t0, c->ev_t1));
    *ms = f;
    return RGBL_OK;
}

/* ---- profiling ---- */
int rgbl_profile_enable(rgbl_ctx* ctx, int on) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    c->prof_on = on != 0;
    c->prof_serial = on == 2;
    return RGBL_OK;
}
int rgbl_profile_reset(rgbl_ctx* ctx) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    for (int i = 0; i < kNumStages; ++i) { c->st_ms[i] = 0; c->st_launches[i] = 0; c->st_calls[i] = 0; }
    c->host_quadtree_ms = 0; c->total_launches = 0;
    return RGBL_OK;
}
int rgbl_profile_num_stages(void) { return kNumStages; }
const char* rgbl_profile_stage_name(int stage) { return (stage >= 0 && stage < kNumStages) ? kStageNames[stage] : ""; }
int rgbl_profile_read(const rgbl_ctx* ctx, int stage, double* total_ms, int64_t* kernel_launches, int64_t* calls) {
    const Ctx* c = reinterpret_cast<const Ctx*>(ctx);
    if (!c || stage < 0 || stage >= kNumStages) return RGBL_E_INVALID;
    if (total_ms) *total_ms = c->st_ms[stage];
    if (kernel_launches) *kernel_launches = c->st_launches[stage];
    if (calls) *calls = c->st_calls[stage];
    return RGBL_OK;
}
int rgbl_profile_totals(const rgbl_ctx* ctx, int64_t* kernel_launches, double* host_quadtree_ms) {
    const Ctx* c = reinterpret_cast<const Ctx*>(ctx);
    if (!c) return RGBL_E_INVALID;
    if (kernel_launches) *kernel_launches = c->total_launches;
    if (host_quadtree_ms) *host_quadtree_ms = c->host_quadtree_ms;
    return RGBL_OK;
}

}  // extern "C"
