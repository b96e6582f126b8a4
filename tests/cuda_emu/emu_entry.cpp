// TEST INFRASTRUCTURE: C entry points that run the library's kernels (device code paths) on the CUDA-on-CPU shim.
// The marshalling mirrors the host-twin hooks of the product library; the difference is that these go through the real
// launchers (launch_fast_strips, launch_describe_staged, launch_quadtree) and therefore through the kernels' device branches.
// A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu.py calls it.
#include <cstring>
#include <string>
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_internal.h"
#include "rgbl_kernels.h"

using namespace rgbl;

extern "C" {

int emu_fast_strips(const rgbl_orb_params* orb, int width, int height, int level, const uint8_t* level_img, int stride, int max_cells,
                    int max_width, int32_t* out_xys, int cap) {
    OrbTables tab;
    int rc = compute_orb_tables(*orb, tab);
    if (rc) return rc;
    std::vector<LevelGeom> levels; std::vector<CellInfo> cells; std::vector<LinCoef> coefs; size_t fb = 0; std::string err;
    rc = build_geometry(width, height, tab, levels, cells, coefs, fb, err);
    if (rc) return rc;
    std::vector<StripInfo> strips; int rows_cap = 0, list_cap = 0;
    build_fast_strips(cells, max_cells, max_width, strips, rows_cap, list_cap);
    const LevelGeom& lg = levels[level];
    std::vector<uint8_t> pyr(fb + 256, 0);
    for (int y = 0; y < lg.h; ++y) std::memcpy(&pyr[lg.off + (size_t)y * lg.pitch], level_img + (size_t)y * stride, lg.w);
    int first = -1, count = 0;
    for (size_t i = 0; i < strips.size(); ++i) if (strips[i].level == level) { if (first < 0) first = (int)i; ++count; }
    std::vector<uint32_t> slots(cells.size() * kCellCap);
    std::vector<int> counts(cells.size(), 0);
    int overflow = 0;
    if (launch_fast_strips(nullptr, pyr.data(), fb, levels.data(), cells.data(), (int)cells.size(), strips.data() + first, count, rows_cap,
                           list_cap, orb->ini_th_fast, orb->min_th_fast, slots.data(), counts.data(), &overflow, 1) != 0) return -100;
    if (overflow) return RGBL_E_CAPACITY;
    int n = 0;
    for (int c = lg.cell_base; c < lg.cell_base + lg.n_cells; ++c)
        for (int k = 0; k < counts[c]; ++k) {
            if (n >= cap) return RGBL_E_CAPACITY;
            const uint32_t p = slots[(size_t)c * kCellCap + k];
            out_xys[3 * n] = (int)(p & 0xfff); out_xys[3 * n + 1] = (int)((p >> 12) & 0xfff); out_xys[3 * n + 2] = (int)(p >> 24);
            ++n;
        }
    return n;
}

int emu_describe_staged(const rgbl_orb_params* orb, const uint8_t* level_img, const uint8_t* blurred_img, int w, int h, int stride, int n,
                        const int32_t* xy, float* angle_out, uint8_t* desc_out) {
    OrbTables tab;
    const int rc = compute_orb_tables(*orb, tab);
    if (rc) return rc;
    LevelGeom lg{};
    lg.w = w; lg.h = h; lg.pitch = (w + 63) & ~63; lg.off = 0; lg.scale = 1.f; lg.inv_scale = 1.f; lg.scaled_patch = kPatchSize;
    const size_t fb = (size_t)lg.pitch * h;
    std::vector<uint8_t> a(fb + 64, 0), b(fb + 64, 0);
    for (int y = 0; y < h; ++y) { std::memcpy(&a[(size_t)y * lg.pitch], level_img + (size_t)y * stride, w); std::memcpy(&b[(size_t)y * lg.pitch], blurred_img + (size_t)y * stride, w); }
    std::vector<SelKp> sel(n + 1);
    for (int i = 0; i < n; ++i) { sel[i].x = (uint16_t)xy[2 * i]; sel[i].y = (uint16_t)xy[2 * i + 1]; sel[i].level = 0; sel[i].score = 0; sel[i].pad = 0; }
    std::vector<rgbl_keypoint> kps(n + 1);
    launch_describe_staged(nullptr, a.data(), b.data(), fb, &lg, sel.data(), &n, n, n, tab.umax, kps.data(), desc_out, 1);
    for (int i = 0; i < n; ++i) angle_out[i] = kps[i].angle;
    return 0;
}

// xys: n x 3 candidates (x, y relative to the FAST window origin, score) in the reference's order; out_xys: survivors in level
// coordinates (+16) in the reference's output order.
int emu_quadtree(const int32_t* xys, int n, int w, int h, int n_desired, int32_t* out_xys, int cap) {
    LevelGeom lg{};
    lg.w = w; lg.h = h; lg.min_bx = kFastBorder; lg.min_by = kFastBorder; lg.max_bx = w - kFastBorder; lg.max_by = h - kFastBorder;
    lg.quota = n_desired;
    std::vector<uint32_t> dense(n + 1);
    for (int i = 0; i < n; ++i) dense[i] = pack_cand(xys[3 * i], xys[3 * i + 1], xys[3 * i + 2]);
    int level_cnt[RGBL_MAX_LEVELS] = {n}, frame_total = n, lvl_region[2] = {0, cap}, status = 0, n_sel = 0, n_sel_lvl[RGBL_MAX_LEVELS] = {0};
    std::vector<unsigned short> pa(n + 8), pb(n + 8), na(n + 8), nb(n + 8);
    std::vector<unsigned long long> scan(n + 16);
    std::vector<unsigned char> quad(n + 8);
    QtScratchDev scr{pa.data(), pb.data(), na.data(), nb.data(), scan.data(), quad.data()};
    std::vector<uint32_t> sel_lvl(cap + 8);
    std::vector<SelKp> sel(cap + 8);
    if (launch_quadtree(nullptr, dense.data(), level_cnt, &frame_total, &lg, 1, scr, sel_lvl.data(), n_sel_lvl, lvl_region, cap, &status,
                        sel.data(), &n_sel, 1, n_desired + 3 <= 512 ? 512 : 1024) != 0) return -100;
    if (status) return RGBL_E_CAPACITY;
    for (int i = 0; i < n_sel; ++i) { out_xys[3 * i] = sel[i].x; out_xys[3 * i + 1] = sel[i].y; out_xys[3 * i + 2] = sel[i].score; }
    return n_sel;
}

// ORBextractor::operator() for one image through the device pipeline of api.cu's run_extract (device quad-tree mode):
// pyramid -> FAST -> compaction -> blur -> quad-tree -> describe.
int emu_extract(const rgbl_orb_params* orb, const uint8_t* img, int width, int height, int stride, rgbl_keypoint* kps_out, uint8_t* desc_out,
                int cap) {
    OrbTables tab;
    int rc = compute_orb_tables(*orb, tab);
    if (rc) return rc;
    std::vector<LevelGeom> levels; std::vector<CellInfo> cells; std::vector<LinCoef> coefs; size_t fb = 0; std::string err;
    rc = build_geometry(width, height, tab, levels, cells, coefs, fb, err);
    if (rc) return rc;
    const int nl = tab.nlevels, n_cells = (int)cells.size();
    std::vector<uint8_t> pyr(fb + 256, 0), blur(fb + 256, 0);
    for (int y = 0; y < height; ++y) std::memcpy(&pyr[levels[0].off + (size_t)y * levels[0].pitch], img + (size_t)y * stride, width);
    if (coefs.empty()) coefs.resize(1);
    launch_pyramid(nullptr, pyr.data(), fb, levels.data(), nl, coefs.data(), 1);
    std::vector<uint32_t> slots((size_t)n_cells * kCellCap);
    std::vector<int> counts(n_cells, 0), cell_off(n_cells + 1, 0);
    int level_cnt[RGBL_MAX_LEVELS] = {0}, frame_total = 0, overflow[4] = {0, 0, 0, 0};
    std::vector<StripInfo> strips; int rows_cap = 0, list_cap = 0;
    build_fast_strips(cells, 8, 264, strips, rows_cap, list_cap);
    if (launch_fast_strips(nullptr, pyr.data(), fb, levels.data(), cells.data(), n_cells, strips.data(), (int)strips.size(), rows_cap, list_cap,
                           orb->ini_th_fast, orb->min_th_fast, slots.data(), counts.data(), overflow, 1) != 0) return -100;
    const int dense_cap = std::max(32768, width * height / 8);
    std::vector<uint32_t> dense(dense_cap + 8);
    launch_compact(nullptr, levels.data(), nl, n_cells, slots.data(), counts.data(), cell_off.data(), level_cnt, &frame_total, dense.data(), dense_cap,
                   overflow, 1);
    if (overflow[0]) return RGBL_E_CAPACITY;
    launch_blur(nullptr, pyr.data(), blur.data(), fb, levels.data(), nl, 1);
    std::vector<int> region(nl + 1, 0);
    for (int l = 0; l < nl; ++l) {
        const LevelGeom& g = levels[l];
        const int n_ini = (int)std::round(static_cast<float>(g.max_bx - g.min_bx) / (g.max_by - g.min_by));
        region[l + 1] = region[l] + std::max(g.quota + 3, 4 * n_ini);
    }
    const int cap_kp = region[nl];
    const int n = frame_total;
    std::vector<unsigned short> pa(n + nl + 8), pb(n + nl + 8), na(n + nl + 8), nb(n + nl + 8);
    std::vector<unsigned long long> scan(n + nl + 16);
    std::vector<unsigned char> quad(n + nl + 8);
    QtScratchDev scr{pa.data(), pb.data(), na.data(), nb.data(), scan.data(), quad.data()};
    std::vector<uint32_t> sel_lvl(cap_kp + 8);
    std::vector<SelKp> sel(cap_kp + 8);
    int n_sel_lvl[RGBL_MAX_LEVELS] = {0}, status = 0, n_sel = 0;
    if (launch_quadtree(nullptr, dense.data(), level_cnt, &frame_total, levels.data(), nl, scr, sel_lvl.data(), n_sel_lvl, region.data(), cap_kp,
                        &status, sel.data(), &n_sel, 1) != 0) return -100;
    if (status) return RGBL_E_CAPACITY;
    if (n_sel > cap) return RGBL_E_CAPACITY;
    launch_describe_staged(nullptr, pyr.data(), blur.data(), fb, levels.data(), sel.data(), &n_sel, cap_kp, n_sel, tab.umax, kps_out, desc_out, 1);
    return n_sel;
}

// ProjectPointcloudToImage + Upsample_InverseDilation: depth_project_kernel, then depth_resolve_dilate_v2_kernel.
// pts: 4 x n planar (x | y | z | 1), mask ku x kv, outputs W x H floats.
int emu_depth_dilate(const float* pts, int n, const float P[12], int W, int H, const uint8_t* mask, int ku, int kv, float min_d, float max_d,
                     float inv_scale, float* raw_out, float* processed_out) {
    DepthDev dd{};
    std::memcpy(dd.P, P, 12 * sizeof(float));
    dd.min_dist = min_d; dd.max_dist = max_d; dd.bf = 0; dd.inv_scale_m = max_d * inv_scale; dd.ku = ku; dd.kv = kv;
    std::memcpy(dd.mask, mask, (size_t)ku * kv);
    dd.method = RGBL_DEPTH_INVERSE_DILATION;
    std::vector<uint32_t> idx((size_t)W * H, 0u);
    launch_depth_project(nullptr, pts, 4 * n, &n, n, dd, W, H, idx.data(), 1u, 1);
    launch_depth_resolve_dilate_v2(nullptr, pts, 4 * n, &n, dd, W, H, idx.data(), 1u, raw_out, processed_out, 1);
    return 0;
}

}  // extern "C"
