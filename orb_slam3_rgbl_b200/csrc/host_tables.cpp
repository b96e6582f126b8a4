// Host-side tables and geometry (product code, no GPU needed).
//   compute_orb_tables  <- ORBextractor::ORBextractor, src/ORBextractor.cc:409-469
//   build_geometry      <- level sizes (src/ORBextractor.cc:1174-1175), FAST cell grid (:781-822),
//                          cv::resize INTER_LINEAR coefficient tables (SURVEY A.1)
//   structuring_element <- cv::getStructuringElement / include/DepthModule.h:138-161
#include <algorithm>
#include <cmath>
#include <cstring>
#include <strings.h>

#include "rgbl_internal.h"

namespace rgbl {

static inline int cv_round_f(float v) { return (int)lrintf(v); }

int compute_orb_tables(const rgbl_orb_params& p, OrbTables& t) {
    if (p.nlevels < 1 || p.nlevels > RGBL_MAX_LEVELS || p.nfeatures < 1 || !(p.scale_factor > 1.0f)) return RGBL_E_INVALID;
    t.nlevels = p.nlevels;
    t.scale[0] = 1.0f; t.sigma2[0] = 1.0f;
    for (int i = 1; i < p.nlevels; ++i) {
        t.scale[i] = t.scale[i - 1] * p.scale_factor;
        t.sigma2[i] = t.scale[i] * t.scale[i];
    }
    for (int i = 0; i < p.nlevels; ++i) {
        t.inv_scale[i] = 1.0f / t.scale[i];
        t.inv_sigma2[i] = 1.0f / t.sigma2[i];
    }
    const float factor = 1.0f / p.scale_factor;
    float desired = p.nfeatures * (1 - factor) / (1 - (float)std::pow((double)factor, (double)p.nlevels));
    int sum = 0;
    for (int l = 0; l < p.nlevels - 1; ++l) {
        t.quota[l] = cv_round_f(desired);
        sum += t.quota[l];
        desired *= factor;
    }
    t.quota[p.nlevels - 1] = std::max(p.nfeatures - sum, 0);

    const int vmax = (int)std::floor(kHalfPatch * std::sqrt(2.f) / 2 + 1);
    const int vmin = (int)std::ceil(kHalfPatch * std::sqrt(2.f) / 2);
    const double hp2 = kHalfPatch * kHalfPatch;
    for (int v = 0; v <= kHalfPatch; ++v) t.umax[v] = 0;
    for (int v = 0; v <= vmax; ++v) t.umax[v] = (int)lrint(std::sqrt(hp2 - v * v));
    for (int v = kHalfPatch, v0 = 0; v >= vmin; --v) {
        while (t.umax[v0] == t.umax[v0 + 1]) ++v0;
        t.umax[v] = v0;
        ++v0;
    }
    return RGBL_OK;
}

void linear_coefs(int src_n, int dst_n, LinCoef* out) {
    const double scale = (double)src_n / (double)dst_n;
    for (int d = 0; d < dst_n; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)std::floor(f);
        f -= (float)s;
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= src_n - 1) { s = src_n - 1; f = 0.f; }
        out[d].s = (int16_t)s;
        out[d].c0 = (int16_t)cv_round_f((1.f - f) * 2048.f);
        out[d].c1 = (int16_t)cv_round_f(f * 2048.f);
        out[d].pad = 0;
    }
}

int build_geometry(int width, int height, const OrbTables& t, std::vector<LevelGeom>& levels,
                   std::vector<CellInfo>& cells, std::vector<LinCoef>& coefs, size_t& frame_bytes, std::string& err) {
    levels.clear(); cells.clear(); coefs.clear();
    size_t off = 0;
    for (int l = 0; l < t.nlevels; ++l) {
        LevelGeom g{};
        g.w = cv_round_f((float)width * t.inv_scale[l]);
        g.h = cv_round_f((float)height * t.inv_scale[l]);
        if (g.w > 4095 + 2 * kFastBorder || g.h > 4095 + 2 * kFastBorder) { err = "image larger than 4127 px is not supported"; return RGBL_E_UNSUPPORTED; }
        if (g.w - 2 * kFastBorder < kCellTarget || g.h - 2 * kFastBorder < kCellTarget) { err = "pyramid level too small for the 35 px FAST cell grid"; return RGBL_E_UNSUPPORTED; }
        g.pitch = (g.w + 63) & ~63;
        g.off = (int)off;
        off += (size_t)g.pitch * g.h;
        off = (off + 255) & ~(size_t)255;
        g.min_bx = kFastBorder; g.min_by = kFastBorder;
        g.max_bx = g.w - kFastBorder; g.max_by = g.h - kFastBorder;
        const float wf = (float)(g.max_bx - g.min_bx), hf = (float)(g.max_by - g.min_by);
        g.n_cols = (int)(wf / (float)kCellTarget);
        g.n_rows = (int)(hf / (float)kCellTarget);
        g.w_cell = (int)std::ceil(wf / g.n_cols);
        g.h_cell = (int)std::ceil(hf / g.n_rows);
        g.quota = t.quota[l];
        g.scale = t.scale[l]; g.inv_scale = t.inv_scale[l];
        g.scaled_patch = (int)(kPatchSize * t.scale[l]);
        g.cell_base = (int)cells.size();
        for (int i = 0; i < g.n_rows; ++i) {
            const float iniY = (float)(g.min_by + i * g.h_cell);
            float maxY = iniY + g.h_cell + 6;
            if (iniY >= g.max_by - 3) continue;
            if (maxY > g.max_by) maxY = (float)g.max_by;
            for (int j = 0; j < g.n_cols; ++j) {
                const float iniX = (float)(g.min_bx + j * g.w_cell);
                float maxX = iniX + g.w_cell + 6;
                if (iniX >= g.max_bx - 6) continue;
                if (maxX > g.max_bx) maxX = (float)g.max_bx;
                CellInfo c{};
                c.level = (int16_t)l;
                c.x0 = (int16_t)iniX; c.y0 = (int16_t)iniY;
                c.cw = (int16_t)((int)maxX - (int)iniX); c.ch = (int16_t)((int)maxY - (int)iniY);
                c.off_x = (int16_t)(j * g.w_cell); c.off_y = (int16_t)(i * g.h_cell);
                if (c.cw > 78 || c.ch > 78) { err = "FAST cell window exceeds the shared-memory tile"; return RGBL_E_UNSUPPORTED; }
                cells.push_back(c);
            }
        }
        g.n_cells = (int)cells.size() - g.cell_base;
        if (l >= 1) {
            g.tabx_off = (int)coefs.size();
            coefs.resize(coefs.size() + g.w);
            linear_coefs(levels[l - 1].w, g.w, &coefs[g.tabx_off]);
            g.taby_off = (int)coefs.size();
            coefs.resize(coefs.size() + g.h);
            linear_coefs(levels[l - 1].h, g.h, &coefs[g.taby_off]);
        }
        levels.push_back(g);
    }
    frame_bytes = off;
    return RGBL_OK;
}

void build_fast_strips(const std::vector<CellInfo>& cells, int max_cells, int max_width, std::vector<StripInfo>& strips, int& rows_max,
                       int& tested_max) {
    strips.clear(); rows_max = 0; tested_max = 0;
    size_t i = 0;
    while (i < cells.size()) {
        const CellInfo& f = cells[i];
        StripInfo s{};
        s.first_cell = (int32_t)i; s.level = f.level; s.x0 = f.x0; s.y0 = f.y0; s.h = f.ch;
        size_t j = i;
        // cells of one row are consecutive in the table, share y0 / ch and their windows advance by wCell
        while (j < cells.size() && (int)(j - i) < max_cells && cells[j].level == f.level && cells[j].y0 == f.y0 && cells[j].ch == f.ch &&
               cells[j].x0 + cells[j].cw - f.x0 <= max_width)
            ++j;
        if (j == i) j = i + 1;                       // a single cell wider than max_width cannot happen (cw <= 78)
        s.n_cells = (int16_t)(j - i);
        s.w = (int16_t)(cells[j - 1].x0 + cells[j - 1].cw - f.x0);
        strips.push_back(s);
        rows_max = std::max(rows_max, (int)s.h);
        if (s.w > 6 && s.h > 6) tested_max = std::max(tested_max, (s.w - 6) * (s.h - 6));
        i = j;
    }
}

int structuring_element(const char* kind, int ku, int kv, uint8_t* mask) {
    if (!kind || !mask || ku < 1 || kv < 1 || ku > 9 || kv > 9) return RGBL_E_INVALID;
    std::memset(mask, 0, (size_t)ku * kv);
    if (!strcasecmp(kind, "Rectangle")) {
        std::memset(mask, 1, (size_t)ku * kv);
    } else if (!strcasecmp(kind, "Cross")) {
        for (int i = 0; i < ku; ++i) mask[(kv / 2) * ku + i] = 1;
        for (int j = 0; j < kv; ++j) mask[j * ku + ku / 2] = 1;
    } else if (!strcasecmp(kind, "Ellipse")) {
        const int r = kv / 2, c = ku / 2;
        const double inv_r2 = r ? 1.0 / ((double)r * r) : 0.0;
        for (int i = 0; i < kv; ++i) {
            const int dy = i - r;
            if (std::abs(dy) > r) continue;
            const int dx = (int)lrint(c * std::sqrt((r * r - dy * dy) * inv_r2));
            for (int j = std::max(c - dx, 0); j < std::min(c + dx + 1, ku); ++j) mask[i * ku + j] = 1;
        }
    } else if (!strcasecmp(kind, "Diamond")) {
        // only KernelSize_u is considered and only 3/5/7/9 exist (src/DepthModule.cc:241-253)
        if (ku != 3 && ku != 5 && ku != 7 && ku != 9) return RGBL_E_INVALID;
        if (kv != ku) return RGBL_E_INVALID;
        const int r = ku / 2;
        for (int j = 0; j < ku; ++j)
            for (int i = 0; i < ku; ++i) mask[j * ku + i] = (std::abs(i - r) + std::abs(j - r) <= r) ? 1 : 0;
    } else {
        return RGBL_E_INVALID;
    }
    return RGBL_OK;
}

}  // namespace rgbl

extern "C" {

int rgbl_abi_version(void) { return 5; }

int rgbl_orb_tables(const rgbl_orb_params* p, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                    int32_t* features_per_level, int32_t* umax16) {
    if (!p) return RGBL_E_INVALID;
    rgbl::OrbTables t;
    int rc = rgbl::compute_orb_tables(*p, t);
    if (rc) return rc;
    for (int l = 0; l < t.nlevels; ++l) {
        if (scale) scale[l] = t.scale[l];
        if (inv_scale) inv_scale[l] = t.inv_scale[l];
        if (sigma2) sigma2[l] = t.sigma2[l];
        if (inv_sigma2) inv_sigma2[l] = t.inv_sigma2[l];
        if (features_per_level) features_per_level[l] = t.quota[l];
    }
    if (umax16) for (int v = 0; v <= rgbl::kHalfPatch; ++v) umax16[v] = t.umax[v];
    return RGBL_OK;
}

int rgbl_depth_structuring_element(const char* kind, int ku, int kv, uint8_t* mask) {
    return rgbl::structuring_element(kind, ku, kv, mask);
}

int rgbl_descriptor_distance(const uint8_t a[32], const uint8_t b[32]) {
    int d = 0;
    for (int i = 0; i < 4; ++i) {
        uint64_t x, y;
        std::memcpy(&x, a + 8 * i, 8);
        std::memcpy(&y, b + 8 * i, 8);
        d += __builtin_popcountll(x ^ y);
    }
    return d;
}

#ifdef RGBL_TESTING_EXPORTS        // test hook: only in librgbl_b200_testing.so (csrc/rgbl_testing.h)
int rgbl_quadtree_select(const int32_t* xys, int n, int min_x, int max_x, int min_y, int max_y, int n_desired,
                         int32_t* out_idx, int cap) {
    if (n < 0 || (n > 0 && !xys) || !out_idx || max_x <= min_x || max_y <= min_y) return RGBL_E_INVALID;
    return rgbl::quadtree_select(xys, n, min_x, max_x, min_y, max_y, n_desired, out_idx, cap);
}
#endif

}  // extern "C"
