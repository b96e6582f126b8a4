// Internal declarations shared by the host side and the CUDA translation units of librgbl_b200.so.
#ifndef RGBL_INTERNAL_H
#define RGBL_INTERNAL_H

#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/rgbl_b200.h"

namespace rgbl {

constexpr int kEdgeThreshold = 19;   // src/ORBextractor.cc:73
constexpr int kHalfPatch = 15;       // src/ORBextractor.cc:72
constexpr int kPatchSize = 31;       // src/ORBextractor.cc:71
constexpr int kFastBorder = 16;      // EDGE_THRESHOLD - 3, src/ORBextractor.cc:789
constexpr int kCellTarget = 35;      // W, src/ORBextractor.cc:785
constexpr int kCellCap = 256;        // staged FAST survivors per cell (overflow is reported, never dropped)
constexpr int kGridCols = 64, kGridRows = 48;   // FRAME_GRID_COLS / FRAME_GRID_ROWS, include/Frame.h:46-47

// Geometry of one pyramid level (identical for every frame of a context).
struct LevelGeom {
    int w, h, pitch;           // level size and row pitch in bytes (pitch % 64 == 0)
    int off;                   // byte offset of the level inside one frame's pyramid block
    int min_bx, min_by, max_bx, max_by;   // FAST window, src/ORBextractor.cc:789-792
    int n_cols, n_rows, w_cell, h_cell;   // :797-803
    int cell_base, n_cells;    // first index / count in the flat cell table
    int quota;                 // mnFeaturesPerLevel
    int tabx_off, taby_off;    // offsets of this level's resize coefficient tables (level >= 1)
    float scale, inv_scale;    // mvScaleFactor / mvInvScaleFactor
    int scaled_patch;          // (int)(PATCH_SIZE * scale), :880
};

// One FAST cell window (src/ORBextractor.cc:805-822).
struct CellInfo {
    int16_t level;
    int16_t x0, y0;            // window origin in level coordinates
    int16_t cw, ch;            // window size
    int16_t off_x, off_y;      // j*wCell, i*hCell: added to the FAST keypoint (:863-868)
    int16_t pad;
};

// A run of consecutive FAST cells of one cell row, handled by one CTA of the strip kernel (fast_strip.cuh).
struct StripInfo {
    int32_t first_cell;        // index into the flat cell table
    int16_t level, n_cells;
    int16_t x0, y0, w, h;      // union of the cells' windows (level coordinates)
};

// Bilinear resize coefficient (SURVEY A.1): source index and the two 11-bit weights.
struct LinCoef {
    int16_t s;                 // left/top source index
    int16_t c0, c1;            // weights (sum 2048)
    int16_t pad;
};

// Pinhole camera + distortion of Frame::UndistortKeyPoints as cvUndistortPointsInternal holds them: K (float) and mDistCoef converted to
// double, ifx = 1. / fx, ify = 1. / fy; k = OpenCV's 12 distortion coefficients (k1, k2, p1, p2, k3, then zeros for a 4- or 5-element mDistCoef).
struct UndistortDev {
    double fx, fy, cx, cy, ifx, ify;
    double k[12];
};

struct OrbTables {
    int nlevels;
    float scale[RGBL_MAX_LEVELS], inv_scale[RGBL_MAX_LEVELS];
    float sigma2[RGBL_MAX_LEVELS], inv_sigma2[RGBL_MAX_LEVELS];
    int quota[RGBL_MAX_LEVELS];
    int umax[kHalfPatch + 1];
};

// host-only
int compute_orb_tables(const rgbl_orb_params& p, OrbTables& t);
int build_geometry(int width, int height, const OrbTables& t, std::vector<LevelGeom>& levels,
                   std::vector<CellInfo>& cells, std::vector<LinCoef>& coefs, size_t& frame_bytes, std::string& err);
// cv::resize INTER_LINEAR coefficients of one axis, src_n -> dst_n samples (SURVEY A.1): the pyramid's level tables and the input resize's
void linear_coefs(int src_n, int dst_n, LinCoef* out);
// cells -> strips of at most max_cells cells and max_width px; returns the largest window height and tested-pixel count
void build_fast_strips(const std::vector<CellInfo>& cells, int max_cells, int max_width, std::vector<StripInfo>& strips, int& rows_max,
                       int& tested_max);
int quadtree_select(const int32_t* xys, int n, int min_x, int max_x, int min_y, int max_y, int n_desired,
                    int32_t* out_idx, int cap);
int structuring_element(const char* kind, int ku, int kv, uint8_t* mask);

// Packed FAST candidate: x | y << 12 | score << 24 (x, y relative to the FAST window origin (16,16)).
inline uint32_t pack_cand(int x, int y, int s) { return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)s << 24); }

}  // namespace rgbl

#endif
