/* TEST INFRASTRUCTURE, not part of the product ABI: host twins of device algorithms, exported only by librgbl_b200_testing.so (built from
 * the same sources with -DRGBL_TESTING_EXPORTS; include/rgbl_b200.h and librgbl_b200.so do not carry these symbols).  The CPU tests
 * (tests/test_host_abi.py) use them to check the device algorithms' logic against the oracle without a GPU.                     */
#ifndef RGBL_TESTING_H
#define RGBL_TESTING_H
#include "../../include/rgbl_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- host-only pieces exported for tests (no GPU needed) ---- */
/* DistributeOctTree (src/ORBextractor.cc:555-779) on candidates given relative to (minX,minY).
 * xys: n x 3 int32 (x, y, score) in reference order.  out_idx: indices into the input, in the
 * reference's output order.  Returns the number selected (<= N + 3).                             */
int rgbl_quadtree_select(const int32_t* xys, int n, int min_x, int max_x, int min_y, int max_y, int n_desired,
                         int32_t* out_idx, int cap);

/* Test hooks (host-only): the device quad-tree's block algorithm executed phase-sequentially on the host (budget |n_desired|), and
 * the restated libstdc++ std::sort it falls back to.  out_xys: n x 3 survivors in the reference's output order.              */
int rgbl_quadtree_select_block_emulation(const int32_t* xys, int n, int min_x, int max_x, int min_y, int max_y, int n_desired,
                                         int32_t* out_xys, int cap);
int rgbl_std_sort_emulation(const int32_t* size_ulx, int n, int32_t* perm_out);
/* The block-parallel formulation of that sort (mode 0; mode > 0: depth limit mode - 1, which forces the heapsort fallback) or,
 * as ground truth, the C++ library's own std::sort with the reference's comparator (mode < 0).  n <= 1024.                */
int rgbl_std_sort_block_emulation(const int32_t* size_ulx, int n, int mode, int32_t* perm_out);

/* Test hook (host-only): the strip formulation of the per-cell FAST detection (fast_strip.cuh; src/ORBextractor.cc:805-868)
 * executed phase-sequentially on the host for pyramid level `level` of a width x height image.  level_img: that level's
 * pixels (row stride `stride`); strips hold at most max_cells (1..8) cells / max_width (78..264) px.  out_xys: n x 3
 * (x, y relative to the FAST window origin (16, 16), cv score) in the reference's order.  Returns n or a negative status. */
int rgbl_fast_strips_emulation(const rgbl_orb_params* orb, int width, int height, int level, const uint8_t* level_img, int stride,
                               int max_cells, int max_width, int32_t* out_xys, int cap);

/* Test hook (host-only): orientation (degrees) and 32-byte rBRIEF descriptor of n keypoints (xy: n x 2 level coordinates, at
 * least 19 px from the border) of one pyramid level and its blurred copy, computed by the host twin of the staged describe
 * kernel (describe_warp.cuh; IC_Angle src/ORBextractor.cc:76-103, computeOrbDescriptor :107-146).                          */
int rgbl_describe_staged_emulation(const rgbl_orb_params* orb, const uint8_t* level_img, const uint8_t* blurred_img, int w, int h,
                                   int stride, int n, const int32_t* xy, float* angle_out, uint8_t* desc_out);

#ifdef __cplusplus
}
#endif
#endif /* RGBL_TESTING_H */
