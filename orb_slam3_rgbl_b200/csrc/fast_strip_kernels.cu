// FAST kernel (strip formulation, fast_strip.cuh): kernel wrapper, launcher, host twin and its test hook.  The host twin is checked
// against the oracle on the CPU (tests/test_host_abi.py), the device path on the CUDA-on-CPU shim and on the GPU.
#include <cstring>
#include <string>
#include <vector>

#include "fast_strip.cuh"
#include "rgbl_kernels.h"
#ifdef RGBL_TESTING_EXPORTS
#include "rgbl_testing.h"
#endif

namespace rgbl {

// dynamic shared memory: tile | score map | survivor list (+ score-word list from its end) | counts | misc
static size_t strip_smem_bytes(int rows_cap, int list_cap) {
    return 2 * (size_t)rows_cap * fs::kPitch + (((size_t)list_cap * 2 + 15) & ~(size_t)15) + (size_t)(fs::kCntInts + fs::kMiscInts) * sizeof(int);
}

__global__ void __launch_bounds__(256) fast_strips_kernel(const uint8_t* __restrict__ pyr, size_t frame_stride,
                                                          const LevelGeom* __restrict__ levels, const CellInfo* __restrict__ cells,
                                                          int n_cells, const StripInfo* __restrict__ strips, int ini_th, int min_th,
                                                          uint32_t* __restrict__ slots, int* __restrict__ counts,
                                                          int* __restrict__ overflow, int rows_cap, int list_cap) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* tile = smem;
    uint8_t* sc = tile + (size_t)rows_cap * fs::kPitch;
    uint16_t* list = reinterpret_cast<uint16_t*>(sc + (size_t)rows_cap * fs::kPitch);
    int* cnt = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(list) + (((size_t)list_cap * 2 + 15) & ~(size_t)15));
    int* misc = cnt + fs::kCntInts;
    const StripInfo si = strips[blockIdx.x];
    const LevelGeom lg = levels[si.level];
    const int frame = blockIdx.y;
    fs::run(pyr + (size_t)frame * frame_stride + lg.off, lg.pitch, si, cells, lg.min_bx, lg.min_by, ini_th, min_th, tile, sc, list, list_cap, cnt,
            misc, slots + (size_t)frame * n_cells * kCellCap, counts + (size_t)frame * n_cells, overflow);
}

int launch_fast_strips(cudaStream_t st, const uint8_t* pyr, size_t frame_stride, const LevelGeom* d_levels, const CellInfo* d_cells,
                       int n_cells, const StripInfo* d_strips, int n_strips, int rows_cap, int list_cap, int ini_th, int min_th,
                       uint32_t* slots, int* counts, int* overflow, int n_frames) {
    const size_t bytes = strip_smem_bytes(rows_cap, list_cap);
    if (cudaFuncSetAttribute(fast_strips_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) return -1;
    fast_strips_kernel<<<dim3(n_strips, n_frames), 256, bytes, st>>>(pyr, frame_stride, d_levels, d_cells, n_cells, d_strips, ini_th,
                                                                     min_th, slots, counts, overflow, rows_cap, list_cap);
    return 0;
}

// Host execution of the same strip body (phase-sequential) on one level image.
void fast_strips_host(const uint8_t* level_img, int pitch, const LevelGeom& lg, const std::vector<CellInfo>& cells,
                      const std::vector<StripInfo>& strips, int rows_cap, int list_cap, int ini_th, int min_th, uint32_t* slots,
                      int* counts, int* overflow) {
    std::vector<uint32_t> tile((size_t)rows_cap * fs::kPitch / 4 + 4), sc((size_t)rows_cap * fs::kPitch / 4 + 4);
    std::vector<uint16_t> list((size_t)list_cap + 4);
    std::vector<int> cnt(fs::kCntInts), misc(fs::kMiscInts);
    for (const StripInfo& si : strips) {
        if (si.level != cells[lg.cell_base].level) continue;
        // stale contents on purpose: the device tile is not cleared between CTAs either
        fs::run(level_img, pitch, si, cells.data(), lg.min_bx, lg.min_by, ini_th, min_th, reinterpret_cast<uint8_t*>(tile.data()),
                reinterpret_cast<uint8_t*>(sc.data()), list.data(), list_cap, cnt.data(), misc.data(), slots, counts, overflow);
    }
}

}  // namespace rgbl

#ifdef RGBL_TESTING_EXPORTS        // test hooks: only in librgbl_b200_testing.so (csrc/rgbl_testing.h)
extern "C" {

// test hook: strip FAST of pyramid level `level` of a width x height image, run on the host.  level_img: that level's pixels
// (levels[level].w x .h, row stride `stride`).  out_xys: n x 3 (x, y, score relative to the FAST window origin) in the
// reference's order (cells row-major, cv::FAST order inside a cell); returns n, or a negative rgbl_status.
int rgbl_fast_strips_emulation(const rgbl_orb_params* orb, int width, int height, int level, const uint8_t* level_img, int stride,
                               int max_cells, int max_width, int32_t* out_xys, int cap) {
    using namespace rgbl;
    if (!orb || !level_img || !out_xys || level < 0) return RGBL_E_INVALID;
    OrbTables tab;
    int rc = compute_orb_tables(*orb, tab);
    if (rc) return rc;
    if (level >= tab.nlevels) return RGBL_E_INVALID;
    std::vector<LevelGeom> levels; std::vector<CellInfo> cells; std::vector<LinCoef> coefs; size_t fb = 0; std::string err;
    rc = build_geometry(width, height, tab, levels, cells, coefs, fb, err);
    if (rc) return rc;
    if (max_cells < 1 || max_cells > fs::kMaxCells || max_width < 78 || max_width > fs::kMaxWidth) return RGBL_E_INVALID;
    std::vector<StripInfo> strips; int rows_cap = 0, list_cap = 0;
    build_fast_strips(cells, max_cells, max_width, strips, rows_cap, list_cap);
    const LevelGeom& lg = levels[level];
    // padded copy with the device pitch so that the aligned word loads of the last strip stay inside the row
    std::vector<uint8_t> img((size_t)lg.pitch * lg.h + 64, 0);
    for (int y = 0; y < lg.h; ++y) std::memcpy(&img[(size_t)y * lg.pitch], level_img + (size_t)y * stride, lg.w);
    std::vector<uint32_t> slots(cells.size() * kCellCap);
    std::vector<int> counts(cells.size(), 0);
    int overflow = 0;
    fast_strips_host(img.data(), lg.pitch, lg, cells, strips, rows_cap, list_cap, orb->ini_th_fast, orb->min_th_fast, slots.data(),
                     counts.data(), &overflow);
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

}  // extern "C"
#endif  // RGBL_TESTING_EXPORTS
