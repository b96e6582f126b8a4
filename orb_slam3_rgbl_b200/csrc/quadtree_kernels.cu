// Device quad-tree distribution (one CTA per (frame, level)) + packing of the per-level survivor lists into the
// per-frame SelKp list the describe kernel consumes.  Algorithm: quadtree_block.cuh.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "quadtree_block.cuh"
#include "rgbl_kernels.h"
#ifdef RGBL_TESTING_EXPORTS
#include "rgbl_testing.h"
#endif

namespace rgbl {

template <int MAXN>
__global__ void __launch_bounds__(512, MAXN <= 512 ? 2 : 1) quadtree_kernel(const uint32_t* __restrict__ dense, const int* __restrict__ level_cnt,
                                                       const int* __restrict__ frame_total, const LevelGeom* __restrict__ levels,
                                                       int n_levels, QtScratchDev scr, uint32_t* __restrict__ sel_lvl,
                                                       int* __restrict__ n_sel_lvl, const int* __restrict__ lvl_region,
                                                       int cap_kp, int* __restrict__ status, int dyn_bytes) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    typedef qt::SharedT<MAXN> SharedX;
    SharedX& s = *reinterpret_cast<SharedX*>(smem_raw);
    // level-major block order: with one CTA per SM (the key arrays take the whole shared memory) a batch is more than one wave, and a
    // level's run time grows with its candidate count - the long level-0 trees start first, the short ones fill the tail
    const int l = blockIdx.y, f = blockIdx.x;
    int off = 0;
    for (int k = 0; k < f; ++k) off += frame_total[k];
    for (int k = 0; k < l; ++k) off += level_cnt[f * RGBL_MAX_LEVELS + k];
    const int n = level_cnt[f * RGBL_MAX_LEVELS + l];
    const LevelGeom lg = levels[l];
    qt::Scratch g;
    const int so = off + (f * n_levels + l);          // one extra scan slot per preceding tree
    // The per-key arrays (two permutations, two node maps as 16-bit indices, packed scan counters, quadrants: 17 bytes per key) are walked by
    // every subdivision pass with a dozen barrier-separated phases; in global memory each phase pays an L2 round trip.  They
    // live in the rest of the CTA's shared memory whenever the level's candidates fit (falls back to the global scratch).
    const size_t key_bytes = (size_t)(n + 1) * 8 + (size_t)(n + 1) * (4 * 2 + 1) + 64;
    if (sizeof(SharedX) + key_bytes <= (size_t)dyn_bytes) {
        unsigned char* base = smem_raw + ((sizeof(SharedX) + 15) & ~(size_t)15);
        g.scan = reinterpret_cast<unsigned long long*>(base); base += (size_t)(n + 1) * 8;
        const size_t kb = ((size_t)n * sizeof(qt::KeyIdx) + 7) & ~(size_t)7;
        g.perm_a = reinterpret_cast<qt::KeyIdx*>(base); base += kb;
        g.perm_b = reinterpret_cast<qt::KeyIdx*>(base); base += kb;
        g.node_a = reinterpret_cast<qt::KeyIdx*>(base); base += kb;
        g.node_b = reinterpret_cast<qt::KeyIdx*>(base); base += kb;
        g.quad = base;
    } else {
        g.perm_a = scr.perm_a + off; g.perm_b = scr.perm_b + off; g.node_a = scr.node_a + off; g.node_b = scr.node_b + off;
        g.scan = scr.scan + so; g.quad = scr.quad + off;
    }
    uint32_t* out = sel_lvl + (size_t)f * cap_kp + lvl_region[l];
    const int region_cap = lvl_region[l + 1] - lvl_region[l];
#ifdef QT_TIMING
    const long long qt_t0 = clock64();
#endif
    const int m = qt::distribute(s, dense + off, n, lg.max_bx - lg.min_bx, lg.max_by - lg.min_by, lg.quota, g, out, region_cap);
#ifdef QT_TIMING
    if (threadIdx.x == 0 && f == 0) printf("quadtree level %d: n=%d quota=%d selected=%d keys_on_chip=%d cycles=%lld\n", l, n, lg.quota, m, (int)(sizeof(SharedX) + key_bytes <= (size_t)dyn_bytes), clock64() - qt_t0);
#endif
    if (threadIdx.x == 0) {
        if (m < 0 || m > region_cap) { atomicExch(status, 1); n_sel_lvl[f * RGBL_MAX_LEVELS + l] = 0; }
        else n_sel_lvl[f * RGBL_MAX_LEVELS + l] = m;
    }
}

// per frame: concatenate the level regions -> SelKp list (+16 offset applied) and n_sel
__global__ void __launch_bounds__(256) sel_pack_kernel(const uint32_t* __restrict__ sel_lvl, const int* __restrict__ n_sel_lvl,
                                                       const int* __restrict__ lvl_region, int n_levels, int cap_kp,
                                                       SelKp* __restrict__ sel, int* __restrict__ n_sel) {
    const int f = blockIdx.x;
    int base = 0;
    for (int l = 0; l < n_levels; ++l) {
        const int m = n_sel_lvl[f * RGBL_MAX_LEVELS + l];
        const uint32_t* src = sel_lvl + (size_t)f * cap_kp + lvl_region[l];
        for (int i = threadIdx.x; i < m; i += 256) {
            const uint32_t c = src[i];
            SelKp k;
            k.x = (uint16_t)((c & 0xfffu) + kFastBorder); k.y = (uint16_t)(((c >> 12) & 0xfffu) + kFastBorder);
            k.level = (uint8_t)l; k.score = (uint8_t)(c >> 24); k.pad = 0;
            sel[(size_t)f * cap_kp + base + i] = k;
        }
        base += m;
    }
    if (threadIdx.x == 0) n_sel[f] = base;
}

int quadtree_smem_bytes() { return (int)sizeof(qt::SharedT<512>); }

// dynamic shared memory of one variant: everything an SM offers divided by the resident CTAs (tree state + the per-key arrays when they fit)
template <int MAXN>
static int quadtree_dyn_bytes(int ctas_per_sm) {
    int dev = 0, optin = 0, per_sm = 0;
    cudaFuncAttributes fa{};
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, quadtree_kernel<MAXN>) != cudaSuccess) return -1;
    int avail = optin - (int)fa.sharedSizeBytes - 256;
    if (ctas_per_sm > 1) avail = std::min(avail, per_sm / ctas_per_sm - 1024 /* reserved per CTA */ - (int)fa.sharedSizeBytes - 256);
    if (avail < (int)sizeof(qt::SharedT<MAXN>)) return -1;
    if (cudaFuncSetAttribute(quadtree_kernel<MAXN>, cudaFuncAttributeMaxDynamicSharedMemorySize, avail) != cudaSuccess) return -1;
    return avail;
}

int launch_quadtree(cudaStream_t st, const uint32_t* dense, const int* level_cnt, const int* frame_total, const LevelGeom* d_levels,
                    int n_levels, const QtScratchDev& scr, uint32_t* sel_lvl, int* n_sel_lvl, const int* lvl_region, int cap_kp,
                    int* status, SelKp* sel, int* n_sel, int n_frames, int max_nodes) {
    // max_nodes = the largest node list any level of the context needs (max(quota + 3, 4 nIni)): <= 512 selects the half-size tree state
    // with two CTAs per SM
    static int dyn512 = 0, dyn1024 = 0;
    const bool small = max_nodes <= 512;
    int& dyn_bytes = small ? dyn512 : dyn1024;
    if (!dyn_bytes) dyn_bytes = small ? quadtree_dyn_bytes<512>(2) : quadtree_dyn_bytes<1024>(1);
    if (dyn_bytes <= 0) return -1;
    if (small)
        quadtree_kernel<512><<<dim3(n_frames, n_levels), 512, dyn_bytes, st>>>(dense, level_cnt, frame_total, d_levels, n_levels, scr, sel_lvl, n_sel_lvl,
                                                                             lvl_region, cap_kp, status, dyn_bytes);
    else
        quadtree_kernel<1024><<<dim3(n_frames, n_levels), 512, dyn_bytes, st>>>(dense, level_cnt, frame_total, d_levels, n_levels, scr, sel_lvl, n_sel_lvl,
                                                                              lvl_region, cap_kp, status, dyn_bytes);
    sel_pack_kernel<<<n_frames, 256, 0, st>>>(sel_lvl, n_sel_lvl, lvl_region, n_levels, cap_kp, sel, n_sel);
    return 0;
}

// Host execution of the SAME block algorithm (phase-sequential): CPU validation of the device logic.
int quadtree_block_host(const uint32_t* cand, int n, int width, int height, int N, uint32_t* out, int out_cap) {
    std::vector<qt::KeyIdx> pa(n + 1), pb(n + 1), na(n + 1), nb(n + 1);
    std::vector<unsigned long long> scan(n + 2);
    std::vector<unsigned char> quad(n + 1);
    qt::Scratch g{pa.data(), pb.data(), na.data(), nb.data(), scan.data(), quad.data()};
    qt::Shared* s = new qt::Shared();
    const int m = qt::distribute(*s, cand, n, width, height, N, g, out, out_cap);
    delete s;
    return m;
}

}  // namespace rgbl

#ifdef RGBL_TESTING_EXPORTS        // test hooks: only in librgbl_b200_testing.so (csrc/rgbl_testing.h)
extern "C" {

// test hook: the block algorithm run on the host; xys n x 3 (x, y, score) like rgbl_quadtree_select.  The budget is |n_desired|: the
// sign once chose between two sort formulations with the same survivors, and callers that still pass it get the one that remains.
int rgbl_quadtree_select_block_emulation(const int32_t* xys, int n, int min_x, int max_x, int min_y, int max_y, int n_desired,
                                         int32_t* out_xys, int cap) {
    if (n < 0 || (n > 0 && !xys) || !out_xys) return RGBL_E_INVALID;
    std::vector<uint32_t> c(n), o(cap);
    for (int i = 0; i < n; ++i) c[i] = rgbl::pack_cand(xys[3 * i], xys[3 * i + 1], xys[3 * i + 2]);
    const int m = rgbl::quadtree_block_host(c.data(), n, max_x - min_x, max_y - min_y, n_desired < 0 ? -n_desired : n_desired, o.data(), cap);
    if (m < 0) return RGBL_E_UNSUPPORTED;
    if (m > cap) return RGBL_E_CAPACITY;
    for (int i = 0; i < m; ++i) { out_xys[3 * i] = (int)(o[i] & 0xfff); out_xys[3 * i + 1] = (int)((o[i] >> 12) & 0xfff); out_xys[3 * i + 2] = (int)(o[i] >> 24); }
    return m;
}

// test hook: the restated libstdc++ introsort on (size, ulx) pairs; returns the permutation
int rgbl_std_sort_emulation(const int32_t* size_ulx, int n, int32_t* perm_out) {
    std::vector<rgbl::qt::SortItem> v(n);
    for (int i = 0; i < n; ++i) { v[i].size = size_ulx[2 * i]; v[i].ulx = size_ulx[2 * i + 1]; v[i].node = i; }
    rgbl::qt::std_sort(v.data(), n);
    for (int i = 0; i < n; ++i) perm_out[i] = v[i].node;
    return 0;
}

// test hook: the block-parallel formulation of the same sort (phase-sequential on the host) and, as ground truth, the
// C++ library's own std::sort with the reference's comparator.  mode 0: block formulation with the reference depth limit,
// mode > 0: block formulation with depth limit `mode - 1` (exercises the heapsort fallback), mode < 0: real std::sort.
int rgbl_std_sort_block_emulation(const int32_t* size_ulx, int n, int mode, int32_t* perm_out) {
    if (n < 0 || n > rgbl::qt::kMaxNodes || (n > 0 && (!size_ulx || !perm_out))) return RGBL_E_INVALID;
    std::vector<rgbl::qt::SortItem> v(n + 1), tmp(n + 1);
    for (int i = 0; i < n; ++i) { v[i].size = size_ulx[2 * i]; v[i].ulx = size_ulx[2 * i + 1]; v[i].node = i; }
    if (mode < 0) {
        std::sort(v.begin(), v.begin() + n, [](const rgbl::qt::SortItem& a, const rgbl::qt::SortItem& b) { return rgbl::qt::item_less(a, b); });
    } else {
        rgbl::qt::Shared* s = new rgbl::qt::Shared();
        rgbl::qt::block_std_sort(*s, v.data(), tmp.data(), n, mode - 1);
        delete s;
    }
    for (int i = 0; i < n; ++i) perm_out[i] = v[i].node;
    return 0;
}

}  // extern "C"
#endif  // RGBL_TESTING_EXPORTS
