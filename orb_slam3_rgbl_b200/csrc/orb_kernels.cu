// ORB extractor kernels for sm_90a: pyramid, candidate compaction, 7x7 Gaussian pre-filter and the
// padded copy of a level.
// Reference semantics: src/ORBextractor.cc (cited per kernel) with the OpenCV primitives restated
// in integer/fixed-point form (SURVEY.md Appendix A).  Every frame of a batch is processed by the
// same launch (blockIdx.z / blockIdx.y = frame slot).
#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

// ------------------------------------------------------------------------------------------------
// Pyramid: level l = cv::resize(level l-1, INTER_LINEAR)  (src/ORBextractor.cc:1183, SURVEY A.1).
// One thread produces 4 horizontally adjacent output bytes (one 32-bit store).
// ------------------------------------------------------------------------------------------------
// CTA tile: 128 x 16 outputs.  The source rectangle of the tile (<= 22 rows x 176 bytes at scale 1.2) is staged in shared
// memory with 16-byte loads (rows are 64-byte aligned); every thread then produces 4 adjacent outputs in two rows from
// shared-memory bytes.  (The first version gathered 16 single bytes per thread straight from global memory and was bound by
// the number of load instructions, not by HBM.)
constexpr int kRzTW = 128, kRzTH = 16, kRzSrcRows = 24, kRzSrcVec = 12;     // staged source: 24 rows x 192 bytes max
__global__ void __launch_bounds__(256) resize_level_kernel(uint8_t* __restrict__ pyr, size_t frame_stride,
                                                           LevelGeom src, LevelGeom dst,
                                                           const LinCoef* __restrict__ tabx,
                                                           const LinCoef* __restrict__ taby) {
    __shared__ uint4 tile[kRzSrcRows][kRzSrcVec];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const int x0 = blockIdx.x * kRzTW, y0 = blockIdx.y * kRzTH;
    const uint8_t* s = pyr + (size_t)blockIdx.z * frame_stride + src.off;
    uint8_t* d = pyr + (size_t)blockIdx.z * frame_stride + dst.off;
    // source rectangle of this tile (tables are monotone)
    const int xl = min(x0 + kRzTW - 1, dst.w - 1), yl = min(y0 + kRzTH - 1, dst.h - 1);
    const int sx_lo = tabx[x0].s & ~15, sx_hi = min(tabx[xl].s + 1, src.w - 1);
    const int sy_lo = taby[y0].s, sy_hi = min(taby[yl].s + 1, src.h - 1);
    const int n_vec = min(min((sx_hi - sx_lo) / 16 + 1, kRzSrcVec), (src.pitch - sx_lo) / 16);
    const int n_rows = min(sy_hi - sy_lo + 1, kRzSrcRows);
    for (int i = tid; i < n_rows * n_vec; i += 256) {
        const int r = i / n_vec, v = i - r * n_vec;
        tile[r][v] = __ldg(reinterpret_cast<const uint4*>(s + (size_t)(sy_lo + r) * src.pitch + sx_lo) + v);
    }
    __syncthreads();
    const int x4 = x0 + 4 * tx;
    if (x4 >= dst.w) return;
    const uint8_t* tb = reinterpret_cast<const uint8_t*>(&tile[0][0]);
    constexpr int kTP = kRzSrcVec * 16;
    int s0[4], s1[4], c0[4], c1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const LinCoef cx = tabx[min(x4 + i, dst.w - 1)];
        s0[i] = cx.s - sx_lo; s1[i] = min(cx.s + 1, src.w - 1) - sx_lo; c0[i] = cx.c0; c1[i] = cx.c1;
    }
#pragma unroll
    for (int ry = 0; ry < 2; ++ry) {
        const int y = y0 + ty + 8 * ry;
        if (y >= dst.h) break;
        const LinCoef cy = taby[y];
        const uint8_t* r0 = tb + (cy.s - sy_lo) * kTP;
        const uint8_t* r1 = tb + (min(cy.s + 1, src.h - 1) - sy_lo) * kTP;
        const int b0 = cy.c0, b1 = cy.c1;
        uint32_t out = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (x4 + i < dst.w) {
                const int h0 = (int)r0[s0[i]] * c0[i] + (int)r0[s1[i]] * c1[i];
                const int h1 = (int)r1[s0[i]] * c0[i] + (int)r1[s1[i]] * c1[i];
                const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
                out |= (uint32_t)(v & 0xff) << (8 * i);
            }
        }
        *reinterpret_cast<uint32_t*>(d + (size_t)y * dst.pitch + x4) = out;
    }
}

// Fallback for level ratios whose source rectangle does not fit the staged tile (scale factors above ~1.35): one thread
// gathers the 16 source bytes of 4 adjacent outputs directly from global memory.
__global__ void __launch_bounds__(256) resize_level_gather_kernel(uint8_t* __restrict__ pyr, size_t frame_stride,
                                                                  LevelGeom src, LevelGeom dst,
                                                                  const LinCoef* __restrict__ tabx,
                                                                  const LinCoef* __restrict__ taby) {
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x4 >= dst.w || y >= dst.h) return;
    const uint8_t* s = pyr + (size_t)blockIdx.z * frame_stride + src.off;
    uint8_t* d = pyr + (size_t)blockIdx.z * frame_stride + dst.off;
    const LinCoef cy = taby[y];
    const uint8_t* r0 = s + (size_t)cy.s * src.pitch;
    const uint8_t* r1 = s + (size_t)min(cy.s + 1, src.h - 1) * src.pitch;
    const int b0 = cy.c0, b1 = cy.c1;
    uint32_t out = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int x = x4 + i;
        if (x < dst.w) {
            const LinCoef cx = tabx[x];
            const int s0 = cx.s, s1 = min(s0 + 1, src.w - 1);
            const int h0 = (int)__ldg(r0 + s0) * cx.c0 + (int)__ldg(r0 + s1) * cx.c1;
            const int h1 = (int)__ldg(r1 + s0) * cx.c0 + (int)__ldg(r1 + s1) * cx.c1;
            const int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            out |= (uint32_t)(v & 0xff) << (8 * i);
        }
    }
    *reinterpret_cast<uint32_t*>(d + (size_t)y * dst.pitch + x4) = out;
}

// ------------------------------------------------------------------------------------------------
// Candidate compaction.  Pass A (one CTA per frame): exclusive scan of the cell counts in reference
// cell order -> per-cell offsets, per-level counts/offsets, frame total.  Pass B (grid of CTAs):
// every CTA recomputes the tiny prefix over frame totals and copies its cells' slot arrays into one
// dense buffer, so the host fetches exactly sum(total) candidates with a single copy.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cand_scan_kernel(const int* __restrict__ counts, int n_cells,
                                                        const LevelGeom* __restrict__ levels, int n_levels,
                                                        int* __restrict__ cell_off, int* __restrict__ level_cnt,
                                                        int* __restrict__ frame_total) {
    __shared__ int warp_sums[8];
    __shared__ int carry;
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int* c = counts + (size_t)frame * n_cells;
    int* o = cell_off + (size_t)frame * n_cells;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int b = 0; b < n_cells; b += 256) {
        const int i = b + tid;
        const int v = (i < n_cells) ? c[i] : 0;
        int incl = v;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, k);
            if (lane >= k) incl += t;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        int base = carry;
        for (int w = 0; w < warp; ++w) base += warp_sums[w];
        if (i < n_cells) o[i] = base + incl - v;
        __syncthreads();
        if (tid == 255) carry = base + incl;
        __syncthreads();
    }
    if (tid < n_levels) {
        const LevelGeom lg = levels[tid];
        int s = 0;
        for (int k = 0; k < lg.n_cells; ++k) s += c[lg.cell_base + k];
        level_cnt[frame * RGBL_MAX_LEVELS + tid] = s;
    }
    if (tid == 0) frame_total[frame] = carry;
}

__global__ void __launch_bounds__(256) cand_gather_kernel(const uint32_t* __restrict__ slots,
                                                          const int* __restrict__ counts,
                                                          const int* __restrict__ cell_off,
                                                          const int* __restrict__ frame_total, int n_cells,
                                                          uint32_t* __restrict__ dense, int dense_cap,
                                                          int* __restrict__ overflow) {
    const int frame = blockIdx.y;
    int fbase = 0;
    for (int f = 0; f < frame; ++f) fbase += frame_total[f];
    const int warp_global = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    const int n_warps = gridDim.x * 8;
    for (int cell = warp_global; cell < n_cells; cell += n_warps) {
        const int n = counts[(size_t)frame * n_cells + cell];
        const int off = fbase + cell_off[(size_t)frame * n_cells + cell];
        const uint32_t* s = slots + ((size_t)frame * n_cells + cell) * kCellCap;
        for (int k = lane; k < n; k += 32) {
            if (off + k < dense_cap) dense[off + k] = s[k];
            else atomicExch(overflow, 2);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// cv::GaussianBlur(7x7, sigma 2, BORDER_REFLECT_101) on each un-padded level (src/ORBextractor.cc:
// 1132-1133; SURVEY A.2): 8.8 fixed-point kernel {18,34,48,56,48,34,18}, exact separable sums, one
// final rounding.  CTA tile: 64 x 32 outputs; each thread writes 4 adjacent bytes.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int reflect101(int p, int n) {
    if (p < 0) p = -p;
    if (p >= n) p = 2 * (n - 1) - p;
    return p;
}

__global__ void __launch_bounds__(256) blur_level_kernel(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ blur,
                                                         size_t frame_stride, LevelGeom lg) {
    // CTA tile: 128 x 32 outputs.  Input rows are staged as 32-bit words (aligned loads in the interior, per-byte
    // REFLECT_101 assembly on the level's edges); the horizontal pass keeps 8.8 sums packed as u16x2; the vertical
    // pass gives every thread a 4 x 4 output block (one 32-bit store per row).
    constexpr int TW = 128, TH = 32, IH = TH + 6, IWW = (TW + 8) / 4;     // 34 input words per row: x0-4 .. x0+131
    __shared__ uint32_t in[IH][IWW + 1];
    __shared__ uint32_t hb[IH][TW / 2 + 1];
    const uint8_t* s = pyr + (size_t)blockIdx.z * frame_stride + lg.off;
    uint8_t* d = blur + (size_t)blockIdx.z * frame_stride + lg.off;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int r = warp; r < IH; r += 8) {
        const int gy = reflect101(y0 + r - 3, lg.h);
        const uint8_t* row = s + (size_t)gy * lg.pitch;
        for (int w = lane; w < IWW; w += 32) {
            const int gx = x0 - 4 + 4 * w;
            uint32_t v;
            if (gx >= 0 && gx + 3 < lg.w) {
                v = __ldg(reinterpret_cast<const uint32_t*>(row + gx));
            } else {
                v = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    int px = gx + k;
                    px = reflect101(px, lg.w);
                    px = min(max(px, 0), lg.w - 1);             // tiles hanging far over the right edge: value unused
                    v |= (uint32_t)__ldg(row + px) << (8 * k);
                }
            }
            in[r][w] = v;
        }
    }
    __syncthreads();
    for (int item = tid; item < IH * 32; item += 256) {
        const int r = item >> 5, g = item & 31;                 // g: group of 4 output columns
        const uint32_t w0 = in[r][g], w1 = in[r][g + 1], w2 = in[r][g + 2];
        int b[12];
#pragma unroll
        for (int k = 0; k < 4; ++k) { b[k] = (w0 >> (8 * k)) & 0xff; b[4 + k] = (w1 >> (8 * k)) & 0xff; b[8 + k] = (w2 >> (8 * k)) & 0xff; }
        uint32_t acc[4];
#pragma unroll
        for (int jx = 0; jx < 4; ++jx)
            acc[jx] = 18 * (b[1 + jx] + b[7 + jx]) + 34 * (b[2 + jx] + b[6 + jx]) + 48 * (b[3 + jx] + b[5 + jx]) + 56 * b[4 + jx];
        hb[r][2 * g] = acc[0] | (acc[1] << 16);
        hb[r][2 * g + 1] = acc[2] | (acc[3] << 16);
    }
    __syncthreads();
    {
        const int g = lane, rg = warp;                          // 32 column groups x 8 row groups of 4 rows
        const int gx = x0 + 4 * g;
        if (gx >= lg.w) return;
        uint32_t c0[10], c1[10];
#pragma unroll
        for (int k = 0; k < 10; ++k) { c0[k] = hb[4 * rg + k][2 * g]; c1[k] = hb[4 * rg + k][2 * g + 1]; }
#pragma unroll
        for (int ry = 0; ry < 4; ++ry) {
            const int gy = y0 + 4 * rg + ry;
            if (gy >= lg.h) break;
            uint32_t out = 0;
#pragma unroll
            for (int jx = 0; jx < 4; ++jx) {
                uint32_t h[7];
#pragma unroll
                for (int k = 0; k < 7; ++k) {
                    const uint32_t w = (jx < 2) ? c0[ry + k] : c1[ry + k];
                    h[k] = (jx & 1) ? (w >> 16) : (w & 0xffffu);
                }
                const uint32_t acc = 18u * (h[0] + h[6]) + 34u * (h[1] + h[5]) + 48u * (h[2] + h[4]) + 56u * h[3];
                out |= ((acc + 32768u) >> 16) << (8 * jx);
            }
            *reinterpret_cast<uint32_t*>(d + (size_t)gy * lg.pitch + gx) = out;
        }
    }
}

// mvImagePyramid[level] with its 19 px BORDER_REFLECT_101 frame (src/ORBextractor.cc:1185-1191),
// synthesised on demand: the hot path itself never reads the border (SURVEY App. C).
__global__ void padded_level_kernel(const uint8_t* __restrict__ pyr, size_t frame_stride, int frame, LevelGeom lg,
                                    uint8_t* __restrict__ dst, int dst_pitch) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const int W = lg.w + 2 * kEdgeThreshold, H = lg.h + 2 * kEdgeThreshold;
    if (x >= W || y >= H) return;
    const uint8_t* s = pyr + (size_t)frame * frame_stride + lg.off;
    dst[(size_t)y * dst_pitch + x] = s[(size_t)reflect101(y - kEdgeThreshold, lg.h) * lg.pitch + reflect101(x - kEdgeThreshold, lg.w)];
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
void launch_pyramid(cudaStream_t st, uint8_t* pyr, size_t frame_stride, const LevelGeom* h_levels, int n_levels,
                    const LinCoef* d_coefs, int n_frames) {
    for (int l = 1; l < n_levels; ++l) {
        const LevelGeom& src = h_levels[l - 1];
        const LevelGeom& dst = h_levels[l];
        const double rx = (double)src.w / dst.w, ry = (double)src.h / dst.h;
        if (rx * (kRzTW - 1) + 18.0 <= kRzSrcVec * 16 - 1 && ry * (kRzTH - 1) + 3.0 <= kRzSrcRows) {
            dim3 grd((dst.w + kRzTW - 1) / kRzTW, (dst.h + kRzTH - 1) / kRzTH, n_frames);
            resize_level_kernel<<<grd, 256, 0, st>>>(pyr, frame_stride, src, dst, d_coefs + dst.tabx_off, d_coefs + dst.taby_off);
        } else {
            dim3 blk(32, 8), grd(((dst.w + 3) / 4 + 31) / 32, (dst.h + 7) / 8, n_frames);
            resize_level_gather_kernel<<<grd, blk, 0, st>>>(pyr, frame_stride, src, dst, d_coefs + dst.tabx_off, d_coefs + dst.taby_off);
        }
    }
}

void launch_compact(cudaStream_t st, const LevelGeom* d_levels, int n_levels, int n_cells, const uint32_t* slots,
                    const int* counts, int* cell_off, int* level_cnt, int* frame_total, uint32_t* dense, int dense_cap,
                    int* overflow, int n_frames) {
    cand_scan_kernel<<<n_frames, 256, 0, st>>>(counts, n_cells, d_levels, n_levels, cell_off, level_cnt, frame_total);
    const int gx = (n_cells + 63) / 64;
    cand_gather_kernel<<<dim3(gx, n_frames), 256, 0, st>>>(slots, counts, cell_off, frame_total, n_cells, dense,
                                                         dense_cap, overflow);
}

void launch_blur(cudaStream_t st, const uint8_t* pyr, uint8_t* blur, size_t frame_stride, const LevelGeom* h_levels,
                 int n_levels, int n_frames) {
    for (int l = 0; l < n_levels; ++l) {
        const LevelGeom& lg = h_levels[l];
        dim3 grd((lg.w + 127) / 128, (lg.h + 31) / 32, n_frames);
        blur_level_kernel<<<grd, 256, 0, st>>>(pyr, blur, frame_stride, lg);
    }
}

void launch_padded_level(cudaStream_t st, const uint8_t* pyr, size_t frame_stride, int frame, const LevelGeom& lg,
                         uint8_t* dst, int dst_pitch) {
    const int W = lg.w + 2 * kEdgeThreshold, H = lg.h + 2 * kEdgeThreshold;
    padded_level_kernel<<<dim3((W + 31) / 32, (H + 7) / 8), dim3(32, 8), 0, st>>>(pyr, frame_stride, frame, lg, dst, dst_pitch);
}

}  // namespace rgbl
