// Strip formulation of the per-cell FAST detection (src/ORBextractor.cc:805-868): one CTA handles a run of consecutive
// cells of one cell row ("strip") instead of one cell.
//
// Why it is the same function.  The cells' windows overlap by 6 px, but the pixels cv::FAST *tests* in a window are
// [3, cw-3) x [3, ch-3), and those regions tile the level without overlap.  The score of a pixel (arc strength K-1, 0 when
// K <= minTh) does not depend on the cell; the only cell-dependent steps are
//   * non-maximum suppression: neighbours outside the cell's tested region count as 0 (cv::FAST never scores them),
//   * the iniTh -> minTh fallback, decided per cell ("no keypoint at iniTh in this cell"),
//   * the output order: row-major inside the cell, cells in table order.
// So a strip scores every pixel once (a CTA per cell would re-read the 3 px halo of every cell and pay its fixed costs
// per 30 x 30 px), masks the NMS comparisons at the inner cell boundaries, and emits per cell.
//
// The body is bulk-synchronous (FS_FOR loops separated by FS_SYNC) and compiles for the host as well, where every phase
// runs its "threads" one after the other: tests/test_host_abi.py checks that twin against the oracle's per-cell FAST on
// real pyramid levels, so what remains to be validated on a GPU are only the device-only helpers (shared-memory atomics,
// the shuffle scan) and the launch geometry.
#ifndef RGBL_FAST_STRIP_CUH
#define RGBL_FAST_STRIP_CUH

#include <stdint.h>

#include "rgbl_device.cuh"

#if defined(__CUDA_ARCH__)
#define FS_DEVICE 1
#define FS_FN __device__ __forceinline__
#define FS_TID ((int)threadIdx.x)
#define FS_NT ((int)blockDim.x)
#define FS_SYNC() __syncthreads()
#else
#define FS_DEVICE 0
#define FS_FN inline
#define FS_TID 0
#define FS_NT 1
#define FS_SYNC()
#include <cstring>
#endif
#define FS_FOR(i, n) for (int i = FS_TID; i < (n); i += FS_NT)

namespace rgbl {
namespace fs {

constexpr int kPitch = 272;            // tile row pitch in bytes: <= 3 alignment bytes + <= 264 px window + slack for the x+3 word
constexpr int kMaxWidth = 264;         // strip window width limit
constexpr int kMaxCells = 8;           // cells per strip
constexpr int kMaxRows = 78;           // window height limit (the same limit build_geometry enforces per cell)
constexpr int kCntInts = kMaxCells * (kMaxRows - 6) + 8;
// misc[] layout
constexpr int kNList = 0, kAnyIni = 1, kCellL = kAnyIni + kMaxCells, kCellR = kCellL + kMaxCells, kWarpSums = kCellR + kMaxCells,
              kNWords = kWarpSums + 32, kMiscInts = kNWords + 1;

// ---- packed 16x2 helpers (VIMNMX.S16x2 / VIADD.16x2 / PRMT on sm_90a; plain C on the host) -------------------------------
FS_FN uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
#if FS_DEVICE
    return __byte_perm(a, b, sel);
#else
    const uint64_t src = (uint64_t)a | ((uint64_t)b << 32);
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((src >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
#endif
}
FS_FN uint32_t min2(uint32_t a, uint32_t b) {
#if FS_DEVICE
    return __vmins2(a, b);
#else
    const int16_t a0 = (int16_t)a, a1 = (int16_t)(a >> 16), b0 = (int16_t)b, b1 = (int16_t)(b >> 16);
    return (uint32_t)(uint16_t)(a0 < b0 ? a0 : b0) | ((uint32_t)(uint16_t)(a1 < b1 ? a1 : b1) << 16);
#endif
}
FS_FN uint32_t max2(uint32_t a, uint32_t b) {
#if FS_DEVICE
    return __vmaxs2(a, b);
#else
    const int16_t a0 = (int16_t)a, a1 = (int16_t)(a >> 16), b0 = (int16_t)b, b1 = (int16_t)(b >> 16);
    return (uint32_t)(uint16_t)(a0 > b0 ? a0 : b0) | ((uint32_t)(uint16_t)(a1 > b1 ? a1 : b1) << 16);
#endif
}
FS_FN int popc(uint32_t v) {
#if FS_DEVICE
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}
FS_FN int imax(int a, int b) { return a > b ? a : b; }
FS_FN uint32_t pack(int x, int y, int s) { return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)s << 24); }   // = pack_cand
FS_FN uint32_t sub2(uint32_t a, uint32_t b) {                 // per-half wrapping a - b
#if FS_DEVICE
    return __vsub2(a, b);
#else
    return (uint32_t)(uint16_t)((uint16_t)a - (uint16_t)b) | ((uint32_t)(uint16_t)((uint16_t)(a >> 16) - (uint16_t)(b >> 16)) << 16);
#endif
}

FS_FN uint32_t shl8(uint32_t prev, uint32_t cur) {             // bytes of `cur` moved up one position, byte 3 of `prev` shifted in: byte k = pixel k-1
#if FS_DEVICE
    return __funnelshift_l(prev, cur, 8);
#else
    return (cur << 8) | (prev >> 24);
#endif
}
FS_FN uint32_t shr8(uint32_t cur, uint32_t next) {             // byte k = pixel k+1
#if FS_DEVICE
    return __funnelshift_r(cur, next, 8);
#else
    return (cur >> 8) | (next << 24);
#endif
}
FS_FN uint32_t even_bytes(uint32_t w) { return w & 0x00ff00ffu; }          // bytes 0, 2 widened to 16x2
FS_FN uint32_t odd_bytes(uint32_t w) { return (w >> 8) & 0x00ff00ffu; }    // bytes 1, 3

// Flattened 2-D iteration (y, x) over ny x nx items without a division per item: item i = FS_TID + k * FS_NT.
struct Iter2D { int i, n, y, x, q, r, nx; };
FS_FN Iter2D it_begin(int ny, int nx) {
    Iter2D it;
    it.nx = nx; it.n = (ny > 0 && nx > 0) ? ny * nx : 0; it.i = FS_TID;
    it.y = it.n ? it.i / nx : 0; it.x = it.i - it.y * nx;
    it.q = it.n ? FS_NT / nx : 0; it.r = FS_NT - it.q * nx;
    return it;
}
FS_FN void it_next(Iter2D& it) {
    it.i += FS_NT; it.x += it.r; it.y += it.q;
    if (it.x >= it.nx) { it.x -= it.nx; ++it.y; }
}

// High-speed test of 4 horizontally adjacent pixels (the word `ctr` of row `row`): bit k of the result is set when pixel k has
// at least two of its four compass ring points brighter than v + th, or at least two darker than v - th (a 9-arc of the
// 16-ring always contains two adjacent compass points, so this is necessary for a corner at threshold th).
// "At least two of four above hi" <=> the second largest is above hi; computed on two pixels at a time in 16-bit halves.
FS_FN uint32_t quick_test4(uint32_t ctr, uint32_t up, uint32_t dn, uint32_t lf, uint32_t rt, uint32_t th2) {
    const uint32_t w12 = prmt(lf, ctr, 0x4321), w4 = prmt(ctr, rt, 0x6543);      // p[-3], p[+3] of the four pixels
    uint32_t bits = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t sel = h ? 0x4342u : 0x4140u;           // bytes (2h, 2h+1) widened to 16x2
        const uint32_t v = prmt(ctr, 0, sel), a = prmt(dn, 0, sel), b = prmt(up, 0, sel), c = prmt(w4, 0, sel), d = prmt(w12, 0, sel);
        const uint32_t mn1 = min2(a, b), mx1 = max2(a, b), mn2 = min2(c, d), mx2 = max2(c, d);
        const uint32_t second_largest = max2(max2(mn1, mn2), min2(mx1, mx2));
        const uint32_t second_smallest = min2(min2(mx1, mx2), max2(mn1, mn2));
        const uint32_t kq = max2(sub2(second_largest, v), sub2(v, second_smallest));
        const uint32_t neg = sub2(th2, kq) & 0x80008000u;     // th - kq < 0  <=>  kq > th   (|values| <= 510: no wrap)
        bits |= (((neg >> 15) & 1u) | ((neg >> 30) & 2u)) << (2 * h);
    }
    return bits;
}

// fast_arc_strength16 (rgbl_device.cuh) on two pixels at once: every value is a 16x2 pair (pixel A low half, pixel B high half).
FS_FN uint32_t arc_strength16_x2(uint32_t v, const uint32_t r[16]) {
    uint32_t m2[16], M2[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) { m2[s] = min2(r[s], r[(s + 1) & 15]); M2[s] = max2(r[s], r[(s + 1) & 15]); }
    uint32_t m4[16], M4[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) { m4[s] = min2(m2[s], m2[(s + 2) & 15]); M4[s] = max2(M2[s], M2[(s + 2) & 15]); }
    uint32_t lo = 0x00ff00ffu, hi = 0;
#pragma unroll
    for (int s = 0; s < 16; ++s) {
        const uint32_t m8 = min2(m4[s], m4[(s + 4) & 15]), M8 = max2(M4[s], M4[(s + 4) & 15]);
        const uint32_t m9 = min2(m8, r[(s + 8) & 15]), M9 = max2(M8, r[(s + 8) & 15]);
        lo = min2(lo, M9);
        hi = max2(hi, m9);
    }
    return max2(sub2(v, lo), sub2(hi, v));
}

// cv scores (K-1 at threshold th, 0 when not a corner) of the pixels at tile positions pa and pb
FS_FN void score_pair(const uint8_t* tile, int pa, int pb, int th, int* sa, int* sb) {
    constexpr int P = kPitch;
    constexpr int off[16] = {3 * P, 3 * P + 1, 2 * P + 2, P + 3, 3, -P + 3, -2 * P + 2, -3 * P + 1,
                             -3 * P, -3 * P - 1, -2 * P - 2, -P - 3, -3, P - 3, 2 * P - 2, 3 * P - 1};     // ring order of SURVEY A.3
    const uint8_t* a = tile + pa;
    const uint8_t* b = tile + pb;
    uint32_t r[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) r[k] = (uint32_t)a[off[k]] | ((uint32_t)b[off[k]] << 16);
    const uint32_t K = arc_strength16_x2((uint32_t)a[0] | ((uint32_t)b[0] << 16), r);
    const int ka = (int)(int16_t)(K & 0xffffu), kb = (int)(int16_t)(K >> 16);      // K < 0 when every arc has pixels on both sides of v
    *sa = ka > th ? ka - 1 : 0;
    *sb = kb > th ? kb - 1 : 0;
}

FS_FN uint32_t byte_range_mask(int lo, int hi) {               // bytes [lo, hi) of a word, clipped to [0, 4)
    const uint32_t m_hi = hi >= 4 ? 0xffffffffu : (hi <= 0 ? 0u : ((1u << (8 * hi)) - 1u));
    const uint32_t m_lo = lo <= 0 ? 0xffffffffu : (lo >= 4 ? 0u : ~((1u << (8 * lo)) - 1u));
    return m_hi & m_lo;
}

// Exclusive prefix sum of v[0..n) in place, v[n] = total.  Device: n <= any size (every thread owns a contiguous chunk).
FS_FN void exclusive_scan(int* v, int n, int* warp_sums) {
#if FS_DEVICE
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
    const int per = (n + blockDim.x - 1) / blockDim.x;
    const int b = min(tid * per, n), e = min(b + per, n);
    int s = 0;
    for (int i = b; i < e; ++i) s += v[i];
    int incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    int run = incl - s;
    for (int w = 0; w < n_warps; ++w) if (w < warp) run += warp_sums[w];
    for (int i = b; i < e; ++i) { const int t = v[i]; v[i] = run; run += t; }
    if (tid == (int)blockDim.x - 1) v[n] = run;
    __syncthreads();
#else
    (void)warp_sums;
    int run = 0;
    for (int i = 0; i < n; ++i) { const int t = v[i]; v[i] = run; run += t; }
    v[n] = run;
#endif
}

// One strip of one frame.  lvl: this frame's level origin; tile / sc: rows_cap x kPitch bytes each (16-byte aligned);
// list: list_cap entries, one per tested pixel of the strip (the list of score-carrying words grows down from its end); cnt: kCntInts;
// misc: kMiscInts.
FS_FN void run(const uint8_t* lvl, int pitch, const StripInfo si, const CellInfo* cells, int min_bx, int min_by, int ini_th, int min_th,
               uint8_t* tile, uint8_t* sc, uint16_t* list, int list_cap, int* cnt, int* misc, uint32_t* slots, int* counts, int* overflow) {
    constexpr int P = kPitch, PW = kPitch / 4;
    uint32_t* tile32 = reinterpret_cast<uint32_t*>(tile);
    uint32_t* sc32 = reinterpret_cast<uint32_t*>(sc);
    const int a = si.x0 & 3;                               // tile byte 0 = level column x0 - a (word aligned in global memory)
    const int w = si.w, h = si.h, n_cells = si.n_cells;
    const int nw = (w + a + 3) >> 2;                       // words per row holding the window
    const uint8_t* src = lvl + (size_t)si.y0 * pitch + (si.x0 - a);

    // ---- P0: window -> shared memory, score map cleared, per-cell tested column ranges ---------------------------------
    for (Iter2D it = it_begin(h, nw); it.i < it.n; it_next(it)) {
        uint32_t v;
#if FS_DEVICE
        v = __ldg(reinterpret_cast<const uint32_t*>(src + (size_t)it.y * pitch) + it.x);
#else
        std::memcpy(&v, src + (size_t)it.y * pitch + 4 * it.x, 4);
#endif
        tile32[it.y * PW + it.x] = v;
        sc32[it.y * PW + it.x] = 0;
    }
    FS_FOR(k, n_cells) {
        const CellInfo ci = cells[si.first_cell + k];
        misc[kCellL + k] = ci.x0 - si.x0 + a + 3;          // tested columns [L, R) of cell k in tile coordinates
        misc[kCellR + k] = ci.x0 - si.x0 + a + ci.cw - 3;
        misc[kAnyIni + k] = 0;
    }
    if (FS_TID == 0) { misc[kNList] = 0; misc[kNWords] = 0; }
    // per tile word: 0x00 in the bytes whose pixel is the first (lmask) / last (rmask) tested column of a cell - the NMS of that pixel
    // does not look at its left / right neighbours (they belong to another cv::FAST call).  cnt[] is free until P4.
    uint32_t* lmask = reinterpret_cast<uint32_t*>(cnt);
    uint32_t* rmask = lmask + PW;
    FS_FOR(c, PW) {
        uint32_t lm = 0xffffffffu, rm = 0xffffffffu;
        for (int k = 0; k < n_cells; ++k) {
            const CellInfo ci = cells[si.first_cell + k];
            const int L = ci.x0 - si.x0 + a + 3, R1 = ci.x0 - si.x0 + a + ci.cw - 4;
            if ((L >> 2) == c) lm &= ~(0xffu << (8 * (L & 3)));
            if (R1 >= 0 && (R1 >> 2) == c) rm &= ~(0xffu << (8 * (R1 & 3)));
        }
        lmask[c] = lm; rmask[c] = rm;
    }
    FS_SYNC();

    const int ny = h > 6 ? h - 6 : 0;                      // tested rows [3, h-3)
    const int tx0 = a + 3, tx1 = a + w - 3;                // tested columns [tx0, tx1) of the strip
    const int wb = tx0 >> 2, nxw = (w > 6) ? ((tx1 - 1) >> 2) - wb + 1 : 0;

    // ---- P1: high-speed test, 4 pixels per item; survivors appended to the list ---------------------------------------
    {
        const uint32_t th2 = (uint32_t)min_th * 0x00010001u;
        for (Iter2D it = it_begin(ny, nxw); it.i < it.n; it_next(it)) {
            const int row = it.y + 3, c = wb + it.x;
            const uint32_t* t = tile32 + row * PW + c;
            uint32_t bits = quick_test4(t[0], t[-3 * PW], t[3 * PW], t[-1], t[1], th2);
            const int lo = tx0 - 4 * c, hi = tx1 - 4 * c;    // valid pixel range of this word
            bits &= (hi >= 4 ? 0xfu : ((1u << hi) - 1u)) & (lo <= 0 ? 0xfu : (0xfu << lo));
            if (bits) {
#if FS_DEVICE
                int base = atomicAdd(&misc[kNList], popc(bits));
#else
                int base = misc[kNList];
                for (uint32_t b = bits; b; b &= b - 1) ++misc[kNList];
#endif
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (bits & (1u << k)) list[base++] = (uint16_t)(row * P + 4 * c + k);
            }
        }
    }
    FS_SYNC();

    // ---- P2: arc strength of the listed pixels (dense over the CTA).  A corner's score goes into the score map with an OR on its
    //          word (the map was cleared in P0, every byte is written once); the pixel that finds the word still empty appends the
    //          word to a second list, so that P3 runs densely over the words that hold a score at all (about one in five) instead of
    //          branching around the others with every warp paying for the full path.  The word list grows DOWN from the end of the
    //          pixel list's buffer (an own buffer cost a resident CTA per SM): that is safe when both lists fit, nl + min(nl, words)
    //          <= list_cap, which only a window where nearly every pixel passes the high-speed test violates - then P3 walks all words. --
    const int nl = misc[kNList];
    const int n_tested_words = ny * nxw;
    const bool dense_nms = nl + (nl < n_tested_words ? nl : n_tested_words) <= list_cap;
    uint16_t* words_top = list + list_cap - 1;             // word k of the second list = words_top[-k]
    {
        FS_FOR(j, (nl + 1) >> 1) {                         // two listed pixels per item, packed 16x2
            const int pa = list[2 * j], pb = (2 * j + 1 < nl) ? list[2 * j + 1] : pa;
            int sa, sb;
            score_pair(tile, pa, pb, min_th, &sa, &sb);
            if (pb == pa) sb = 0;
            if (!dense_nms) {
                sc[pa] = (uint8_t)sa;
                if (pb != pa) sc[pb] = (uint8_t)sb;
                continue;
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int pp = u ? pb : pa, sv = u ? sb : sa;
                if (sv == 0) continue;
                const uint32_t add = (uint32_t)sv << (8 * (pp & 3));
#if FS_DEVICE
                const uint32_t old = atomicOr(&sc32[pp >> 2], add);
                if (!old) words_top[-atomicAdd(&misc[kNWords], 1)] = (uint16_t)(pp >> 2);
#else
                const uint32_t old = sc32[pp >> 2];
                sc32[pp >> 2] = old | add;
                if (!old) words_top[-(misc[kNWords]++)] = (uint16_t)(pp >> 2);
#endif
            }
        }
    }
    FS_SYNC();

    // ---- P3: 3x3 non-maximum suppression inside each cell's tested region; flags (1 = survivor at minTh, 3 = also at iniTh)
    //          overwrite the (no longer needed) pixel tile words of the score-carrying words.  Four pixels per item, branch-free: the eight neighbour scores of the
    //          word's pixels are byte-shifted copies of nine score words; byte maxima are taken on even / odd bytes widened to 16x2
    //          (VIMNMX.U16x2), "s > m" and "s >= iniTh" are bit 8 of s + 255 - m and s + 256 - iniTh per half. -------------------
    {
        const uint32_t ini2 = (uint32_t)(ini_th < 0 ? 0 : (ini_th > 256 ? 256 : ini_th)) * 0x00010001u;   // scores are <= 255
        auto nms_word = [&](const int wi, const int c) {
            const uint32_t* q = sc32 + wi;
            const uint32_t mid = q[0];
            uint32_t flags = 0;
            {
                const uint32_t up = q[-PW], dn = q[PW];
                const uint32_t l0 = shl8(q[-PW - 1], up), l1 = shl8(q[-1], mid), l2 = shl8(q[PW - 1], dn);
                const uint32_t r0 = shr8(up, q[-PW + 1]), r1 = shr8(mid, q[1]), r2 = shr8(dn, q[PW + 1]);
                const uint32_t lm = lmask[c], rm = rmask[c];
                uint32_t res[2];
#pragma unroll
                for (int o = 0; o < 2; ++o) {              // o = 0: pixels 0, 2 of the word; o = 1: pixels 1, 3
#define RGBL_H(w) (o ? odd_bytes(w) : even_bytes(w))
                    const uint32_t ml = max2(max2(RGBL_H(l0), RGBL_H(l1)), RGBL_H(l2)) & RGBL_H(lm);
                    const uint32_t mr = max2(max2(RGBL_H(r0), RGBL_H(r1)), RGBL_H(r2)) & RGBL_H(rm);
                    const uint32_t m = max2(max2(RGBL_H(up), RGBL_H(dn)), max2(ml, mr));
                    const uint32_t sv = RGBL_H(mid);
#undef RGBL_H
                    const uint32_t gt = ((sv + 0x00ff00ffu - m) >> 8) & 0x00010001u;          // s > m  (s > m >= 0 implies s > 0)
                    const uint32_t ge = ((sv + 0x01000100u - ini2) >> 8) & 0x00010001u;       // s >= iniTh
                    res[o] = gt | ((gt & ge) << 1);
                }
                flags = res[0] | (res[1] << 8);
                uint32_t ini = flags & 0x02020202u;
                while (ini) {                              // rare: a survivor at iniTh marks its cell
#if FS_DEVICE
                    const int k = (__ffs(ini) - 1) >> 3;
#else
                    int k = 0; while (!((ini >> (8 * k)) & 0xff)) ++k;
#endif
                    ini &= ~(0xffu << (8 * k));
                    const int x = 4 * c + k;
                    int cell = 0;
                    while (cell < n_cells - 1 && x >= misc[kCellR + cell]) ++cell;
#if FS_DEVICE
                    atomicOr(&misc[kAnyIni + cell], 1);     // several survivors of a cell may set it: keep racecheck clean
#else
                    misc[kAnyIni + cell] = 1;
#endif
                }
            }
            tile32[wi] = flags;              // dense form: only the listed words hold flags, the others still pixels (P4 looks at sc32 first)
        };
        if (dense_nms) {
            const int n_words = misc[kNWords];
            FS_FOR(j, n_words) {
                const int wi = words_top[-j], row = wi / PW;
                nms_word(wi, wi - row * PW);
            }
        } else {
            for (Iter2D it = it_begin(ny, nxw); it.i < it.n; it_next(it)) {
                const int wi = (it.y + 3) * PW + wb + it.x;
                if (sc32[wi]) nms_word(wi, wb + it.x); else tile32[wi] = 0;
            }
        }
    }
    FS_SYNC();

    // ---- P4: per (cell, row) counts -> exclusive scan -> ordered emission --------------------------------------------------
    const int n_items = n_cells * ny;
    FS_FOR(it, n_items) {
        const int k = it / ny, row = it - k * ny + 3;
        const int L = misc[kCellL + k], R = misc[kCellR + k];
        const uint32_t sel = misc[kAnyIni + k] ? 0x02020202u : 0x01010101u;
        int n = 0;
        if (R > L)
            for (int wd = L >> 2; wd <= (R - 1) >> 2; ++wd)
                if (sc32[row * PW + wd]) n += popc(tile32[row * PW + wd] & sel & byte_range_mask(L - 4 * wd, R - 4 * wd));
        cnt[it] = n;
    }
    FS_SYNC();
    exclusive_scan(cnt, n_items, misc + kWarpSums);
    FS_FOR(it, n_items) {
        const int k = it / ny, row = it - k * ny + 3;
        const int L = misc[kCellL + k], R = misc[kCellR + k];
        const uint32_t sel = misc[kAnyIni + k] ? 0x02020202u : 0x01010101u;
        int pos = cnt[it] - cnt[k * ny];
        uint32_t* out = slots + (size_t)(si.first_cell + k) * kCellCap;
        if (R > L)
            for (int wd = L >> 2; wd <= (R - 1) >> 2; ++wd) {
                uint32_t f = sc32[row * PW + wd] ? (tile32[row * PW + wd] & sel & byte_range_mask(L - 4 * wd, R - 4 * wd)) : 0u;
                while (f) {
#if FS_DEVICE
                    const int b = (__ffs(f) - 1) >> 3;
#else
                    int b = 0; while (!((f >> (8 * b)) & 0xff)) ++b;
#endif
                    f &= ~(0xffu << (8 * b));
                    const int x = 4 * wd + b;
                    if (pos < kCellCap)
                        out[pos] = pack(si.x0 - a + x - min_bx, si.y0 + row - min_by, sc[row * P + x]);
                    ++pos;
                }
            }
    }
    FS_FOR(k, n_cells) {
        const int total = ny ? cnt[(k + 1) * ny] - cnt[k * ny] : 0;
        counts[si.first_cell + k] = total < kCellCap ? total : kCellCap;
        if (total > kCellCap) {
#if FS_DEVICE
            atomicExch(overflow, 1);
#else
            *overflow = 1;
#endif
        }
    }
}

}  // namespace fs
}  // namespace rgbl

#endif
