// Block-parallel quad-tree keypoint distribution: the semantics of ORBextractor::DistributeOctTree
// (src/ORBextractor.cc:555-779) for ONE (frame, level), executed by one CTA.  The sequential reference
// (std::list + std::vector per node + std::sort) is re-expressed as bulk-synchronous passes:
//
//   * the node "list" is an array kept in list order and rebuilt every pass:
//        new list = reverse(children pushed this pass, in push order)  ++  surviving old nodes in old order
//   * every node owns a contiguous segment of one key permutation; dividing a set D of nodes is a segmented,
//     stable 4-way partition computed with one block-wide scan of packed quadrant counters
//   * the budgeted expansion (":689-754") sorts (size, UL.x) with an exact re-implementation of libstdc++'s
//     std::sort (introsort: median-of-3 to first, unguarded partition, heapsort fallback, final insertion
//     sort with threshold 16) so that ties land exactly where the reference's sort puts them, then finds how
//     many nodes the sequential loop would divide before the list reaches N with a prefix sum
//   * survivors = first key with the maximal response per node, emitted in list order.
//
// The same source compiles for the host (QT_HOST: every phase runs its "threads" sequentially) so the logic is
// validated on the CPU against the oracle's std::list restatement (tests/test_host_abi.py).
#ifndef RGBL_QUADTREE_BLOCK_CUH
#define RGBL_QUADTREE_BLOCK_CUH

#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define QT_DEVICE 1
#define QT_FN __device__
#define QT_BIG __device__ __noinline__
#define QT_NT ((int)blockDim.x)
#define QT_FOR(i, n) for (int i = threadIdx.x; i < (n); i += blockDim.x)
#define QT_SYNC() __syncthreads()
#define QT_SINGLE if (threadIdx.x == 0)
#else
#define QT_DEVICE 0
#define QT_FN inline
#define QT_BIG inline
#define QT_NT 1
#define QT_FOR(i, n) for (int i = 0; i < (n); ++i)
#define QT_SYNC()
#define QT_SINGLE
#include <cmath>
#endif

namespace rgbl {
namespace qt {

constexpr int kMaxNodes = 1024;       // list capacity (needs quota + 3 <= kMaxNodes and 4 * nIni <= kMaxNodes)
constexpr int kMaxRoots = 64;

struct SortItem { int size; int ulx; int node; };

QT_FN bool item_less(const SortItem& a, const SortItem& b) {       // compareNodes, src/ORBextractor.cc:538-553
    if (a.size < b.size) return true;
    if (a.size > b.size) return false;
    return a.ulx < b.ulx;
}

// ---- libstdc++ std::sort, restated (bits/stl_algo.h: __introsort_loop, __final_insertion_sort; bits/stl_heap.h) ----
QT_FN void qs_swap(SortItem* v, int a, int b) { const SortItem t = v[a]; v[a] = v[b]; v[b] = t; }

QT_FN void qs_adjust_heap(SortItem* first, int hole, int len, SortItem value) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (item_less(first[child], first[child - 1])) --child;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    int parent = (hole - 1) / 2;                       // __push_heap
    while (hole > top && item_less(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}

QT_FN void qs_heapsort(SortItem* first, int len) {     // __partial_sort(first, last, last): make_heap + sort_heap
    if (len < 2) return;
    for (int parent = (len - 2) / 2;; --parent) {
        const SortItem v = first[parent];
        qs_adjust_heap(first, parent, len, v);
        if (parent == 0) break;
    }
    for (int last = len; last > 1;) {
        --last;
        const SortItem v = first[last];
        first[last] = first[0];
        qs_adjust_heap(first, 0, last, v);
    }
}

QT_FN void qs_unguarded_linear_insert(SortItem* v, int last) {
    const SortItem val = v[last];
    int next = last - 1;
    while (item_less(val, v[next])) { v[last] = v[next]; last = next; --next; }
    v[last] = val;
}

QT_FN void qs_insertion_sort(SortItem* v, int first, int last) {
    if (first == last) return;
    for (int i = first + 1; i != last; ++i) {
        if (item_less(v[i], v[first])) {
            const SortItem val = v[i];
            for (int k = i; k > first; --k) v[k] = v[k - 1];
            v[first] = val;
        } else {
            qs_unguarded_linear_insert(v, i);
        }
    }
}

QT_BIG void std_sort(SortItem* v, int n) {
    if (n <= 1) return;
    // iterative form of __introsort_loop: an explicit stack of (first, last, depth) for the right-hand recursions
    int stk_first[64], stk_last[64], stk_depth[64], sp = 0;
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg;
    stk_first[0] = 0; stk_last[0] = n; stk_depth[0] = 2 * lg; sp = 1;
    while (sp > 0) {
        --sp;
        int first = stk_first[sp], last = stk_last[sp], depth = stk_depth[sp];
        while (last - first > 16) {
            if (depth == 0) { qs_heapsort(v + first, last - first); break; }
            --depth;
            // __unguarded_partition_pivot
            const int mid = first + (last - first) / 2;
            {   // __move_median_to_first(first, first+1, mid, last-1)
                const int a = first + 1, b = mid, c = last - 1;
                if (item_less(v[a], v[b])) {
                    if (item_less(v[b], v[c])) qs_swap(v, first, b);
                    else if (item_less(v[a], v[c])) qs_swap(v, first, c);
                    else qs_swap(v, first, a);
                } else if (item_less(v[a], v[c])) qs_swap(v, first, a);
                else if (item_less(v[b], v[c])) qs_swap(v, first, c);
                else qs_swap(v, first, b);
            }
            int lo = first + 1, hi = last;
            for (;;) {   // __unguarded_partition(first+1, last, pivot=first)
                while (item_less(v[lo], v[first])) ++lo;
                --hi;
                while (item_less(v[first], v[hi])) --hi;
                if (!(lo < hi)) break;
                qs_swap(v, lo, hi);
                ++lo;
            }
            const int cut = lo;
            // recurse on [cut, last) (the reference recurses first, then loops on [first, cut)): the two ranges
            // are disjoint, so the processing order does not change the result
            stk_first[sp] = cut; stk_last[sp] = last; stk_depth[sp] = depth; ++sp;
            last = cut;
        }
    }
    // __final_insertion_sort
    if (n > 16) {
        qs_insertion_sort(v, 0, 16);
        for (int i = 16; i < n; ++i) qs_unguarded_linear_insert(v, i);
    } else {
        qs_insertion_sort(v, 0, n);
    }
}

// ---- shared-memory state of one tree ------------------------------------------------------------------
// MAXN = node list capacity (needs quota + 3 <= MAXN and 4 * nIni <= MAXN): 1024 in general; 512 when every level of the context fits, which
// halves this state (~56 KB) so that TWO trees are resident per SM - a tree is a chain of barrier-separated phases that leaves the SM idle
// most of the time, and a batch is 8 trees per frame.
template <int MAXN>
struct NodeTableT {
    short ulx[MAXN], uly[MAXN], brx[MAXN], bry[MAXN];
    int beg[MAXN], end[MAXN];
};

template <int MAXN>
struct SharedT {
    static constexpr int kNodes = MAXN;
    NodeTableT<MAXN> tab[2];
    // per node of the current table
    int cc[MAXN][4];          // child key counts of a node that is being divided
    short pushes[MAXN];       // non-empty children (0 if the node is not divided this pass)
    short proc[MAXN];         // processing rank inside D (-1 = not divided)
    int pushbase[MAXN];       // exclusive prefix of pushes in processing order (indexed by processing rank)
    int keepbase[MAXN];       // exclusive prefix of "survives" flags in list order
    short by_rank[MAXN];      // node index by processing rank
    SortItem open[2][MAXN];   // expandable children: [cur] produced by the last pass, [1-cur] being built
    int open_slot[MAXN * 4];  // per push index: position in the next open list, or -1
    int n_nodes, n_open, cur_tab, cur_open, n_div, total_push, n_keep, n_expand, scan_total, flag;
    int root_cnt[kMaxRoots + 1];
    unsigned long long scan_carry[1024 + 32];
};
typedef SharedT<kMaxNodes> Shared;
typedef NodeTableT<kMaxNodes> NodeTable;

// global scratch of one tree (segments of the per-batch arrays)
typedef unsigned short KeyIdx;               // key positions and node indices fit 16 bits (n < 65535 keys, <= 1024 nodes): 17 instead of 25 bytes per key
struct Scratch {
    KeyIdx* perm_a; KeyIdx* perm_b;          // key permutation (ping-pong)
    KeyIdx* node_a; KeyIdx* node_b;          // node index of the key at each position (ping-pong)
    unsigned long long* scan;                // n + 1 packed quadrant counters
    unsigned char* quad;                     // quadrant of the key at each position (4 = not moving)
};

// Exclusive scan of packed counters a[0..n) -> a (exclusive), a[n] = total.  Block-parallel on the device:
// per-thread chunks, warp shuffle scan of the chunk sums, then a scan of the <= 32 warp totals by warp 0.
template <class SharedX>
QT_BIG void scan_u64(unsigned long long* a, int n, SharedX& s) {
#if QT_DEVICE
    const int nt = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int per = (n + nt - 1) / nt;
    const int b = min(tid * per, n), e = min(b + per, n);
    unsigned long long sum = 0;
    for (int i = b; i < e; ++i) sum += a[i];
    unsigned long long incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s.scan_carry[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned long long v = (lane < nw) ? s.scan_carry[lane] : 0ull, w = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
        if (lane < nw) s.scan_carry[lane] = w - v;
        if (lane == nw - 1) a[n] = w;
    }
    __syncthreads();
    unsigned long long run = s.scan_carry[warp] + incl - sum;
    for (int i = b; i < e; ++i) { const unsigned long long v = a[i]; a[i] = run; run += v; }
    __syncthreads();
#else
    unsigned long long run = 0;
    for (int i = 0; i < n; ++i) { const unsigned long long v = a[i]; a[i] = run; run += v; }
    a[n] = run;
    (void)s;
#endif
}

// Exclusive scan of ints in shared memory (n <= 2 * blockDim), total returned through *total (shared).
template <class SharedX>
QT_BIG void scan_int(int* a, int n, int* total, SharedX& s) {
#if QT_DEVICE
    const int nt = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int per = (n + nt - 1) / nt;
    const int b = min(tid * per, n), e = min(b + per, n);
    int sum = 0;
    for (int i = b; i < e; ++i) sum += a[i];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    int* carry = reinterpret_cast<int*>(s.scan_carry);
    if (lane == 31) carry[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int v = (lane < nw) ? carry[lane] : 0, w = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
        if (lane < nw) carry[lane] = w - v;
        if (lane == nw - 1) *total = w;
    }
    __syncthreads();
    int run = carry[warp] + incl - sum;
    for (int i = b; i < e; ++i) { const int v = a[i]; a[i] = run; run += v; }
    __syncthreads();
#else
    int run = 0;
    for (int i = 0; i < n; ++i) { const int v = a[i]; a[i] = run; run += v; }
    *total = run;
    (void)s;
#endif
}

// ---- libstdc++ std::sort, block-parallel --------------------------------------------------------------------------
// Produces exactly what std_sort() above produces (ties included), with the CTA instead of one thread:
//   * __introsort_loop recurses on [cut, last) and loops on [first, cut): the ranges are disjoint, so all segments of one
//     recursion depth can be partitioned at the same time (breadth first);
//   * __unguarded_partition is a pairing: with L_1 < L_2 < ... the positions (ascending) whose value is not less than the
//     pivot and R_1 > R_2 > ... the positions (descending) whose value is not greater, the sequential loop swaps
//     (L_k, R_k) for k = 1..m, m = the number of k with L_k < R_k, and returns cut = min(L_{m+1}, R_m) (the pointers never
//     revisit a swapped position, so the stoppers of the ORIGINAL segment decide).  Ranks come from one block scan of
//     packed flags; the pairs swap in parallel;
//   * __final_insertion_sort is an insertion sort (guarded or not), i.e. a STABLE sort of what the partitions left:
//     computed as a rank sort (rank = smaller-or-equal elements before + smaller elements after);
//   * a segment that exhausts the depth limit (heapsort in the reference; never seen on quad-tree inputs) makes the whole
//     call fall back to the one-thread restatement on the saved input.
// v: n items (shared memory); tmp: n items of scratch; the int scratch comes from fields of `s` that are dead between two
// divide passes.  depth_limit < 0: the reference's 2 * floor(log2 n).
struct SortSeg { short first, last, depth, m; };

template <class SharedX>
QT_BIG void block_std_sort(SharedX& s, SortItem* v, SortItem* tmp, int n, int depth_limit) {
    if (n <= 1) return;
    int* const scanbuf = &s.cc[0][0];                       // n + 1 packed flags / prefixes
    int* const posL = s.pushbase;                           // stoppers by rank, segment-relative slots
    int* const posR = s.keepbase;
    SortSeg* const seg[2] = {reinterpret_cast<SortSeg*>(&s.cc[0][0] + SharedX::kNodes + 8), reinterpret_cast<SortSeg*>(&s.cc[0][0] + SharedX::kNodes + 8) + 128};
    int* const ctl = &s.cc[0][0] + SharedX::kNodes + 8 + 512;     // [0] segments of this level, [1] of the next, [2] fallback flag
    QT_FOR(i, n) tmp[i] = v[i];                             // saved input for the fallback
    QT_SINGLE {
        int lg = 0;
        for (int t = n; t > 1; t >>= 1) ++lg;
        ctl[0] = 0; ctl[1] = 0; ctl[2] = 0;
        if (n > 16) { seg[0][0].first = 0; seg[0][0].last = (short)n; seg[0][0].depth = (short)(depth_limit < 0 ? 2 * lg : depth_limit); ctl[0] = 1; }
    }
    QT_SYNC();
    int cur = 0;
    for (;;) {
        const int ns = ctl[0];
        if (ns == 0 || ctl[2]) break;
        SortSeg* S = seg[cur];
        SortSeg* Nx = seg[cur ^ 1];
        QT_FOR(sg, ns) {                                    // pivot selection: __move_median_to_first(first, first+1, mid, last-1)
            SortSeg& q = S[sg];
            q.m = 0;
            if (q.depth == 0) { ctl[2] = 1; }
            else {
                --q.depth;
                const int first = q.first, a = first + 1, b = first + (q.last - first) / 2, c = q.last - 1;
                if (item_less(v[a], v[b])) {
                    if (item_less(v[b], v[c])) qs_swap(v, first, b);
                    else if (item_less(v[a], v[c])) qs_swap(v, first, c);
                    else qs_swap(v, first, a);
                } else if (item_less(v[a], v[c])) qs_swap(v, first, a);
                else if (item_less(v[b], v[c])) qs_swap(v, first, c);
                else qs_swap(v, first, b);
            }
        }
        QT_SYNC();
        if (ctl[2]) break;
        QT_FOR(i, n) {                                      // stopper flags: low half "not less than the pivot", high half "not greater"
            int f = 0;
            for (int sg = 0; sg < ns; ++sg)
                if (i > S[sg].first && i < S[sg].last) {
                    const SortItem piv = v[S[sg].first];
                    f = (item_less(v[i], piv) ? 0 : 1) | (item_less(piv, v[i]) ? 0 : 0x10000);
                    break;
                }
            scanbuf[i] = f;
        }
        QT_SYNC();
        scan_int(scanbuf, n, &s.scan_total, s);
        QT_SINGLE { scanbuf[n] = s.scan_total; }
        QT_SYNC();
        QT_FOR(i, n) {
            const int e = scanbuf[i], f = scanbuf[i + 1] - e;
            if (f) {
                for (int sg = 0; sg < ns; ++sg)
                    if (i > S[sg].first && i < S[sg].last) {
                        const int base = S[sg].first + 1, e0 = scanbuf[base], e1 = scanbuf[S[sg].last];
                        if (f & 0xffff) posL[base + ((e - e0) & 0xffff)] = i;
                        if (f >> 16) posR[base + ((e1 - e0) >> 16) - 1 - ((e - e0) >> 16)] = i;
                        break;
                    }
            }
        }
        QT_SYNC();
        QT_FOR(i, n) {                                      // pair k of its segment: swap while L_k < R_k
            for (int sg = 0; sg < ns; ++sg)
                if (i > S[sg].first && i < S[sg].last) {
                    const int base = S[sg].first + 1, k = i - base, d = scanbuf[S[sg].last] - scanbuf[base];
                    const int nL = d & 0xffff, nR = d >> 16, np = nL < nR ? nL : nR;
                    if (k < np && posL[base + k] < posR[base + k]) {
                        qs_swap(v, posL[base + k], posR[base + k]);
                        if (k + 1 >= np || !(posL[base + k + 1] < posR[base + k + 1])) S[sg].m = (short)(k + 1);
                    }
                    break;
                }
        }
        QT_SYNC();
        QT_FOR(sg, ns) {                                    // cut = min(L_{m+1}, R_m); children longer than 16 go to the next level
            const SortSeg q = S[sg];
            const int base = q.first + 1, d = scanbuf[q.last] - scanbuf[base], nL = d & 0xffff, m = q.m;
            int cut = q.last;
            if (m > 0) cut = posR[base + m - 1];
            if (m < nL && posL[base + m] < cut) cut = posL[base + m];
            for (int h = 0; h < 2; ++h) {
                const int f = h ? q.first : cut, l = h ? cut : q.last;
                if (l - f > 16) {
#if QT_DEVICE
                    const int slot = atomicAdd(&ctl[1], 1);
#else
                    const int slot = ctl[1]++;
#endif
                    Nx[slot].first = (short)f; Nx[slot].last = (short)l; Nx[slot].depth = q.depth; Nx[slot].m = 0;
                }
            }
        }
        QT_SYNC();
        QT_SINGLE { ctl[0] = ctl[1]; ctl[1] = 0; }
        QT_SYNC();
        cur ^= 1;
    }
    if (ctl[2]) {                                           // depth limit reached somewhere: the reference heap-sorts that segment
        QT_SYNC();
        QT_FOR(i, n) v[i] = tmp[i];
        QT_SYNC();
        QT_SINGLE { std_sort(v, n); }
        QT_SYNC();
        return;
    }
    QT_FOR(i, n) {                                          // __final_insertion_sort == stable sort of the current order
        const SortItem x = v[i];
        int r = 0;
        for (int j = 0; j < i; ++j) r += item_less(x, v[j]) ? 0 : 1;
        for (int j = i + 1; j < n; ++j) r += item_less(v[j], x) ? 1 : 0;
        tmp[r] = x;
    }
    QT_SYNC();
    QT_FOR(i, n) v[i] = tmp[i];
    QT_SYNC();
}

QT_FN int cand_x(unsigned int c) { return (int)(c & 0xfffu); }
QT_FN int cand_y(unsigned int c) { return (int)((c >> 12) & 0xfffu); }
QT_FN int cand_s(unsigned int c) { return (int)(c >> 24); }

// Divide the nodes marked in s.proc (processing rank >= 0, s.n_div of them, s.by_rank filled) and rebuild the list.
// On exit: s.cur_tab flipped, s.n_nodes updated, s.open[1-cur_open] holds the new expandable children in push
// order and s.cur_open is flipped; perm/node arrays flipped by the caller-visible flag `pp` (returns new value).
template <class SharedX>
QT_BIG int divide_pass(SharedX& s, const unsigned int* cand, int n, Scratch g, int pp) {
    auto& T = s.tab[s.cur_tab];
    auto& U = s.tab[1 - s.cur_tab];
    KeyIdx* perm = pp ? g.perm_b : g.perm_a;
    KeyIdx* perm2 = pp ? g.perm_a : g.perm_b;
    KeyIdx* nod = pp ? g.node_b : g.node_a;
    KeyIdx* nod2 = pp ? g.node_a : g.node_b;
    const int nn = s.n_nodes;

    // quadrant of every key that belongs to a divided node
    QT_FOR(p, n) {
        const int nd = nod[p];
        unsigned long long v = 0;
        unsigned char q = 4;
        if (s.proc[nd] >= 0) {
            const int hx = (T.brx[nd] - T.ulx[nd] + 1) >> 1;           // ceil(float(w)/2) for w >= 0
            const int hy = (T.bry[nd] - T.uly[nd] + 1) >> 1;
            const int mx = T.ulx[nd] + hx, my = T.uly[nd] + hy;
            const unsigned int c = cand[perm[p]];
            q = (unsigned char)((cand_x(c) < mx) ? ((cand_y(c) < my) ? 0 : 2) : ((cand_y(c) < my) ? 1 : 3));
            v = 1ull << (16 * q);
        }
        g.quad[p] = q;
        g.scan[p] = v;
    }
    QT_SYNC();
    scan_u64(g.scan, n, s);
    QT_SYNC();
    // child counts and number of pushes per divided node
    QT_FOR(i, nn) {
        int k = 0;
        if (s.proc[i] >= 0) {
            const unsigned long long d = g.scan[T.end[i]] - g.scan[T.beg[i]];
            for (int q = 0; q < 4; ++q) { const int c = (int)((d >> (16 * q)) & 0xffffu); s.cc[i][q] = c; k += (c > 0); }
        }
        s.pushes[i] = (short)k;
    }
    QT_SYNC();
    // prefix of pushes in processing order, prefix of survivors in list order (block scans)
    QT_FOR(r, s.n_div) s.pushbase[r] = s.pushes[s.by_rank[r]];
    QT_FOR(i, nn) s.keepbase[i] = (s.proc[i] < 0) ? 1 : 0;
    QT_SYNC();
    scan_int(s.pushbase, s.n_div, &s.total_push, s);
    QT_SYNC();
    scan_int(s.keepbase, nn, &s.n_keep, s);
    QT_SYNC();
    const int total_push = s.total_push;
    // new node table: children (reverse push order) then survivors
    QT_FOR(i, nn) {
        if (s.proc[i] < 0) {
            const int j = total_push + s.keepbase[i];
            U.ulx[j] = T.ulx[i]; U.uly[j] = T.uly[i]; U.brx[j] = T.brx[i]; U.bry[j] = T.bry[i];
            U.beg[j] = T.beg[i]; U.end[j] = T.end[i];
        } else {
            const int hx = (T.brx[i] - T.ulx[i] + 1) >> 1, hy = (T.bry[i] - T.uly[i] + 1) >> 1;
            const int mx = T.ulx[i] + hx, my = T.uly[i] + hy;
            const int x0[4] = {T.ulx[i], mx, T.ulx[i], mx}, y0[4] = {T.uly[i], T.uly[i], my, my};
            const int x1[4] = {mx, T.brx[i], mx, T.brx[i]}, y1[4] = {my, my, T.bry[i], T.bry[i]};
            int push = s.pushbase[s.proc[i]], start = T.beg[i];
            for (int q = 0; q < 4; ++q) {
                const int c = s.cc[i][q];
                if (c == 0) continue;
                const int j = total_push - 1 - push;
                U.ulx[j] = (short)x0[q]; U.uly[j] = (short)y0[q]; U.brx[j] = (short)x1[q]; U.bry[j] = (short)y1[q];
                U.beg[j] = start; U.end[j] = start + c;
                s.open_slot[push] = (c > 1) ? 1 : 0;
                start += c;
                ++push;
            }
        }
    }
    QT_SYNC();
    // expandable children in push order -> next open list (compaction through a scan of the flags)
    scan_int(s.open_slot, total_push, &s.n_expand, s);
    QT_SYNC();
    {
        SortItem* o = s.open[1 - s.cur_open];
        QT_FOR(push, total_push) {
            const int nxt = (push + 1 < total_push) ? s.open_slot[push + 1] : s.n_expand;
            if (nxt != s.open_slot[push]) {
                const int j = total_push - 1 - push, m = s.open_slot[push];
                o[m].size = U.end[j] - U.beg[j]; o[m].ulx = U.ulx[j]; o[m].node = j;
            }
        }
    }
    // move the keys: stable 4-way partition inside every divided segment; everything else keeps its place
    QT_FOR(p, n) {
        const int nd = nod[p];
        int np = p, nj;
        if (s.proc[nd] < 0) {
            nj = total_push + s.keepbase[nd];
        } else {
            const int q = g.quad[p], b = T.beg[nd];
            int before = 0, rankq = 0;
            for (int qq = 0; qq < q; ++qq) before += s.cc[nd][qq];
            int nonempty_before = 0;
            for (int qq = 0; qq < q; ++qq) nonempty_before += (s.cc[nd][qq] > 0);
            rankq = (int)(((g.scan[p] - g.scan[b]) >> (16 * q)) & 0xffffu);
            np = b + before + rankq;
            nj = total_push - 1 - (s.pushbase[s.proc[nd]] + nonempty_before);
        }
        perm2[np] = perm[p];
        nod2[np] = nj;
    }
    QT_SYNC();
    QT_SINGLE {
        s.n_nodes = total_push + s.n_keep;
        s.cur_tab = 1 - s.cur_tab;
        s.cur_open = 1 - s.cur_open;
        s.n_open = s.n_expand;
    }
    QT_SYNC();
    return 1 - pp;
}

// Whole DistributeOctTree.  cand: n packed candidates (x, y relative to (minX, minY), reference order).
// out: packed candidates of the survivors in the reference's output order.  Returns the count (or -1 if the
// configuration exceeds the on-chip capacities; the caller then uses the host implementation).
template <class SharedX>
QT_FN int distribute(SharedX& s, const unsigned int* cand, int n, int width, int height, int N, Scratch g,
                     unsigned int* out, int out_cap) {
    if (n <= 0) return 0;
#if QT_DEVICE
    const int n_ini = (int)roundf(static_cast<float>(width) / height);
#else
    const int n_ini = (int)std::round(static_cast<float>(width) / height);
#endif
    if (n_ini < 1 || n_ini > kMaxRoots || 4 * n_ini > SharedX::kNodes || N + 3 > SharedX::kNodes || n >= 65535) return -1;
    const float hX = static_cast<float>(width) / n_ini;

    // ---- roots: stable bucket of the candidates by root index ----
    QT_FOR(r, n_ini + 1) s.root_cnt[r] = 0;
    QT_SYNC();
    int pp = 0;
    // one stable pass per root (n_ini is tiny): positions from a scan of the membership flags
    QT_SINGLE { s.flag = 0; }
    QT_SYNC();
    for (int r = 0; r < n_ini; ++r) {
        QT_FOR(p, n) {
            int rr = (int)(static_cast<float>(cand_x(cand[p])) / hX);
            if (rr >= n_ini) rr = n_ini - 1;
            g.scan[p] = (rr == r) ? 1ull : 0ull;
        }
        QT_SYNC();
        scan_u64(g.scan, n, s);
        QT_SYNC();
        const int base = s.flag;
        QT_FOR(p, n) {
            int rr = (int)(static_cast<float>(cand_x(cand[p])) / hX);
            if (rr >= n_ini) rr = n_ini - 1;
            if (rr == r) g.perm_a[base + (int)g.scan[p]] = p;
        }
        QT_SYNC();
        QT_SINGLE { s.root_cnt[r] = (int)g.scan[n]; s.flag = base + (int)g.scan[n]; }
        QT_SYNC();
    }
    QT_SINGLE {
        auto& T = s.tab[0];
        int m = 0, start = 0;
        for (int r = 0; r < n_ini; ++r) {
            const int c = s.root_cnt[r];
            if (c > 0) {
                T.ulx[m] = (short)(int)(hX * static_cast<float>(r)); T.uly[m] = 0;
                T.brx[m] = (short)(int)(hX * static_cast<float>(r + 1)); T.bry[m] = (short)height;
                T.beg[m] = start; T.end[m] = start + c;
                ++m;
            }
            start += c;
        }
        s.n_nodes = m; s.cur_tab = 0; s.cur_open = 0; s.n_open = 0;
    }
    QT_SYNC();
    {
        const auto& T = s.tab[0];
        const int m = s.n_nodes;
        QT_FOR(i, m) { for (int p = T.beg[i]; p < T.end[i]; ++p) g.node_a[p] = i; }
    }
    QT_SYNC();

    // ---- subdivision loop (src/ORBextractor.cc:609-755) ----
    for (;;) {
        const int prev = s.n_nodes;
        {   // full pass: D = every node with more than one key, processed in list order (ranks from a block scan of the flags)
            const auto& T = s.tab[s.cur_tab];
            QT_FOR(i, prev) s.pushbase[i] = (T.end[i] - T.beg[i] > 1) ? 1 : 0;
            QT_SYNC();
            scan_int(s.pushbase, prev, &s.n_div, s);
            QT_SYNC();
            QT_FOR(i, prev) {
                if (T.end[i] - T.beg[i] > 1) { const int r = s.pushbase[i]; s.proc[i] = (short)r; s.by_rank[r] = (short)i; }
                else s.proc[i] = -1;
            }
            QT_SYNC();
        }
        pp = divide_pass(s, cand, n, g, pp);
        const int size = s.n_nodes, n_expand = s.n_open;
        if (size >= N || size == prev) break;
        if (size + n_expand * 3 > N) {
            // budgeted expansion: biggest nodes first, stop as soon as the list holds N nodes
            bool done = false;
            while (!done) {
                const int prev2 = s.n_nodes;
                const int n_open = s.n_open;
                block_std_sort(s, s.open[s.cur_open], s.open[s.cur_open ^ 1], n_open, -1);
                QT_SYNC();
                // child counts of every open node (they are all candidates for division)
                {
                    const auto& T = s.tab[s.cur_tab];
                    QT_FOR(i, prev2) s.proc[i] = -1;
                    QT_SYNC();
                    QT_FOR(k, n_open) { const int r = n_open - 1 - k; s.proc[s.open[s.cur_open][k].node] = (short)r; s.by_rank[r] = (short)s.open[s.cur_open][k].node; }
                    QT_SYNC();
                    // count non-empty children per open node with a direct scan of its (small) key segment
                    KeyIdx* perm = pp ? g.perm_b : g.perm_a;
                    QT_FOR(r, n_open) {
                        const int nd = s.by_rank[r];
                        const int hx = (T.brx[nd] - T.ulx[nd] + 1) >> 1, hy = (T.bry[nd] - T.uly[nd] + 1) >> 1;
                        const int mx = T.ulx[nd] + hx, my = T.uly[nd] + hy;
                        int mask = 0;
                        for (int p = T.beg[nd]; p < T.end[nd]; ++p) {
                            const unsigned int c = cand[perm[p]];
                            mask |= 1 << ((cand_x(c) < mx) ? ((cand_y(c) < my) ? 0 : 2) : ((cand_y(c) < my) ? 1 : 3));
                        }
                        s.pushes[nd] = (short)(((mask >> 0) & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1) + ((mask >> 3) & 1));
                    }
                    QT_SYNC();
                    // the list grows by pushes - 1 >= 0 per division: the sequential loop stops after the first rank
                    // whose running size reaches N, i.e. m = 1 + #{r : size after r < N} (capped at n_open)
                    QT_FOR(r, n_open) s.keepbase[r] = s.pushes[s.by_rank[r]] - 1;
                    QT_SINGLE { s.n_div = 0; }
                    QT_SYNC();
                    scan_int(s.keepbase, n_open, &s.scan_total, s);
                    QT_SYNC();
                    QT_FOR(r, n_open) {
                        const int incl = prev2 + ((r + 1 < n_open) ? s.keepbase[r + 1] : s.scan_total);
                        const int incl_next = (r + 1 < n_open) ? prev2 + ((r + 2 < n_open) ? s.keepbase[r + 2] : s.scan_total) : N;
                        if (r == 0 && incl >= N) s.n_div = 1;
                        if (incl < N && incl_next >= N) s.n_div = (r + 2 < n_open) ? r + 2 : n_open;
                    }
                    QT_SYNC();
                    {   // nodes beyond the stopping rank are not divided in this iteration
                        const int m = s.n_div;
                        QT_FOR(r, n_open) if (r >= m) s.proc[s.by_rank[r]] = -1;
                    }
                    QT_SYNC();
                }
                pp = divide_pass(s, cand, n, g, pp);
                if (s.n_nodes >= N || s.n_nodes == prev2) done = true;
            }
            break;
        }
    }

    // ---- best key per node, in list order (src/ORBextractor.cc:757-776) ----
    {
        const auto& T = s.tab[s.cur_tab];
        const KeyIdx* perm = pp ? g.perm_b : g.perm_a;
        const int m = s.n_nodes;
        QT_FOR(i, m) {
            unsigned int best = cand[perm[T.beg[i]]];
            for (int p = T.beg[i] + 1; p < T.end[i]; ++p) {
                const unsigned int c = cand[perm[p]];
                if (cand_s(c) > cand_s(best)) best = c;
            }
            if (i < out_cap) out[i] = best;
        }
        QT_SYNC();
        return m;
    }
}

}  // namespace qt
}  // namespace rgbl
#endif
