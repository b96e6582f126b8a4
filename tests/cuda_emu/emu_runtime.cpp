// TEST INFRASTRUCTURE: thread-per-CUDA-thread execution of one CTA (or one thread-block cluster) at a time (see cuda_runtime.h in this
// directory).
#include "cuda_runtime.h"

thread_local uint3 threadIdx;
thread_local uint3 blockIdx;
dim3 blockDim, gridDim;
namespace emu {
// CUDA graphs are not emulated (cuda_runtime.h): make the library replay its tracking chain launch by launch
static const int g_no_graphs = setenv("RGBL_CHAIN_GRAPH", "0", 1);
thread_local Cta* g_cta = nullptr;
static int g_fail_countdown = -1;          // allocations happen on the host thread only
bool allocation_fails() {
    if (g_fail_countdown < 0 || --g_fail_countdown > 0) return false;
    g_fail_countdown = -1;
    return true;
}
thread_local int t_warp = 0, t_lane = 0;
thread_local Cluster* t_cluster = nullptr;
thread_local unsigned t_rank = 0;
alignas(64) unsigned char g_window[kMaxClusterCtas][kCtaWindow];
std::mutex g_mbar_mu;
std::condition_variable g_mbar_cv;
static unsigned g_next_cluster = 0;        // launches happen on the host thread only
void next_launch_cluster(unsigned n) { g_next_cluster = n; }

size_t window_reserve(size_t size, size_t align) {
    static std::mutex mu;
    static size_t top = 0;
    std::lock_guard<std::mutex> lk(mu);
    const size_t off = (top + align - 1) / align * align;
    if (off + size > kCtaWindow) fail("the shared variables of a cluster kernel exceed the emulated window");
    top = off + size;
    return off;
}

void run(const Cfg& c, const std::function<void()>& body) {
    const unsigned cs = g_next_cluster ? g_next_cluster : 1;
    g_next_cluster = 0;
    if (cs > kMaxClusterCtas || c.grid.x % cs) fail("cluster size does not divide the grid (or exceeds 16)");
    gridDim = c.grid; blockDim = c.block;
    const int nt = (int)(c.block.x * c.block.y * c.block.z), nw = (nt + 31) / 32;
    for (unsigned bz = 0; bz < c.grid.z; ++bz)
        for (unsigned by = 0; by < c.grid.y; ++by)
            for (unsigned bx0 = 0; bx0 < c.grid.x; bx0 += cs) {
                if (cs > 1) std::memset(g_window, 0, cs * kCtaWindow);      // a missing mbarrier.init then fails (count == 0), not a stale word
                Cluster cl;
                cl.size = cs;
                cl.bar = std::make_unique<std::barrier<>>((std::ptrdiff_t)cs * nt);
                std::vector<std::unique_ptr<Cta>> ctas;
                for (unsigned r = 0; r < cs; ++r) {
                    auto cta = std::make_unique<Cta>();
                    cta->bar = std::make_unique<std::barrier<>>(nt);
                    cta->slot.resize(nw);
                    for (int w = 0; w < nw; ++w) cta->warp_bar.push_back(std::make_unique<std::barrier<>>(std::min(32, nt - 32 * w)));
                    ctas.push_back(std::move(cta));
                }
                std::vector<std::thread> th;
                th.reserve((size_t)cs * nt);
                for (unsigned r = 0; r < cs; ++r)
                    for (int t = 0; t < nt; ++t)
                        th.emplace_back([&, r, t] {
                            Cta& cta = *ctas[r];
                            g_cta = &cta; t_cluster = &cl; t_rank = r;
                            blockIdx = uint3{bx0 + r, by, bz};
                            threadIdx = uint3{(unsigned)(t % c.block.x), (unsigned)((t / c.block.x) % c.block.y), (unsigned)(t / (c.block.x * c.block.y))};
                            t_warp = t / 32; t_lane = t % 32;
                            body();
                            cta.warp_bar[t_warp]->arrive_and_drop();     // a thread that has left the kernel no longer takes part
                            cta.bar->arrive_and_drop();
                            cl.bar->arrive_and_drop();
                            g_cta = nullptr; t_cluster = nullptr; t_rank = 0;
                        });
                for (auto& x : th) x.join();
            }
}
}  // namespace emu

extern "C" int emu_fail_allocation(int nth) {
    const int prev = emu::g_fail_countdown;
    emu::g_fail_countdown = nth;
    return prev;
}
