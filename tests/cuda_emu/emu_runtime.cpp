// TEST INFRASTRUCTURE: thread-per-CUDA-thread execution of one CTA at a time (see cuda_runtime.h in this directory).
#include "cuda_runtime.h"

thread_local uint3 threadIdx;
uint3 blockIdx;
dim3 blockDim, gridDim;
namespace emu {
// CUDA graphs are not emulated (cuda_runtime.h): make the library replay its tracking chain launch by launch
static const int g_no_graphs = setenv("RGBL_CHAIN_GRAPH", "0", 1);
Cta* g_cta = nullptr;
static int g_fail_countdown = -1;          // allocations happen on the host thread only
bool allocation_fails() {
    if (g_fail_countdown < 0 || --g_fail_countdown > 0) return false;
    g_fail_countdown = -1;
    return true;
}
thread_local int t_warp = 0, t_lane = 0;

void run(const Cfg& c, const std::function<void()>& body) {
    gridDim = c.grid; blockDim = c.block;
    const int nt = (int)(c.block.x * c.block.y * c.block.z), nw = (nt + 31) / 32;
    for (unsigned bz = 0; bz < c.grid.z; ++bz)
        for (unsigned by = 0; by < c.grid.y; ++by)
            for (unsigned bx = 0; bx < c.grid.x; ++bx) {
                blockIdx = uint3{bx, by, bz};
                Cta cta;
                cta.bar = std::make_unique<std::barrier<>>(nt);
                cta.slot.resize(nw);
                for (int w = 0; w < nw; ++w) cta.warp_bar.push_back(std::make_unique<std::barrier<>>(std::min(32, nt - 32 * w)));
                g_cta = &cta;
                std::vector<std::thread> th;
                th.reserve(nt);
                for (int t = 0; t < nt; ++t)
                    th.emplace_back([&, t] {
                        threadIdx = uint3{(unsigned)(t % c.block.x), (unsigned)((t / c.block.x) % c.block.y), (unsigned)(t / (c.block.x * c.block.y))};
                        t_warp = t / 32; t_lane = t % 32;
                        body();
                        cta.warp_bar[t_warp]->arrive_and_drop();     // a thread that has left the kernel no longer takes part
                        cta.bar->arrive_and_drop();
                    });
                for (auto& x : th) x.join();
                g_cta = nullptr;
            }
}
}  // namespace emu

extern "C" int emu_fail_allocation(int nth) {
    const int prev = emu::g_fail_countdown;
    emu::g_fail_countdown = nth;
    return prev;
}
