// TEST INFRASTRUCTURE: runs the multi-CTA TrackLocalMap glue kernel of chain_kernels.cu (tlm_prepare: ordered compaction by "publish and look
// back") on the CUDA-on-CPU shim and compares them with a serial restatement that walks the same arrays in index order.
// A unit of the emulated library (tests/cuda_emu/build.py); tests/test_cuda_emu.py::test_tlm_kernels_device_path calls it.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

using namespace rgbl;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails < 20) { std::printf("FAIL %s:%d: ", __FILE__, __LINE__); std::printf(__VA_ARGS__); std::printf("\n"); } ++fails; } } while (0)

// one random frame, pose and ring from `seed`; returns the number of mismatches (0 = identical)
extern "C" int emu_tlm_check(unsigned seed) {
    fails = 0;
    std::mt19937 rng(seed);
    std::uniform_real_distribution<float> U(0.f, 1.f);
    const int K = 3, cap = 700 + (int)(seed % 5) * 97;        // not a multiple of the CTA size
    const int n_ring = K * cap, n_f = cap - 13;
    // frame + pose
    FrameDev f{};
    int n_f_dev = n_f;
    std::vector<rgbl_keypoint> keys(cap);
    std::vector<float> uright(cap);
    for (int i = 0; i < cap; ++i) { keys[i] = rgbl_keypoint{U(rng) * 1241.f, U(rng) * 376.f, 31.f, U(rng) * 360.f, 20.f, (int)(U(rng) * 8) & 7, -1}; uright[i] = U(rng) < 0.4f ? -1.f : keys[i].x - 30.f * U(rng); }
    f.n = &n_f_dev; f.keys = keys.data(); f.uright = uright.data(); f.desc = nullptr;
    f.min_x = 0; f.max_x = 1241; f.min_y = 0; f.max_y = 376; f.inv_w = 64.f / 1241.f; f.inv_h = 48.f / 376.f; f.n_levels = 8;
    f.scale[0] = 1.f; for (int l = 1; l < 8; ++l) f.scale[l] = f.scale[l - 1] * 1.2f;
    f.fx = 718.856f; f.fy = 718.856f; f.cx = 607.19f; f.cy = 185.2f; f.bf = 386.1f; f.mb = f.bf / f.fx; f.log_scale_factor = std::log(1.2f);
    float pose[7] = {0.01f, -0.02f, 0.005f, 0.f, -0.3f, 0.05f, 0.1f};
    pose[3] = std::sqrt(1.f - pose[0] * pose[0] - pose[1] * pose[1] - pose[2] * pose[2]);
    // ring
    std::vector<uint8_t> r_valid(n_ring), r_desc((size_t)n_ring * 32);
    std::vector<float> r_xw(3 * n_ring), r_normal(3 * n_ring), r_min(n_ring), r_max(n_ring);
    for (int p = 0; p < n_ring; ++p) {
        r_valid[p] = U(rng) < 0.8f;
        const float z = 5.f + 40.f * U(rng);
        r_xw[3 * p] = (U(rng) * 1.6f - 0.8f) * z * 1.2f; r_xw[3 * p + 1] = (U(rng) * 0.6f - 0.3f) * z * 1.2f; r_xw[3 * p + 2] = z * (U(rng) < 0.05f ? -1.f : 1.f);
        float n[3] = {r_xw[3 * p] + 0.3f, r_xw[3 * p + 1], r_xw[3 * p + 2]};
        const float nn = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        for (int k = 0; k < 3; ++k) r_normal[3 * p + k] = (U(rng) < 0.1f ? -1.f : 1.f) * n[k] / nn;
        r_max[p] = nn * (0.7f + U(rng)); r_min[p] = r_max[p] / 3.58f;
        for (int k = 0; k < 32; ++k) r_desc[(size_t)p * 32 + k] = (uint8_t)(rng() & 0xff);
    }
    int ring_count = 7;
    LocalRingDev ring{K, cap, r_valid.data(), r_xw.data(), r_normal.data(), r_min.data(), r_max.data(), r_desc.data(), &ring_count};
    // first search + pose result
    std::vector<int> match_last(cap, -1), e_idx;
    std::vector<uint8_t> e_out, state(cap, 7);
    for (int i = 0; i < n_f; ++i) if (U(rng) < 0.3f) { match_last[i] = (int)(U(rng) * cap) % cap; e_idx.push_back(i); e_out.push_back(U(rng) < 0.2f); }
    int n_edges = (int)e_idx.size();
    const std::vector<int> match_last0 = match_last;
    // outputs of prepare
    const int n_lq = n_ring;
    std::vector<uint8_t> lq_u8(2 * n_lq, 0), lq_desc((size_t)n_lq * 32, 0);
    std::vector<float> lq_f(8 * (size_t)n_lq, -7.f);
    std::vector<int> lq_i(2 * (size_t)n_lq, -7);
    int nq = -1, fail = 0;
    LocalQueriesDev lq{};
    lq.cap = n_lq; lq.n = &nq; lq.in_view = lq_u8.data(); lq.obs_pos = lq_u8.data() + n_lq;
    lq.proj_x = lq_f.data(); lq.proj_y = lq_f.data() + n_lq; lq.proj_xr = lq_f.data() + 2 * (size_t)n_lq; lq.depth = lq_f.data() + 3 * (size_t)n_lq;
    lq.view_cos = lq_f.data() + 4 * (size_t)n_lq; lq.xw = lq_f.data() + 5 * (size_t)n_lq; lq.level = lq_i.data(); lq.src = lq_i.data() + n_lq; lq.desc = lq_desc.data();
    std::vector<int> lookback(tlm_lookback_ints(), 0);
    for (int rep = 0; rep < 2; ++rep) {          // twice: the slot arrays must be clean again after a launch
        match_last = match_last0;
        launch_tlm_prepare(nullptr, f, pose, ring, 0.5f, &n_edges, e_idx.data(), e_out.data(), state.data(), match_last.data(), lq, lookback.data(), &fail);
        CHECK(fail == 0, "fail flag %d", fail);
        for (int v : lookback) CHECK(v == 0, "lookback slots not clean after tlm_prepare");
        // serial restatement
        FrustumParams prm{};
        quatf_to_matrix(pose, prm.Rcw);
        float qinv[4]; se3f_inverse(pose, qinv, prm.Ow);
        prm.tcw[0] = pose[4]; prm.tcw[1] = pose[5]; prm.tcw[2] = pose[6]; prm.cos_limit = 0.5f;
        int pos = 0;
        for (int p = 0; p < n_ring; ++p) {
            if (!r_valid[p]) continue;
            const FrustumOut o = frustum_point(f, prm, &r_xw[3 * p], &r_normal[3 * p], r_min[p], r_max[p]);
            if (!o.in_view) continue;
            CHECK(lq.src[pos] == p, "src[%d] = %d, expected %d", pos, lq.src[pos], p);
            CHECK(lq.proj_x[pos] == o.px && lq.proj_y[pos] == o.py && lq.proj_xr[pos] == o.pxr && lq.depth[pos] == o.depth && lq.view_cos[pos] == o.view_cos && lq.level[pos] == o.level,
                  "fields of query %d", pos);
            CHECK(lq.in_view[pos] == 1 && lq.obs_pos[pos] == 1, "flags of query %d", pos);
            CHECK(lq.xw[3 * pos] == r_xw[3 * p] && lq.xw[3 * pos + 1] == r_xw[3 * p + 1] && lq.xw[3 * pos + 2] == r_xw[3 * p + 2], "xw of query %d", pos);
            CHECK(std::memcmp(&lq_desc[(size_t)pos * 32], &r_desc[(size_t)p * 32], 32) == 0, "descriptor of query %d", pos);
            ++pos;
        }
        CHECK(nq == pos, "n queries %d, expected %d", nq, pos);
        std::vector<int> ml = match_last0;
        std::vector<uint8_t> st_ref(cap, 7);
        for (int i = 0; i < n_f; ++i) st_ref[i] = ml[i] >= 0 ? 1 : 0;
        for (int e = 0; e < n_edges; ++e) if (e_out[e]) { st_ref[e_idx[e]] = 0; ml[e_idx[e]] = -1; }
        for (int i = 0; i < cap; ++i) { CHECK(state[i] == st_ref[i], "state[%d]", i); CHECK(match_last[i] == ml[i], "match_last[%d]", i); }
    }
    std::printf("tlm_prepare: %d queries of %d ring points, %d mismatches\n", nq, n_ring, fails);
    std::fflush(stdout);
    return fails;
}
