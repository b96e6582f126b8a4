// Optimizer::PoseOptimization (src/Optimizer.cc:814-1114) as ONE thread-block CLUSTER of 16 CTAs (16 SMs) per frame: the whole
// 4 x (<= 10 Levenberg-Marquardt iterations x <= 10 trials) schedule of g2o runs on the device in FP64 with no host round trip.
// The ~500-800 edges of a frame are strided over the 16 x 64 threads of the cluster (one pass; the per-edge Jacobian / J^T W J work
// is bound by the FP64 issue rate of an SM, so sixteen SMs cut it sixteen ways).  J^T W J (21 unique entries), J^T W r (6) and the robust
// chi2 are reduced inside each CTA with warp shuffles + a fixed shared-memory tree, the partial sums of the CTAs are exchanged through
// distributed shared memory (each CTA pushes its sums into every CTA's exchange slot with st.async, no cluster barrier) and added in
// rank order by every CTA, so all of them hold bit-identical systems and take the LM decisions redundantly: no broadcast.  One exchange
// per evaluated trial: the pass that evaluates a trial also builds the system at the trial's pose, which is the next iteration's
// system when the trial is accepted, and the classification pass at the end of a round builds the next round's first system.  In each
// CTA, lane 0 of warp w solves the damped 6x6 system of trial w (LDL^T), applies the SE3 exponential update.
// g2o semantics reproduced (Thirdparty/g2o/g2o/: core/optimization_algorithm_levenberg.cpp:61-185,
// core/base_unary_edge.hpp:43-72, core/robust_kernel_impl.cpp:65-91, types/se3quat.h:104-110,214-254,280-285,
// types/types_six_dof_expmap.cpp:339-404; src/OptimizableTypes.cpp:49-63):
//   * update T <- exp(delta) * T, delta = (omega, upsilon); quaternion normalised with w >= 0;
//   * H += rho' J^T Omega J, b -= rho' J^T Omega e (no second-order Huber term); Huber dsqr is a float;
//   * stereo edge: float invz in cam_project, double Jacobian; mono edge: -projectJac * SE3deriv;
//   * lambda0 = 1e-5 * max diag(H) at iteration 0 of every round; rho test; nu doubling; <= 10 trials;
//     stop when (ini - cur) * 1e3 < ini three times in a row;
//   * every round restarts from the frame's initial pose; inlier edges are classified with the error of
//     the LAST evaluated trial (g2o does not recompute it), outlier edges are recomputed.
// A round that would repeat the previous one bit for bit (no level changed, and the same robust flag or no Huber linear-region
// evaluation) is not run: its estimate, errors and classification are already in place (end of the round loop).
#include <atomic>
#include <cfloat>
#include <string>
#include <cooperative_groups.h>

#include "rgbl_device.cuh"
#include "rgbl_kernels.h"

namespace rgbl {

namespace cg = cooperative_groups;

namespace {

struct Se3d { double qx, qy, qz, qw, tx, ty, tz; };

// SE3Quat::normalizeRotation (se3quat.h:280-285).  A product of unit quaternions has |q|^2 = 1 + d with |d| ~ 1e-16, where
// 1/sqrt(1 + d) = 1 - d/2 to far below one ulp: one FMA instead of an rsqrt on the serial FP64 chain; anything farther
// from unit norm (the caller's initial pose) takes the general path.
__device__ __forceinline__ void normalize_rotation(Se3d& T) {
    if (T.qw < 0) { T.qx *= -1; T.qy *= -1; T.qz *= -1; T.qw *= -1; }
    const double n2 = T.qx * T.qx + T.qy * T.qy + T.qz * T.qz + T.qw * T.qw;
    const double inv = (fabs(n2 - 1.0) < 1e-7) ? 1.5 - 0.5 * n2 : rsqrt(n2);
    T.qx *= inv; T.qy *= inv; T.qz *= inv; T.qw *= inv;
}

__device__ __forceinline__ void quat_rotate(const Se3d& q, const double v[3], double out[3]) {
    double uv[3] = {q.qy * v[2] - q.qz * v[1], q.qz * v[0] - q.qx * v[2], q.qx * v[1] - q.qy * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    const double c[3] = {q.qy * uv[2] - q.qz * uv[1], q.qz * uv[0] - q.qx * uv[2], q.qx * uv[1] - q.qy * uv[0]};
    out[0] = v[0] + q.qw * uv[0] + c[0]; out[1] = v[1] + q.qw * uv[1] + c[1]; out[2] = v[2] + q.qw * uv[2] + c[2];
}

__device__ __forceinline__ void se3_map(const Se3d& T, const double p[3], double out[3]) {
    quat_rotate(T, p, out);
    out[0] += T.tx; out[1] += T.ty; out[2] += T.tz;
}

// Taylor coefficients in th^2 (k = 0..8), generated from exact rationals: sin(th/2)/th, cos(th/2), (1-cos th)/th^2, (th-sin th)/th^3
__device__ constexpr double kQs[9] = {0.5, -0.020833333333333332, 0.00026041666666666666, -1.5500992063492063e-06, 5.382288910934745e-09, -1.2232474797578965e-11, 1.9603324996120133e-14, -2.333729166204778e-17, 2.1449716601146855e-20};   // (-1)^k / (2 4^k (2k+1)!)
__device__ constexpr double kQc[9] = {1.0, -0.125, 0.0026041666666666665, -2.170138888888889e-05, 9.68812003968254e-08, -2.691144455467372e-10, 5.096864498991235e-13, -7.001187498614334e-16, 7.292903644389931e-19};   // (-1)^k / (4^k (2k)!)
__device__ constexpr double kB[9] = {0.5, -0.041666666666666664, 0.001388888888888889, -2.48015873015873e-05, 2.755731922398589e-07, -2.08767569878681e-09, 1.1470745597729725e-11, -4.779477332387385e-14, 1.5619206968586225e-16};   // (-1)^k / (2k+2)!
__device__ constexpr double kC[9] = {0.16666666666666666, -0.008333333333333333, 0.0001984126984126984, -2.7557319223985893e-06, 2.505210838544172e-08, -1.6059043836821613e-10, 7.647163731819816e-13, -2.8114572543455206e-15, 8.22063524662433e-18};   // (-1)^k / (2k+3)!

// SE3Quat::exp (Thirdparty/g2o/g2o/types/se3quat.h:214-254).  g2o builds R = I + a*Omega + b*Omega^2 with
// a = sin(th)/th, b = (1-cos th)/th^2, c = (th - sin th)/th^3, V = I + b*Omega + c*Omega^2, converts R to a quaternion and
// normalises.  The same rotation in closed form is q = (omega * sin(th/2)/th, cos(th/2)).  All four scalar functions are even
// in th, i.e. power series in th^2: for th^2 < 0.25 (every LM step of a tracking problem) they are evaluated as degree-8
// Horner polynomials in th^2 (truncation < 1e-20, and no th - sin th cancellation), which takes sqrt, sincos and three
// divisions off the serial FP64 dependency chain; larger steps use sincos.  Equal to g2o's value up to rounding (for
// th < 1e-5 g2o switches to R = V = I + Omega + Omega^2, a first-order form that differs from the exact series used here by
// < 1e-10, far inside the parity tolerance).
__device__ __forceinline__ void se3_exp(const double* u, Se3d& T) {
    const double om[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
    const double t = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
    const double O[3][3] = {{0, -om[2], om[1]}, {om[2], 0, -om[0]}, {-om[1], om[0], 0}};
    double O2[3][3], V[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) O2[i][j] = O[i][0] * O[0][j] + O[i][1] * O[1][j] + O[i][2] * O[2][j];
    double qs, qc, b, c;
    if (t < 0.25) {
        // Estrin's scheme: depth 4 (t^2, t^4, t^8 beside the pair sums) instead of the 9 dependent FMAs of Horner's - this runs on one lane
        // with ~36 cycles per dependent FP64 operation, once per LM iteration; the coefficients fall off so fast that the rounding is the same
        const double t2 = t * t, t4 = t2 * t2, t8 = t4 * t4;
        auto estrin = [&](const double* k) {
            const double a01 = fma(k[1], t, k[0]), a23 = fma(k[3], t, k[2]), a45 = fma(k[5], t, k[4]), a67 = fma(k[7], t, k[6]);
            const double b0 = fma(a23, t2, a01), b1 = fma(a67, t2, a45);
            return fma(k[8], t8, fma(b1, t4, b0));
        };
        qs = estrin(kQs); qc = estrin(kQc); b = estrin(kB); c = estrin(kC);
    } else {
        const double it = rsqrt(t), theta = t * it, it2 = it * it;
        double sh, ch;
        sincos(0.5 * theta, &sh, &ch);
        qs = sh * it; qc = ch;
        b = 2 * sh * sh * it2; c = (theta - 2 * sh * ch) * (it2 * it);
    }
    T.qx = om[0] * qs; T.qy = om[1] * qs; T.qz = om[2] * qs; T.qw = qc;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) V[i][j] = (i == j ? 1.0 : 0.0) + b * O[i][j] + c * O2[i][j];
    T.tx = V[0][0] * up[0] + V[0][1] * up[1] + V[0][2] * up[2];
    T.ty = V[1][0] * up[0] + V[1][1] * up[1] + V[1][2] * up[2];
    T.tz = V[2][0] * up[0] + V[2][1] * up[1] + V[2][2] * up[2];
    // g2o's SE3Quat constructor normalises here; q = (omega sin(th/2)/th, cos(th/2)) IS a unit quaternion up to rounding (|q|^2 - 1 ~ 1e-16)
    // and every caller multiplies it into the estimate with se3_mul, which normalises the product: one normalisation per step, not two
    if (t >= 0.25) normalize_rotation(T);
}

__device__ __forceinline__ void se3_mul(const Se3d& a, const Se3d& b, Se3d& r) {
    const double bt[3] = {b.tx, b.ty, b.tz};
    double rt[3];
    quat_rotate(a, bt, rt);
    r.tx = a.tx + rt[0]; r.ty = a.ty + rt[1]; r.tz = a.tz + rt[2];
    r.qw = a.qw * b.qw - a.qx * b.qx - a.qy * b.qy - a.qz * b.qz;
    r.qx = a.qw * b.qx + a.qx * b.qw + a.qy * b.qz - a.qz * b.qy;
    r.qy = a.qw * b.qy + a.qy * b.qw + a.qz * b.qx - a.qx * b.qz;
    r.qz = a.qw * b.qz + a.qz * b.qw + a.qx * b.qy - a.qy * b.qx;
    normalize_rotation(r);
}

// 1/d for a positive normal double: MUFU.RCP64H seed (~20 bits) + two Newton steps (error ~ 1 ulp), 5 dependent operations
// instead of the ~20 of the IEEE division sequence.
__device__ __forceinline__ double rcp_newton(double d) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
    double e = fma(-d, r, 1.0); r = fma(r, e, r);
    e = fma(-d, r, 1.0);        r = fma(r, e, r);
    return r;
}

// Solves (H + lambda I) x = b for the 6x6 damped normal equations.  H = sum rho' J^T Omega J is positive semi-definite and
// lambda > 0, so the system is SPD and an unpivoted LDL^T (the "small on-device Cholesky") is backward stable; g2o's dense
// solver uses Eigen's diagonally pivoted LDLT (Thirdparty/g2o/g2o/solvers/linear_solver_dense.h), which differs from this by
// rounding only (covered by the 1e-5 pose tolerance of the parity tests; the oracle keeps the pivoted form).  This runs on
// ONE thread and is bound by the latency of dependent FP64 operations (~36 cycles each, measured), so it is written for a
// short dependency chain: compile-time indices (registers), b eliminated alongside the columns, one Newton reciprocal per
// pivot, column-oriented back substitution.  Returns false when a pivot is negative (Eigen's isPositive() == false -> g2o treats
// the trial as failed); an exactly zero pivot (no active edge and lambda == 0) leaves that unknown at 0 like Eigen's solve does.
// A NaN pivot (an edge exactly on the camera plane makes H NaN) is neither positive nor negative for Eigen's sign tracking, so the
// solve "succeeds" with a NaN step, the trial is rejected and its NaN errors are what the classification reads, as in g2o.
__device__ __forceinline__ bool solve6(const double* Hsym /*21 upper*/, double lambda, const double* b, double* x) {
    double L[6][6], dinv[6], y[6];
    // every loop has the constant trip count 6 with compile-time guards: triangular bounds defeat the unroller, and one
    // surviving loop would turn the register arrays into local memory
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j)
            if (j >= i) L[j][i] = Hsym[i * 6 - (i * (i - 1)) / 2 + (j - i)];       // lower triangle, column i
#pragma unroll
    for (int i = 0; i < 6; ++i) { L[i][i] += lambda; y[i] = b[i]; }
    bool positive = true;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double d = L[k][k];
        positive = positive && !(d < 0);
        dinv[k] = (d >= DBL_MIN && d <= DBL_MAX) ? rcp_newton(d) : 0.0;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            if (i > k) {
                const double aik = L[i][k], lik = aik * dinv[k];
#pragma unroll
                for (int j = 0; j < 6; ++j)
                    if (j > k && j < i) L[i][j] -= aik * L[j][k];          // rows j < i already hold the scaled l_jk
                L[i][i] -= aik * lik;
                L[i][k] = lik;
                y[i] -= lik * y[k];                                        // forward substitution rides along
            }
        }
    }
    if (!positive) return false;
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] *= dinv[i];
#pragma unroll
    for (int jj = 0; jj < 5; ++jj) {
        const int j = 5 - jj;
#pragma unroll
        for (int i = 0; i < 6; ++i)
            if (i < j) y[i] -= L[j][i] * y[j];
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) x[i] = y[i];
    return true;
}

// 1/sqrt(x) for a positive normal double: MUFU.RSQ64H seed + two Newton steps (7 dependent operations)
__device__ __forceinline__ double rsqrt_newton(double x) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const double t = x * y, h = 0.5 * y;
        const double e = fma(-t, h, 0.5);       // (1 - x y^2) / 2
        y = fma(y, e, y);
    }
    return y;
}

// reciprocal of the camera-frame depth; the Newton form for every normal value, IEEE division (inf / NaN propagation) otherwise
__device__ __forceinline__ double rcp_depth(double z) {
    const double az = fabs(z);
    return (az >= DBL_MIN && az <= DBL_MAX) ? rcp_newton(z) : 1.0 / z;
}

// RobustKernelHuber::robustify (Thirdparty/g2o/g2o/core/robust_kernel_impl.cpp:65-91), branch-free: rho0 = robust cost,
// rho1 = weight.  sqrt(e2) and delta / sqrt(e2) both come from one Newton rsqrt (the IEEE sqrt followed by an IEEE division is
// ~40 dependent FP64 operations on the per-edge critical path).
__device__ __forceinline__ void huber(double e2, double delta, float dsqr, double& rho0, double& rho1) {
    const double rs = rsqrt_newton(fmax(e2, 1e-300)), sq = e2 * rs;
    const bool in = e2 <= (double)dsqr;
    rho0 = in ? e2 : 2 * sq * delta - (double)dsqr;
    rho1 = in ? 1.0 : delta * rs;
}

// Huber's linear region (huber's `in` is false; a NaN e2 counts as linear): where a robust and a non-robust evaluation differ
__device__ __forceinline__ bool huber_linear(double e2, float dsqr) { return !(e2 <= (double)dsqr); }

constexpr int kAcc = 28;      // 21 H + 6 b + 1 chi; a build's and a trial's exchange add one value (the trial's chi2 in evaluation order)
// the classification's exchange: + the outlier count, the number of edges whose level changed, and the threads that evaluated an
// active edge in Huber's linear region during the round and during the next round's first build
constexpr int kXchgClass = kAcc + 4;
// Cluster shape, measured on an H100 SXM (700 W) through the whole resident chain (tools/pose_variants.sh, bench.py config B,
// us per tracked frame incl. both searches): 4 x 256: 324   8 x 128: 257   8 x 256: 328   16 x 64: 239   16 x 128: 269.
// The build / evaluation passes are bound by one SM's FP64 issue rate (~400 DFMA per edge), so more SMs with fewer threads each
// shorten them; 16 is the largest cluster an H100 runs (non-portable size, opted in at the launch).
#ifndef POSE_CTAS
#define POSE_CTAS 16
#define POSE_THREADS 64
#endif
constexpr int kPoseCtas = POSE_CTAS;      // CTAs (SMs) of the cluster that optimises one frame
constexpr int kPoseThreads = POSE_THREADS, kPoseWarps = kPoseThreads / 32, kPoseStride = kPoseCtas * kPoseThreads;
constexpr int kMaxTrials = 10;    // g2o _maxTrialsAfterFailure (lane l of warp w solves trial w + kPoseWarps * l)
constexpr int kSolveLanes = (kMaxTrials + kPoseWarps - 1) / kPoseWarps;

// ---- cluster-wide sums without a cluster barrier ----------------------------------------------------------------------------------
// barrier.cluster costs ~1.3k cycles here (measured with clock64: arrival skew of four SMs + the L1 invalidation its acquire implies),
// 58 times per call.  Instead every CTA pushes its partial sums straight into the other CTAs' shared memory with st.async, which
// also signals the RECEIVER's mbarrier (complete_tx): a CTA only waits for the kPoseCtas x n x 8 bytes addressed to itself.  Exchanges are
// numbered; exchange s uses buffer / mbarrier s & 1, so a CTA that runs ahead writes into the other buffer (it cannot run two
// exchanges ahead: it needs everybody's data of exchange s + 1 first, and those are sent after exchange s was read).  All CTAs add
// the partials in rank order: bit-identical totals everywhere.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
struct ClusterXchg {
    double (*buf)[kPoseCtas][32];     // [2][kPoseCtas][32], shared
    unsigned long long* mbar;         // [2], shared
    unsigned rank, seq;
    __device__ __forceinline__ void init() {
        if (threadIdx.x == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&mbar[0])));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&mbar[1])));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
    // thread t < n_vals contributes v (its CTA's partial of value t); afterwards out[t] (shared) holds the cluster total, for all threads
    __device__ __forceinline__ void sum(double v, int n_vals, double* out) {
        const unsigned b = seq & 1, parity = (seq >> 1) & 1;
        ++seq;
        const uint32_t mb = smem_u32(&mbar[b]);
        if (threadIdx.x == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(kPoseCtas * n_vals * 8) : "memory");
        if ((int)threadIdx.x < n_vals) {
            const uint32_t slot = smem_u32(&buf[b][rank][threadIdx.x]);
#pragma unroll
            for (unsigned r = 0; r < kPoseCtas; ++r)
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];"
                             :: "r"(mapa_u32(slot, r)), "l"(__double_as_longlong(v)), "r"(mapa_u32(mb, r)) : "memory");
        }
        if (threadIdx.x < 32) {
            uint32_t done = 0, spins = 0;
            while (!done) {
                asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                             : "=r"(done) : "r"(mb), "r"(parity) : "memory");
                if (!done && ++spins > (1u << 24)) __trap();      // a lost exchange must fail loudly, not hang the device
            }
            if ((int)threadIdx.x < n_vals) {
                // pairwise tree in a fixed order (the same in every CTA): depth log2(kPoseCtas) dependent FP64 additions instead of kPoseCtas - 1
                double t[kPoseCtas];
#pragma unroll
                for (int r = 0; r < kPoseCtas; ++r) t[r] = buf[b][r][threadIdx.x];
#pragma unroll
                for (int st = 1; st < kPoseCtas; st <<= 1)
#pragma unroll
                    for (int r = 0; r + st < kPoseCtas; r += 2 * st) t[r] += t[r + st];
                out[threadIdx.x] = t[0];
            }
        }
        __syncthreads();
    }
};

// one level of the halving butterfly below.  The distance is a template argument so that every loop is unrolled and v[] stays in
// registers (with the distance as a loop variable the inner loop was unrolled before the distance was known: v[] in local memory)
template <int H>
__device__ __forceinline__ void butterfly_step(double* v, int lane) {
    const bool up = (lane & H) != 0;
#pragma unroll
    for (int k = 0; k < H; ++k) {
        const double send = up ? v[k] : v[k + H];
        const double keep = up ? v[k + H] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, H);
    }
}

// cluster-wide sums of the kAcc build sums v and of one more value `last`, in one exchange.  Inside a warp the 28 sums are folded
// with a halving butterfly: at distance h every lane keeps one half of its slots and ships the other half to its partner, so
// 16+8+4+2+1 = 31 exchanges replace 28 x 5 and lane L ends up with the warp total of slot L.  `last` is folded with shfl_down into
// lane 0, the order the trial chi2 of the rho test is summed in (the build's chi2, slot 27, has its own order: both are kept, each
// feeds its own LM decision).  The warp totals are added in warp order, the CTA totals go through ClusterXchg: out[0..kAcc + NL).
// The classification folds NL = 4 such values (counts, exact in any order) into its exchange.
template <int NL>
__device__ __forceinline__ void cluster_reduce(ClusterXchg& xc, double* v /* 32 slots, 28..31 zero */, double (&last)[NL],
                                               double* smem /* warps*32 */, double* out /* kAcc + NL, shared */) {
    static_assert(kAcc + NL <= 32, "ClusterXchg slots");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    butterfly_step<16>(v, lane); butterfly_step<8>(v, lane); butterfly_step<4>(v, lane); butterfly_step<2>(v, lane); butterfly_step<1>(v, lane);
#pragma unroll
    for (int j = 0; j < NL; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) last[j] += __shfl_down_sync(0xffffffffu, last[j], o);
    if (lane < kAcc) smem[warp * 32 + lane] = v[0];
    if (lane == 0)
#pragma unroll
        for (int j = 0; j < NL; ++j) smem[warp * 32 + kAcc + j] = last[j];
    __syncthreads();
    double s = 0;
    if (threadIdx.x < kAcc + NL) {
        double t[kPoseWarps];
#pragma unroll
        for (int w = 0; w < kPoseWarps; ++w) t[w] = smem[w * 32 + threadIdx.x];
#pragma unroll
        for (int st = 1; st < kPoseWarps; st <<= 1)
#pragma unroll
            for (int w = 0; w + st < kPoseWarps; w += 2 * st) t[w] += t[w + st];
        s = t[0];
    }
    xc.sum(s, kAcc + NL, out);
}
__device__ __forceinline__ void cluster_reduce(ClusterXchg& xc, double* v, double last, double* smem, double* out) {
    double l[1] = {last};
    cluster_reduce<1>(xc, v, l, smem, out);
}

// structural zeros shared by the mono and the stereo Jacobian (d(u)/d(ty) = d(v)/d(tx) = d(ur)/d(ty) = 0)
__device__ constexpr bool kJnz[3][6] = {{true, true, true, true, false, true}, {true, true, true, false, true, true}, {true, true, true, true, false, true}};

}  // namespace

__global__ void __cluster_dims__(kPoseCtas, 1, 1) __launch_bounds__(kPoseThreads) pose_optimize_kernel(Laned<PoseProblemDev> p_l, Laned<double*> work_l, Laned<uint8_t*> level_l,
                                                            Laned<uint8_t*> outlier_l, Laned<float*> pose_out_l,
                                                            Laned<int*> n_inliers_l, Laned<ChainPrepDev> next_l) {
    __shared__ double red[kPoseWarps * 32];
    __shared__ double acc[kXchgClass];    // the cluster totals of the last exchange: the system the next solves start from + 1 or 4 values
    __shared__ __align__(16) double xchg_buf[2][kPoseCtas][32];      // partial sums of the CTAs (written remotely by st.async)
    __shared__ __align__(8) unsigned long long xchg_mbar[2];
    __shared__ float s_posef[7];
    pdl_trigger();                        // the next kernel of the chain may be scheduled (it waits for this grid's completion itself)
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    ClusterXchg xc{xchg_buf, xchg_mbar, rank, 0u};
    xc.init();
    cluster.sync();                       // every CTA's mbarriers are initialised before anyone sends
    pdl_wait();                           // everything above is on-chip set-up and overlaps the tail of the previous kernel; global memory from here on
    __shared__ Se3d s_est, s_init, s_cand[kMaxTrials];
    __shared__ double s_cinv[kMaxTrials], s_lambda, s_ni, s_current, s_ini;
    __shared__ int s_build, s_nbad_lm, s_ok, s_cok[kMaxTrials], s_continue;
    // sequence lane = the cluster's y (the exchange and the next frame's preparation stay inside the lane's cluster)
    const unsigned ln_ = blockIdx.y;
    const PoseProblemDev p = lane_value(p_l, ln_);
    double* __restrict__ work = lane_value(work_l, ln_);
    uint8_t* __restrict__ level = lane_value(level_l, ln_);
    uint8_t* __restrict__ outlier = lane_value(outlier_l, ln_);
    float* __restrict__ pose_out = lane_value(pose_out_l, ln_);
    int* __restrict__ n_inliers = lane_value(n_inliers_l, ln_);
    const ChainPrepDev next = lane_value(next_l, ln_);
    const int tid = threadIdx.x, n = p.n_dev ? *p.n_dev : p.n;
    const int gtid = (int)rank * kPoseThreads + tid;
#ifdef POSE_TIMING
    long long tm[6] = {0, 0, 0, 0, 0, 0}; int tc[4] = {0, 0, 0, 0}; long long t0_ = clock64(), tA_;
#define TM_START() tA_ = clock64()
#define TM_ADD(i) do { long long tB_ = clock64(); tm[i] += tB_ - tA_; tA_ = tB_; } while (0)
#else
#define TM_START()
#define TM_ADD(i)
#endif
    const float* pose_in = p.pose_in_dev ? p.pose_in_dev : p.pose_in;

    // resident chain: with the final pose known, unproject this frame's LiDAR-depth keypoints for the next frame's search
    // (s_posef = the frame's final float32 pose, computed identically by every CTA; the work is split over the cluster)
    auto prepare_next = [&]() {
        __syncthreads();                  // s_posef written by thread 0
        if (rank == 0 && tid < 7) pose_out[tid] = s_posef[tid];
        if (next.kps) {
            if (rank == 0 && tid == 0) chain_prep_motion(next, s_posef);
            float Rwc[9], Ow[3];
            chain_pose_matrices(s_posef, Rwc, Ow);
            for (int i = gtid; i < next.cap; i += kPoseStride) chain_prep_item(next, Rwc, Ow, i);
        }
        cluster.sync();                   // no CTA may exit while another can still address its shared memory
    };
    if (n < 3) {                      // src/Optimizer.cc:996
        if (tid < 7) s_posef[tid] = pose_in[tid];
        if (rank == 0 && tid == 0) *n_inliers = 0;
        prepare_next();
        return;
    }
    const float delta_mono_f = sqrtf(5.991f), delta_stereo_f = sqrtf(7.815f);           // float deltaMono = sqrt(5.991)
    const double dm = (double)(float)sqrt(5.991), ds = (double)(float)sqrt(7.815);
    (void)delta_mono_f; (void)delta_stereo_f;
    const float dsqr_m = (float)(dm * dm), dsqr_s = (float)(ds * ds);
    const double fx = p.fx, fy = p.fy, cx = p.cx, cy = p.cy, bf = p.bf;

    if (tid == 0) {
        Se3d T = {pose_in[0], pose_in[1], pose_in[2], pose_in[3], pose_in[4], pose_in[5], pose_in[6]};
        normalize_rotation(T);
        s_init = T;
    }
    for (int k = gtid; k < n; k += kPoseStride) { level[k] = 0; outlier[k] = 0; }       // every edge belongs to one thread of the cluster for the whole kernel
    __syncthreads();
    bool robust = true;
    bool lin = false;                     // this thread evaluated an active edge of the round in Huber's linear region (robust rounds)
    int n_bad = 0;

    // One edge at pose T: camera-frame point, 1/z and the reprojection error, one code path for both edge types (no warp
    // divergence between mono and stereo keypoints).  Reference: EdgeSE3ProjectXYZOnlyPose / EdgeStereoSE3ProjectXYZOnlyPose
    // ::computeError (src/OptimizableTypes.h, Thirdparty/g2o/g2o/types/types_six_dof_expmap.cpp:339-404): the stereo
    // projection uses a FLOAT 1/z (cam_project), the mono one fx*x/z in double; 1/z is a Newton reciprocal (<= 1 ulp).
    // All loads are issued up front (none depends on the level test).
    struct Edge { double pc[3], invz, e[3], info; bool st, active; };
    auto load_edge = [&](const Se3d& T, int k, Edge& E) {
        const float xwf[3] = {p.xw[3 * k], p.xw[3 * k + 1], p.xw[3 * k + 2]};
        const float ob[3] = {p.obs[3 * k], p.obs[3 * k + 1], p.obs[3 * k + 2]};
        E.st = p.stereo[k] != 0;
        E.info = (double)p.inv_sigma2[k];
        E.active = level[k] == 0;
        const double xw[3] = {xwf[0], xwf[1], xwf[2]};
        se3_map(T, xw, E.pc);
        E.invz = rcp_depth(E.pc[2]);
        const double iz = E.st ? (double)(float)E.invz : E.invz;
        const double u = E.pc[0] * iz * fx + cx, v = E.pc[1] * iz * fy + cy;
        E.e[0] = (double)ob[0] - u; E.e[1] = (double)ob[1] - v;
        E.e[2] = E.st ? (double)ob[2] - (u - bf * iz) : 0.0;
    };

    // computeActiveErrors + activeRobustChi2 + buildSystem for one active edge at the pose its camera-frame point and errors E were
    // computed at: adds its robust chi2 to v[27], rho' J^T Omega J to v[0..20] (upper triangle) and -rho' J^T Omega e to v[21..26];
    // sets lin when a robust evaluation falls in Huber's linear region
    auto accumulate = [&](const Edge& E, bool rob, double (&v)[32], bool& lin) {
        const bool st = E.st;
        const double info = E.info, x = E.pc[0], y = E.pc[1], invz = E.invz, invz_2 = invz * invz;
        const double e[3] = {E.e[0], E.e[1], E.e[2]};
        double J[3][6];
        // rows 0/1 are the same expressions for both edge types (mono: -projectJac * [-(p)x | I], expanded);
        // the third row of a mono edge is zero, so its terms add exact zeros to the sums
        J[0][0] = x * y * invz_2 * fx;       J[0][1] = -(1 + (x * x * invz_2)) * fx; J[0][2] = y * invz * fx;
        J[0][3] = -invz * fx;                J[0][4] = 0;                           J[0][5] = x * invz_2 * fx;
        J[1][0] = (1 + y * y * invz_2) * fy; J[1][1] = -x * y * invz_2 * fy;        J[1][2] = -x * invz * fy;
        J[1][3] = 0;                         J[1][4] = -invz * fy;                  J[1][5] = y * invz_2 * fy;
        const double sbf = st ? bf : 0.0;
        J[2][0] = st ? J[0][0] - sbf * y * invz_2 : 0.0; J[2][1] = st ? J[0][1] + sbf * x * invz_2 : 0.0;
        J[2][2] = st ? J[0][2] : 0.0;                    J[2][3] = st ? J[0][3] : 0.0;
        J[2][4] = 0;                                     J[2][5] = st ? J[0][5] - sbf * invz_2 : 0.0;
        double chi = 0;
#pragma unroll
        for (int r = 0; r < 3; ++r) chi += e[r] * (info * e[r]);
        double w = 1.0, r0 = chi;
        if (rob) { lin |= huber_linear(chi, st ? dsqr_s : dsqr_m); huber(chi, st ? ds : dm, st ? dsqr_s : dsqr_m, r0, w); }
        v[27] += r0;
        const double wi = w * info;
        double WJ[3][6], we[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            we[r] = wi * e[r];
#pragma unroll
            for (int c = 0; c < 6; ++c) WJ[r][c] = kJnz[r][c] ? wi * J[r][c] : 0.0;
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            double sb = 0;
#pragma unroll
            for (int r = 0; r < 3; ++r) if (kJnz[r][i]) sb += J[r][i] * we[r];
            v[21 + i] -= sb;
#pragma unroll
            for (int j = i; j < 6; ++j) {
                double h = 0;
#pragma unroll
                for (int r = 0; r < 3; ++r) if (kJnz[r][i] && kJnz[r][j]) h += J[r][i] * WJ[r][j];
                v[i * 6 - (i * (i - 1)) / 2 + (j - i)] += h;
            }
        }
    };

    bool first_build = true;              // the round's iteration-0 system needs a build pass of its own
    for (int it = 0; it < 4;) {
        // round 0 starts with a build pass at the initial pose; every later round's iteration-0 system was built by the previous
        // executed round's classification pass, unless that was built with the other robust flag (see the end of the round)
        if (tid == 0) { s_est = s_init; s_ok = 1; s_build = first_build; }
        __syncthreads();
        for (int iter = 0; iter < 10; ++iter) {
            if (!s_ok) break;
            // ---- a build pass of its own only where no pass before built this system: round 0's first one, and after an iteration
            // that ended on a rejected trial without ending the round (rho > 0 with a non-finite chi2, or a NaN rho) ----
            if (s_build) {
                double v[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) v[k] = 0;
                TM_START();
                const Se3d T = s_est;
                for (int k = gtid; k < n; k += kPoseStride) {
                    Edge E;
                    load_edge(T, k, E);
                    if (E.active) accumulate(E, robust, v, lin);
                }
                TM_ADD(0);
                cluster_reduce(xc, v, 0.0, red, acc);
                TM_ADD(1);
#ifdef POSE_TIMING
                tc[0]++;
#endif
            }
            // ---- LM trials.  A rejected trial only changes lambda (x nu, nu doubling), never H, b or the estimate, so the damped solves of all (<= 10) possible trials of this iteration
            // are independent: lane 0 of warp w solves trial w while the other warps would idle anyway, and a retry then
            // costs one error evaluation instead of a serial solve + exp. ----
            TM_START();
            if ((tid & 31) < kSolveLanes && (tid >> 5) + kPoseWarps * (tid & 31) < kMaxTrials) {
                const int w = (tid >> 5) + kPoseWarps * (tid & 31);        // trial w: lane w / 8 of warp w % 8
                // lambda of trial w = lambda * nu * 2nu * ... (w factors); nu is a power of two, so this is one exponent shift
                // (lambda0 = 1e-5 * max diag(H) and nu = 2 at iteration 0 of a round: every solver lane derives them itself
                // from the reduced system, thread 0 also publishes them, so no barrier is needed before this stage)
                double lam_base, ni_base;
                if (iter == 0) {
                    double mx = 0;
#pragma unroll
                    for (int i = 0; i < 6; ++i) mx = fmax(fabs(acc[i * 6 - (i * (i - 1)) / 2]), mx);
                    lam_base = 1e-5 * mx; ni_base = 2;
                } else {
                    lam_base = s_lambda; ni_base = s_ni;
                }
                if (w == 0) {
                    s_current = acc[27]; s_ini = acc[27];
                    if (iter == 0) { s_lambda = lam_base; s_ni = 2; s_nbad_lm = 0; }
                }
                const double lam = scalbn(lam_base, w * ilogb(ni_base) + (w * (w - 1)) / 2);
                double x[6] = {0, 0, 0, 0, 0, 0};
#ifdef POSE_TIMING
                const long long ts_ = clock64();
#endif
                s_cok[w] = solve6(acc, lam, acc + 21, x) ? 1 : 0;
#ifdef POSE_TIMING
                tm[5] += clock64() - ts_;
#endif
                // denominator of the gain ratio, x^T (lambda x + b) + 1e-3 (optimization_algorithm_levenberg.cpp:129-135):
                // known here, so its reciprocal is off the serial accept/reject path
                double scale = 0;
#pragma unroll
                for (int i = 0; i < 6; ++i) scale += x[i] * (lam * x[i] + acc[21 + i]);
                s_cinv[w] = rcp_depth(scale + 1e-3);       // Newton reciprocal (<= 1 ulp): the IEEE division is ~20 dependent operations
                Se3d E, Tn;
                se3_exp(x, E);
                se3_mul(E, s_est, Tn);
                s_cand[w] = Tn;
            }
            __syncthreads();
            TM_ADD(2);
            for (int trial = 0;; ++trial) {
                // ---- one pass evaluates the trial (errors -> work[] for the classification, robust chi2 for the rho test) and builds
                // the system at the trial's pose: if the trial is accepted, that pose is the next iteration's estimate and its
                // solves start from this exchange; if it is rejected, the system is dropped ----
                TM_START();
                double v[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) v[k] = 0;
                double part = 0;
                {
                    const Se3d T = s_cand[trial];
                    for (int k = gtid; k < n; k += kPoseStride) {
                        Edge E;
                        load_edge(T, k, E);
                        if (!E.active) continue;
                        work[3 * (size_t)k] = E.e[0]; work[3 * (size_t)k + 1] = E.e[1]; work[3 * (size_t)k + 2] = E.e[2];
                        double chi = E.e[0] * (E.info * E.e[0]) + E.e[1] * (E.info * E.e[1]) + E.e[2] * (E.info * E.e[2]);
                        if (robust) {
                            double r0, r1;
                            lin |= huber_linear(chi, E.st ? dsqr_s : dsqr_m);
                            huber(chi, E.st ? ds : dm, E.st ? dsqr_s : dsqr_m, r0, r1); chi = r0;
                        }
                        part += chi;
                        accumulate(E, robust, v, lin);
                    }
                }
                TM_ADD(3);
                cluster_reduce(xc, v, part, red, acc);
                if (tid == 0) {            // every CTA takes the decision from the same partials: identical everywhere
                    double temp = acc[kAcc];
                    if (!s_cok[trial]) temp = DBL_MAX;
                    const double rho = (s_current - temp) * s_cinv[trial];
                    if (rho > 0 && isfinite(temp)) {
                        const double r21 = 2 * rho - 1;
                        double alpha = 1. - r21 * r21 * r21;
                        alpha = fmin(alpha, 2. / 3.);
                        const double sf = fmax(1. / 3., alpha);
                        s_lambda *= sf; s_ni = 2; s_current = temp; s_est = s_cand[trial]; s_build = 0;
#ifdef POSE_TIMING
                        tc[2]++;
#endif
                    } else {
                        s_lambda *= s_ni; s_ni *= 2; s_build = 1;       // the estimate is restored = left untouched
                    }
                    const int qmax = trial + 1;
                    const int cont = (rho < 0 && qmax < kMaxTrials) ? 1 : 0;
                    s_continue = cont;
                    if (!cont) {                              // end of this LM iteration: g2o's stop tests
                        int ok = 1;
                        if (qmax == kMaxTrials || rho == 0) ok = 0;
                        else {
                            if ((s_ini - s_current) * 1e3 < s_ini) s_nbad_lm += 1; else s_nbad_lm = 0;
                            if (s_nbad_lm >= 3) ok = 0;
                        }
                        s_ok = ok;
                    }
                }
                __syncthreads();
                TM_ADD(4);
#ifdef POSE_TIMING
                tc[1]++;
#endif
                if (!s_continue) break;
            }
        }
        // ---- classification (src/Optimizer.cc:1014-1100).  Its pass also builds round it + 1's iteration-0 system at the initial
        // pose, with the levels just decided and that round's robust flag; its exchange carries the outlier count, the number of level
        // changes and the linear-region flags of this round and of that build ----
        bool changed = false, lin_round = false, lin_first = false;
        const bool robust_next = it < 2;
        bool lin_next = false;            // this thread's part of lin_first
        {
            const Se3d T = s_est;
            const bool build_next = it < 3 && n >= 10;
            double v[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) v[k] = 0;
            int bad = 0, moved = 0;
            for (int k = gtid; k < n; k += kPoseStride) {
                const bool st = p.stereo[k] != 0;
                const double info = (double)p.inv_sigma2[k];
                double e0, e1, e2 = 0;
                const bool was_out = outlier[k] != 0;         // = level[k] != 0
                if (was_out) {
                    Edge E;
                    load_edge(T, k, E);
                    e0 = E.e[0]; e1 = E.e[1]; e2 = E.e[2];
                    work[3 * (size_t)k] = e0; work[3 * (size_t)k + 1] = e1; work[3 * (size_t)k + 2] = e2;
                } else {
                    e0 = work[3 * (size_t)k]; e1 = work[3 * (size_t)k + 1]; e2 = work[3 * (size_t)k + 2];
                }
                double chi = e0 * (info * e0) + e1 * (info * e1);
                if (st) chi += e2 * (info * e2);
                const float chi2 = (float)chi;
                if (chi2 > (st ? 7.815f : 5.991f)) { outlier[k] = 1; level[k] = 1; ++bad; moved += !was_out; }
                else {
                    outlier[k] = 0; level[k] = 0; moved += was_out;
                    if (build_next) {
                        Edge E;
                        load_edge(s_init, k, E);
                        accumulate(E, robust_next, v, lin_next);
                    }
                }
            }
            double last[4] = {(double)bad, (double)moved, lin ? 1.0 : 0.0, lin_next ? 1.0 : 0.0};
            cluster_reduce<4>(xc, v, last, red, acc);
            n_bad = (int)acc[kAcc];
            changed = acc[kAcc + 1] != 0; lin_round = acc[kAcc + 2] != 0; lin_first = acc[kAcc + 3] != 0;
        }
        if (n < 10) break;
        // ---- rounds that repeat this one.  A round's result is a function of the initial pose, the levels and its robust flag only:
        // the kernel is deterministic (fixed summation orders, no atomics).  So with no level changed, round it + 1 repeats round it
        // bit for bit when its robust flag is the same, and also when it is not but no active edge of round it (its iteration-0
        // system, build passes, every evaluated trial) fell in Huber's linear region: huber() then returns rho = e2 and weight 1.0,
        // the non-robust values.  The repeat would classify every edge as before, so the next round repeats it too: skip them all.
        int next = it + 1;
#ifndef POSE_RUN_ALL_ROUNDS               // test builds only (tests/test_cuda_emu_pose_replica.py): the same kernel running every round
        while (next < 4 && !changed && ((next < 3) == (it < 3) || !lin_round)) {
            ++next;
#ifdef POSE_TIMING
            tc[3]++;
#endif
        }
#endif
        // the classification built the first system with round it + 1's robust flag; the next round to run needs the other one only
        // after a skip from round 0 or 1 to round 3.  That system is the non-robust one too when no edge of its build fell in the
        // linear region, otherwise the round starts with a build pass of its own.
        robust = next < 3;
        first_build = robust != robust_next && lin_first;
        lin = first_build ? false : lin_next;
        it = next;
    }
    if (tid == 0) {
        const Se3d T = s_est;
        // Sophus::SE3<float>(rotation().cast<float>(), ...) (src/Optimizer.cc:1108-1110): the SO3f quaternion constructor normalises in float
        const float qf[4] = {(float)T.qx, (float)T.qy, (float)T.qz, (float)T.qw};
        const float qlen = sqrtf(eig_sum4(__fmul_rn(qf[0], qf[0]), __fmul_rn(qf[1], qf[1]), __fmul_rn(qf[2], qf[2]), __fmul_rn(qf[3], qf[3])));
        s_posef[0] = __fdiv_rn(qf[0], qlen); s_posef[1] = __fdiv_rn(qf[1], qlen); s_posef[2] = __fdiv_rn(qf[2], qlen); s_posef[3] = __fdiv_rn(qf[3], qlen);
        s_posef[4] = (float)T.tx; s_posef[5] = (float)T.ty; s_posef[6] = (float)T.tz;
        if (rank == 0) *n_inliers = n - n_bad;
#ifdef POSE_TIMING
        if (rank == 0) printf("pose n=%d total=%lld build=%lld(%d) breduce=%lld solve=%lld eval=%lld(%d, %d accepted) evalred=%lld solve6=%lld skipped=%d\n", n, clock64() - t0_, tm[0], tc[0], tm[1], tm[2], tm[3], tc[1], tc[2], tm[4], tm[5], tc[3]);
#endif
    }
    prepare_next();
}

const char* pose_cluster_unsupported(int device) {
    // A cluster runs inside one GPC: kPoseCtas SMs of one GPC must be able to hold a CTA each (a full H100 has GPCs of 16-18 SMs; a
    // smaller part or a MIG slice may not).  Sizes above 8 are not portable and need the opt-in.  Checked once per device.
    static std::atomic<int> state[64];            // 0 unknown, 1 runs, 2 cannot
    static const std::string why = "the pose optimisation needs a thread-block cluster of " + std::to_string(kPoseCtas) +
                                   " CTAs in one GPC, which this device (or MIG partition) cannot place";
    if (device < 0 || device >= 64) return why.c_str();
    if (state[device] == 0) {
        int n = 0;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(kPoseCtas); cfg.blockDim = dim3(kPoseThreads);
        const bool ok = cudaSetDevice(device) == cudaSuccess &&
                        (kPoseCtas <= 8 || cudaFuncSetAttribute(pose_optimize_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) &&
                        cudaOccupancyMaxActiveClusters(&n, pose_optimize_kernel, &cfg) == cudaSuccess && n >= 1;
        if (!ok) cudaGetLastError();              // clear the error of the failed query
        state[device] = ok ? 1 : 2;
    }
    return state[device] == 1 ? nullptr : why.c_str();
}

int pose_max_active_clusters(int device) {
    if (pose_cluster_unsupported(device)) return 0;
    int n = 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kPoseCtas); cfg.blockDim = dim3(kPoseThreads);
    if (cudaSetDevice(device) != cudaSuccess || cudaOccupancyMaxActiveClusters(&n, pose_optimize_kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void launch_pose_optimize(cudaStream_t st, const Laned<PoseProblemDev>& p, const Laned<double*>& work, const Laned<uint8_t*>& level,
                          const Laned<uint8_t*>& outlier, const Laned<float*>& pose_out, const Laned<int*>& n_inliers, const Laned<ChainPrepDev>* next,
                          int lanes) {
    launch_kernel(pose_optimize_kernel, dim3(kPoseCtas, lanes), dim3(kPoseThreads), 0, st, chain_launch_pdl(), p, work, level, outlier, pose_out, n_inliers,
                  next ? *next : Laned<ChainPrepDev>());
}

}  // namespace rgbl
