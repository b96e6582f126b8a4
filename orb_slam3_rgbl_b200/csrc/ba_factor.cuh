// The reduced camera system of both bundle adjustments (api_ba.cu): S x_p = b_p - coef, S = L L^T read from the lower triangle of the
// dense n x n system (n = 6 n_opt, row-major), factored in place.  One selection by size (ba_solve_reduced):
//   n_opt <= kSingleCtaMaxOpt   ba_cholesky_kernel: one CTA, two block barriers per column (local BA's 1-64 free key frames)
//   larger                      a blocked right-looking Cholesky over kTile x kTile tiles, across the whole GPU; per tile column k
//     chol_potrf_kernel   one CTA          : L_kk = chol(A_kk)
//     chol_trsm_kernel    CTA per tile     : L_ik = A_ik L_kk^-T, i > k
//     chol_update_kernel  CTA per tile     : A_ij -= L_ik L_jk^T, k < j <= i, on the FP64 tensor cores (mma.sync m8n8k4 .f64)
//   then the substitutions by tile rows, one launch per tile row and a CTA per tile it touches (chol_forward_kernel, chol_back_kernel).
// Both paths fail alike: a non-positive or non-finite pivot sets status[0] = 1 and the solution is zero (g2o: the linear solver fails, the
// LM trial is rejected).  The tiled path checks every pivot of every diagonal tile; a non-finite entry anywhere in S reaches a diagonal
// pivot through the trailing updates (A_ii -= sum_k L_ik^2 over the whole row), so it fails there.  After a failure the later launches
// return at once.
//
// Everything is in this header so that two translation units can compile it: ba_factor.cu for the libraries, and the CPU emulation's
// entry tests/cuda_emu/emu_ba_factor.cpp, whose build transforms the kernel launches of headers in this directory.
#ifndef RGBL_BA_FACTOR_CUH
#define RGBL_BA_FACTOR_CUH
#include <cfloat>
#include <cmath>

#include "rgbl_kernels.h"
#ifdef RGBL_TESTING_EXPORTS
#include "rgbl_testing.h"
#endif

namespace rgbl {
namespace {

// dense Cholesky S = L L^T on the lower triangle, then L L^T x = b_p - coef, by one CTA.  The matrix is staged in shared
// memory when it fits (n <= 160: 6 n_opt squared doubles), else it is factored in place in global memory.  status[0] = 1 on a
// non-positive pivot (g2o: the linear solver fails -> the LM trial is rejected).
__global__ void __launch_bounds__(1024) ba_cholesky_kernel(int n, int use_smem, double* __restrict__ Sg, const double* __restrict__ bp, const double* __restrict__ coef,
                                                           double* __restrict__ x, int* __restrict__ status) {
    extern __shared__ double s_mat[];
    const int tid = threadIdx.x, nt = blockDim.x;
    double* S = use_smem ? s_mat : Sg;
    double* y = use_smem ? s_mat + (size_t)n * n : x;
    if (use_smem) for (int i = tid; i < n * n; i += nt) S[i] = Sg[i];
    for (int i = tid; i < n; i += nt) y[i] = bp[i] - coef[i];
    __syncthreads();
    // two barriers per column: every thread reads the pivot itself (uniform failure test, no broadcast step)
    bool fail = false;
    for (int k = 0; k < n; ++k) {
        const double d = S[(size_t)k * n + k];
        if (!(d > 0) || !(d <= DBL_MAX)) { fail = true; break; }
        const double sd = sqrt(d), inv = 1.0 / sd;
        __syncthreads();                                          // everyone has read the pivot before it is overwritten
        for (int i = k + tid; i < n; i += nt) S[(size_t)i * n + k] = (i == k) ? sd : S[(size_t)i * n + k] * inv;
        __syncthreads();
        // trailing update of the lower triangle (rows i > k, columns k < j <= i) on a 16-wide thread grid: no index divisions
        const int tx = tid & 15, ty = tid >> 4, ny = nt >> 4;
        for (int i = k + 1 + ty; i < n; i += ny) {
            const double lik = S[(size_t)i * n + k];
            for (int j = k + 1 + tx; j <= i; j += 16) S[(size_t)i * n + j] -= lik * S[(size_t)j * n + k];
        }
        __syncthreads();
    }
    if (fail) { if (tid == 0) status[0] = 1; for (int i = tid; i < n; i += nt) x[i] = 0; return; }
    if (tid == 0) status[0] = 0;
    // column-oriented substitutions, one barrier per column: every thread forms y[k] / L[k][k] itself
    for (int k = 0; k < n; ++k) {
        const double yk = y[k] / S[(size_t)k * n + k];
        __syncthreads();
        if (tid == 0) y[k] = yk;
        for (int i = k + 1 + tid; i < n; i += nt) y[i] -= S[(size_t)i * n + k] * yk;
        __syncthreads();
    }
    for (int k = n - 1; k >= 0; --k) {
        const double yk = y[k] / S[(size_t)k * n + k];
        __syncthreads();
        if (tid == 0) y[k] = yk;
        for (int i = tid; i < k; i += nt) y[i] -= S[(size_t)k * n + i] * yk;
        __syncthreads();
    }
    if (use_smem) for (int i = tid; i < n; i += nt) x[i] = y[i];
}

constexpr int kTile = 64;            // tile edge of the blocked path (doubles)
constexpr int kLd = kTile + 1;       // shared-memory row stride of a whole tile (odd: a column walk touches 32 distinct banks pairs)

// a tile of S (rows r0.., columns c0..) into shared memory; entries outside the n x n system are 0, and 1 on the diagonal of a diagonal
// tile, so a partial last tile factors like a full one whose padding is the identity
__device__ __forceinline__ void load_tile(const double* __restrict__ S, int n, int r0, int c0, double (*t)[kLd], bool diag) {
    for (int e = threadIdx.x; e < kTile * kTile; e += blockDim.x) {
        const int r = e / kTile, c = e % kTile;
        t[r][c] = (r0 + r < n && c0 + c < n) ? S[(size_t)(r0 + r) * n + c0 + c] : (diag && r == c ? 1.0 : 0.0);
    }
}

// L_kk = chol(A_kk) of the diagonal tile k, in shared memory, with ba_cholesky_kernel's column loop and pivot test
__global__ void __launch_bounds__(256) chol_potrf_kernel(int n, int k, double* __restrict__ S, int* __restrict__ status) {
    __shared__ double t[kTile][kLd];
    if (status[0]) return;
    const int k0 = k * kTile, m = min(kTile, n - k0), tid = threadIdx.x;
    load_tile(S, n, k0, k0, t, true);
    __syncthreads();
    bool fail = false;
    for (int c = 0; c < m; ++c) {
        const double d = t[c][c];
        if (!(d > 0) || !(d <= DBL_MAX)) { fail = true; break; }
        const double sd = sqrt(d), inv = 1.0 / sd;
        __syncthreads();
        for (int i = c + tid; i < m; i += 256) t[i][c] = (i == c) ? sd : t[i][c] * inv;
        __syncthreads();
        const int tx = tid & 15, ty = tid >> 4;
        for (int i = c + 1 + ty; i < m; i += 16) {
            const double lic = t[i][c];
            for (int j = c + 1 + tx; j <= i; j += 16) t[i][j] -= lic * t[j][c];
        }
        __syncthreads();
    }
    if (fail) { if (tid == 0) status[0] = 1; return; }
    for (int e = tid; e < m * m; e += 256) {
        const int r = e / m, c = e % m;
        if (c <= r) S[(size_t)(k0 + r) * n + k0 + c] = t[r][c];
    }
}

// L_ik = A_ik L_kk^-T for the tiles below diagonal tile k: thread r solves row r of its tile against L_kk, column by column (each row is
// independent, so no barrier inside the solve).  Dynamic shared memory: the two tiles, kTrsmSmem bytes
constexpr int kTrsmSmem = 2 * kTile * kLd * sizeof(double);
__global__ void __launch_bounds__(kTile) chol_trsm_kernel(int n, int k, double* __restrict__ S, const int* __restrict__ status) {
    extern __shared__ double trsm_smem[];
    double (*l)[kLd] = reinterpret_cast<double (*)[kLd]>(trsm_smem);
    double (*a)[kLd] = l + kTile;
    if (status[0]) return;
    const int k0 = k * kTile, i0 = (k + 1 + blockIdx.x) * kTile, r = threadIdx.x;
    load_tile(S, n, k0, k0, l, true);
    load_tile(S, n, i0, k0, a, false);
    __syncthreads();
    for (int c = 0; c < kTile; ++c) {
        double v = a[r][c];
        for (int j = 0; j < c; ++j) v -= a[r][j] * l[c][j];
        a[r][c] = v / l[c][c];
    }
    __syncthreads();
    for (int e = r; e < kTile * kTile; e += kTile) {
        const int rr = e / kTile, c = e % kTile;
        if (i0 + rr < n) S[(size_t)(i0 + rr) * n + k0 + c] = a[rr][c];
    }
}

// D(8x8) += A(8x4, row-major) B(4x8, column-major) on the FP64 tensor cores, a warp-collective (PTX ISA "mma.sync", m8n8k4 .f64): with
// g = lane / 4 and q = lane % 4 the lane holds a = A[g][q], b = B[q][g] and d0, d1 = D[g][2q], D[g][2q + 1]
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
#ifdef RGBL_CUDA_EMU
    // the CPU emulation has no tensor cores: the same warp-collective from shuffles, each element as c + a0 b0 + a1 b1 + a2 b2 + a3 b3
    // with fused multiply-adds in k order (the device's order within one mma is not specified; results are checked against tolerances)
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double ak = __shfl_sync(0xffffffffu, a, 4 * g + k);
        const double b0 = __shfl_sync(0xffffffffu, b, 4 * (2 * q) + k), b1 = __shfl_sync(0xffffffffu, b, 4 * (2 * q + 1) + k);
        d0 = fma(ak, b0, d0);
        d1 = fma(ak, b1, d1);
    }
#else
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
#endif
}

constexpr int kKc = 32;              // K chunk of the trailing update staged in shared memory
constexpr int kLdK = kKc + 4;        // its row stride: the 16 lanes of a half-warp read 16 distinct bank pairs

// A_ij -= L_ik L_jk^T for one tile (i, j), k < j <= i, of the trailing lower triangle (blockIdx.x enumerates them row by row).  Eight
// warps; warp w owns rows 8w..8w+7 of the tile and all 64 columns: eight m8n8k4 accumulators, K = 64 in two staged chunks
__global__ void __launch_bounds__(256) chol_update_kernel(int n, int k, double* __restrict__ S, const int* __restrict__ status) {
    __shared__ double as[kTile][kLdK], bs[kTile][kLdK];
    if (status[0]) return;
    int ti = (int)((sqrt(8.0 * blockIdx.x + 1.0) - 1.0) * 0.5);
    while (ti * (ti + 1) / 2 > (int)blockIdx.x) --ti;
    while ((ti + 1) * (ti + 2) / 2 <= (int)blockIdx.x) ++ti;
    const int tj = blockIdx.x - ti * (ti + 1) / 2;
    const int k0 = k * kTile, i0 = (k + 1 + ti) * kTile, j0 = (k + 1 + tj) * kTile;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    double acc[8][2];
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t][0] = acc[t][1] = 0.0;
    for (int kc = 0; kc < kTile; kc += kKc) {
        __syncthreads();
        for (int e = threadIdx.x; e < kTile * kKc; e += 256) {
            const int r = e / kKc, c = e % kKc;
            as[r][c] = i0 + r < n ? S[(size_t)(i0 + r) * n + k0 + kc + c] : 0.0;
            bs[r][c] = j0 + r < n ? S[(size_t)(j0 + r) * n + k0 + kc + c] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kKc; kk += 4) {
            const double a = as[8 * warp + g][kk + q];
#pragma unroll
            for (int t = 0; t < 8; ++t) dmma_m8n8k4(acc[t][0], acc[t][1], a, bs[8 * t + g][kk + q]);
        }
    }
    const int r = i0 + 8 * warp + g;
    if (r >= n) return;
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = j0 + 8 * t + 2 * q + h;
            if (c < n && (ti != tj || c <= r)) S[(size_t)r * n + c] -= acc[t][h];
        }
}

// w = b_p - coef
__global__ void __launch_bounds__(256) chol_rhs_kernel(int n, const double* __restrict__ bp, const double* __restrict__ coef, double* __restrict__ w) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) w[i] = bp[i] - coef[i];
}

// forward substitution, tile row k: every CTA forms y_k = L_kk^-1 w_k itself (column by column, thread r owns row r); CTA 0 stores it in
// x, CTA b > 0 subtracts L_(k+b),k y_k from w_(k+b).  No CTA writes what another reads in the same launch.
__global__ void __launch_bounds__(kTile) chol_forward_kernel(int n, int k, const double* __restrict__ S, double* __restrict__ w, double* __restrict__ x,
                                                              const int* __restrict__ status) {
    __shared__ double l[kTile][kLd];
    __shared__ double y[kTile];
    if (status[0]) return;
    const int k0 = k * kTile, m = min(kTile, n - k0), r = threadIdx.x;
    load_tile(S, n, k0, k0, l, true);
    double v = r < m ? w[k0 + r] : 0.0;
    __syncthreads();
    for (int c = 0; c < m; ++c) {
        if (r == c) y[c] = v / l[c][c];
        __syncthreads();
        if (r > c) v -= l[r][c] * y[c];
    }
    __syncthreads();
    if (blockIdx.x == 0) { if (r < m) x[k0 + r] = y[r]; return; }
    const int i0 = k0 + blockIdx.x * kTile;
    load_tile(S, n, i0, k0, l, false);
    __syncthreads();
    if (i0 + r >= n) return;
    double s = 0.0;
    for (int c = 0; c < m; ++c) s += l[r][c] * y[c];
    w[i0 + r] -= s;
}

// back substitution, tile row k (descending): every CTA forms z_k = L_kk^-T x_k; CTA k stores it in w, CTA b < k subtracts L_k,b^T z_k
// from x_b
__global__ void __launch_bounds__(kTile) chol_back_kernel(int n, int k, const double* __restrict__ S, double* __restrict__ x, double* __restrict__ w,
                                                           const int* __restrict__ status) {
    __shared__ double l[kTile][kLd];
    __shared__ double z[kTile];
    if (status[0]) return;
    const int k0 = k * kTile, m = min(kTile, n - k0), r = threadIdx.x;
    load_tile(S, n, k0, k0, l, true);
    double v = r < m ? x[k0 + r] : 0.0;
    __syncthreads();
    for (int c = m - 1; c >= 0; --c) {
        if (r == c) z[c] = v / l[c][c];
        __syncthreads();
        if (r < c) v -= l[c][r] * z[c];
    }
    __syncthreads();
    if ((int)blockIdx.x == k) { if (r < m) w[k0 + r] = z[r]; return; }
    const int b0 = blockIdx.x * kTile;
    load_tile(S, n, k0, b0, l, false);
    __syncthreads();
    double s = 0.0;
    for (int c = 0; c < m; ++c) s += l[c][r] * z[c];
    x[b0 + r] -= s;
}

// x = the solution, or zero after a failed factorisation
__global__ void __launch_bounds__(256) chol_out_kernel(int n, const double* __restrict__ w, const int* __restrict__ status, double* __restrict__ x) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) x[i] = status[0] ? 0.0 : w[i];
}

}  // namespace

int ba_solve_reduced(cudaStream_t st, int n, double* S, const double* bp, const double* coef, double* x, double* work, int* status,
                     BaSolvePath path) {
    if (path == BaSolvePath::by_size) path = n <= 6 * kSingleCtaMaxOpt ? BaSolvePath::single_cta : BaSolvePath::tiled;
    static bool attr_done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && !attr_done[dev]) {
        cudaFuncSetAttribute(ba_cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(chol_trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTrsmSmem);
        attr_done[dev] = true;
    }
    if (path == BaSolvePath::single_cta) {
        const size_t chol_need = ((size_t)n * n + n) * sizeof(double);
        const int chol_in_smem = chol_need <= 200 * 1024 ? 1 : 0;
        const size_t chol_smem = chol_in_smem ? chol_need : 0;
        const int chol_threads = n <= 192 ? 256 : 1024;          // small systems: cheaper barriers matter more than lanes
        ba_cholesky_kernel<<<1, chol_threads, chol_smem, st>>>(n, chol_in_smem, S, bp, coef, x, status);
        return 1;
    }
    const int nt = (n + kTile - 1) / kTile;
    int launches = 3;
    cudaMemsetAsync(status, 0, sizeof(int), st);
    chol_rhs_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, bp, coef, work);
    for (int k = 0; k < nt; ++k) {
        chol_potrf_kernel<<<1, 256, 0, st>>>(n, k, S, status);
        const int below = nt - 1 - k;
        if (below > 0) {
            chol_trsm_kernel<<<below, kTile, kTrsmSmem, st>>>(n, k, S, status);
            chol_update_kernel<<<below * (below + 1) / 2, 256, 0, st>>>(n, k, S, status);
            launches += 2;
        }
        ++launches;
    }
    for (int k = 0; k < nt; ++k) chol_forward_kernel<<<nt - k, kTile, 0, st>>>(n, k, S, work, x, status);
    for (int k = nt - 1; k >= 0; --k) chol_back_kernel<<<k + 1, kTile, 0, st>>>(n, k, S, x, work, status);
    chol_out_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, work, status, x);
    return launches + 2 * nt;
}

}  // namespace rgbl

#ifdef RGBL_TESTING_EXPORTS
extern "C" int rgbl_testing_reduced_solve(int n_, const double* S, const double* b, int path, double* x, int* status) {
    using namespace rgbl;
    if (n_ < 1 || !S || !b || !x || !status || path < 0 || path > 2) return RGBL_E_INVALID;
    const size_t n = (size_t)n_;
    double *dS = nullptr, *db = nullptr, *dz = nullptr, *dx = nullptr, *dw = nullptr;
    int* dst = nullptr;
    int rc = RGBL_E_CUDA;
    cudaStream_t st = nullptr;
    if (cudaMalloc(&dS, n * n * sizeof(double)) == cudaSuccess && cudaMalloc(&db, n * sizeof(double)) == cudaSuccess &&
        cudaMalloc(&dz, n * sizeof(double)) == cudaSuccess && cudaMalloc(&dx, n * sizeof(double)) == cudaSuccess &&
        cudaMalloc(&dw, n * sizeof(double)) == cudaSuccess && cudaMalloc(&dst, sizeof(int)) == cudaSuccess &&
        cudaMemcpy(dS, S, n * n * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess &&
        cudaMemcpy(db, b, n * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess && cudaMemset(dz, 0, n * sizeof(double)) == cudaSuccess &&
        cudaMemset(dst, 0, sizeof(int)) == cudaSuccess) {
        ba_solve_reduced(st, n_, dS, db, dz, dx, dw, dst, path == 0 ? BaSolvePath::by_size : path == 1 ? BaSolvePath::single_cta : BaSolvePath::tiled);
        if (cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess &&
            cudaMemcpy(x, dx, n * sizeof(double), cudaMemcpyDeviceToHost) == cudaSuccess &&
            cudaMemcpy(status, dst, sizeof(int), cudaMemcpyDeviceToHost) == cudaSuccess)
            rc = RGBL_OK;
    }
    cudaFree(dS); cudaFree(db); cudaFree(dz); cudaFree(dx); cudaFree(dw); cudaFree(dst);
    return rc;
}
#endif
#endif  // RGBL_BA_FACTOR_CUH
