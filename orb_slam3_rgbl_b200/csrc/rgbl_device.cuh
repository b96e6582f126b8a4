// Device-side arithmetic shared by the kernels.  Every float/double operation that must reproduce
// the reference's CPU result bit for bit uses explicit round-to-nearest intrinsics so that nvcc can
// never contract it into an FMA (the library is additionally built with -fmad=false).
#ifndef RGBL_DEVICE_CUH
#define RGBL_DEVICE_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "rgbl_internal.h"

namespace rgbl {

#if defined(__CUDACC__)
#define RGBL_HD __host__ __device__ __forceinline__
#else
#define RGBL_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define RGBL_FMUL(a, b) __fmul_rn((a), (b))
#define RGBL_FADD(a, b) __fadd_rn((a), (b))
#define RGBL_FSUB(a, b) __fsub_rn((a), (b))
#define RGBL_FDIV(a, b) __fdiv_rn((a), (b))
#define RGBL_DMUL(a, b) __dmul_rn((a), (b))
#define RGBL_DADD(a, b) __dadd_rn((a), (b))
#define RGBL_DSUB(a, b) __dsub_rn((a), (b))
#define RGBL_DDIV(a, b) __ddiv_rn((a), (b))
#else   // host build of the same header (tests/host_math_harness.cpp); compiled with -ffp-contract=off
#define RGBL_FMUL(a, b) ((float)(a) * (float)(b))
#define RGBL_FADD(a, b) ((float)(a) + (float)(b))
#define RGBL_FSUB(a, b) ((float)(a) - (float)(b))
#define RGBL_FDIV(a, b) ((float)(a) / (float)(b))
#define RGBL_DMUL(a, b) ((double)(a) * (double)(b))
#define RGBL_DADD(a, b) ((double)(a) + (double)(b))
#define RGBL_DSUB(a, b) ((double)(a) - (double)(b))
#define RGBL_DDIV(a, b) ((double)(a) / (double)(b))
#endif

// cv::undistortPoints(src, dst, K, D, noArray(), K) for one CV_32FC2 point, as Frame::UndistortKeyPoints and Frame::ComputeImageBounds
// call it (src/Frame.cc:837-899): OpenCV's cvUndistortPointsInternal (calib3d/src/undistort.dispatch.cpp) in double precision with
// its default criterion (MAX_ITER 5) and the operations in its order.  K = P and R = I, so the tilt matrix and R P are exact identities
// and the final projection is xx = fx x + 0 y + cx, yy = 0 x + fy y + cy, ww = 1 / (0 x + 0 y + 1), each term spelled out so that a
// non-finite intermediate propagates as OpenCV's does.  Pinned against python-cv2 (tests/test_oracle_undistort.py).
RGBL_HD void undistort_point(const UndistortDev& m, float px, float py, float* ox, float* oy) {
    const double* k = m.k;
    const double u = px, v = py;
    double x = RGBL_DMUL(RGBL_DSUB(u, m.cx), m.ifx), y = RGBL_DMUL(RGBL_DSUB(v, m.cy), m.ify);
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; ++j) {
        const double r2 = RGBL_DADD(RGBL_DMUL(x, x), RGBL_DMUL(y, y));
        const double num = RGBL_DADD(1.0, RGBL_DMUL(RGBL_DADD(RGBL_DMUL(RGBL_DADD(RGBL_DMUL(k[7], r2), k[6]), r2), k[5]), r2));
        const double den = RGBL_DADD(1.0, RGBL_DMUL(RGBL_DADD(RGBL_DMUL(RGBL_DADD(RGBL_DMUL(k[4], r2), k[1]), r2), k[0]), r2));
        const double icdist = RGBL_DDIV(num, den);
        if (icdist < 0) {                    // OpenCV's regression_14583 guard: back to the distorted point, no further iteration
            x = RGBL_DMUL(RGBL_DSUB(u, m.cx), m.ifx);
            y = RGBL_DMUL(RGBL_DSUB(v, m.cy), m.ify);
            break;
        }
        const double dx = RGBL_DADD(RGBL_DADD(RGBL_DADD(RGBL_DMUL(RGBL_DMUL(RGBL_DMUL(2.0, k[2]), x), y),
                                                        RGBL_DMUL(k[3], RGBL_DADD(r2, RGBL_DMUL(RGBL_DMUL(2.0, x), x)))),
                                              RGBL_DMUL(k[8], r2)),
                                    RGBL_DMUL(RGBL_DMUL(k[9], r2), r2));
        const double dy = RGBL_DADD(RGBL_DADD(RGBL_DADD(RGBL_DMUL(k[2], RGBL_DADD(r2, RGBL_DMUL(RGBL_DMUL(2.0, y), y))),
                                                        RGBL_DMUL(RGBL_DMUL(RGBL_DMUL(2.0, k[3]), x), y)),
                                              RGBL_DMUL(k[10], r2)),
                                    RGBL_DMUL(RGBL_DMUL(k[11], r2), r2));
        x = RGBL_DMUL(RGBL_DSUB(x0, dx), icdist);
        y = RGBL_DMUL(RGBL_DSUB(y0, dy), icdist);
    }
    const double xx = RGBL_DADD(RGBL_DADD(RGBL_DMUL(m.fx, x), RGBL_DMUL(0.0, y)), m.cx);
    const double yy = RGBL_DADD(RGBL_DADD(RGBL_DMUL(0.0, x), RGBL_DMUL(m.fy, y)), m.cy);
    const double ww = RGBL_DDIV(1.0, RGBL_DADD(RGBL_DADD(RGBL_DMUL(0.0, x), RGBL_DMUL(0.0, y)), 1.0));
    *ox = (float)RGBL_DMUL(xx, ww);
    *oy = (float)RGBL_DMUL(yy, ww);
}

// the camera of rgbl_set_camera_distortion as cvUndistortPointsInternal converts it: float K and mDistCoef (n_dist 4 or 5) to double
RGBL_HD UndistortDev make_undistort_dev(float fx, float fy, float cx, float cy, const float* dist, int n_dist) {
    UndistortDev m{};
    m.fx = fx; m.fy = fy; m.cx = cx; m.cy = cy;
    m.ifx = RGBL_DDIV(1.0, m.fx); m.ify = RGBL_DDIV(1.0, m.fy);
    for (int i = 0; i < 12; ++i) m.k[i] = i < n_dist ? (double)dist[i] : 0.0;
    return m;
}

// Frame::ComputeImageBounds (src/Frame.cc:871-899) of a W x H image: k1 != 0 -> the undistorted corners (0,0), (W,0), (0,H), (W,H),
// mnMinX = min(c0.x, c2.x), mnMaxX = max(c1.x, c3.x), mnMinY = min(c0.y, c1.y), mnMaxY = max(c2.y, c3.y); else (0, W, 0, H).
RGBL_HD void image_bounds(const UndistortDev& m, float k1, int W, int H, float b[4]) {
    const float w = (float)W, h = (float)H;
    if (k1 == 0.f) { b[0] = 0.f; b[1] = w; b[2] = 0.f; b[3] = h; return; }
    const float cxs[4] = {0.f, w, 0.f, w}, cys[4] = {0.f, 0.f, h, h};
    float px[4], py[4];
    for (int i = 0; i < 4; ++i) undistort_point(m, cxs[i], cys[i], &px[i], &py[i]);
    b[0] = (px[2] < px[0]) ? px[2] : px[0];          // std::min(a, b) = (b < a) ? b : a, std::max(a, b) = (a < b) ? b : a
    b[1] = (px[1] < px[3]) ? px[3] : px[1];
    b[2] = (py[1] < py[0]) ? py[1] : py[0];
    b[3] = (py[2] < py[3]) ? py[3] : py[2];
}

// cv::fastAtan2 scalar path (SURVEY A.4), degrees in [0, 360).
RGBL_HD float fast_atan2_deg(float y, float x) {
    const float k = (float)(180.0 / 3.14159265358979323846);
    const float p1 = RGBL_FMUL(0.9997878412794807f, k), p3 = RGBL_FMUL(-0.3258083974640975f, k),
                p5 = RGBL_FMUL(0.1555786518463281f, k), p7 = RGBL_FMUL(-0.04432655554792128f, k);
    const float eps = 2.2204460492503131e-16f;
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = RGBL_FDIV(ay, RGBL_FADD(ax, eps));
        c2 = RGBL_FMUL(c, c);
        a = RGBL_FMUL(RGBL_FADD(RGBL_FMUL(RGBL_FADD(RGBL_FMUL(RGBL_FADD(RGBL_FMUL(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = RGBL_FDIV(ax, RGBL_FADD(ay, eps));
        c2 = RGBL_FMUL(c, c);
        a = RGBL_FSUB(90.f, RGBL_FMUL(RGBL_FADD(RGBL_FMUL(RGBL_FADD(RGBL_FMUL(RGBL_FADD(RGBL_FMUL(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = RGBL_FSUB(180.f, a);
    if (y < 0) a = RGBL_FSUB(360.f, a);
    return a;
}

// glibc >= 2.28 sinf/cosf (the "sincosf" double-precision polynomial algorithm), restated so that the
// device reproduces the libm results the reference's computeOrbDescriptor sees (src/ORBextractor.cc:112).
// Verified bit-identical to glibc 2.39 on every float in [0, 6.4] (tests/test_host_math.py samples it).
// Valid for |y| < 120; descriptor angles are in [0, 2*pi].
RGBL_HD uint32_t f32_top12(float x) {
#if defined(__CUDA_ARCH__)
    return (__float_as_uint(x) >> 20) & 0x7ffu;
#else
    union { float f; uint32_t u; } c; c.f = x; return (c.u >> 20) & 0x7ffu;
#endif
}

RGBL_HD float sincosf_poly(double x, double x2, bool neg_cos, int n) {
    // neg_cos selects the second coefficient table (cosine coefficients negated).
    if ((n & 1) == 0) {
        const double s1c = -0x1.555545995a603p-3, s2c = 0x1.1107605230bc4p-7, s3c = -0x1.994eb3774cf24p-13;
        const double x3 = RGBL_DMUL(x, x2);
        const double s1 = RGBL_DADD(s2c, RGBL_DMUL(x2, s3c));
        const double x7 = RGBL_DMUL(x3, x2);
        const double s = RGBL_DADD(x, RGBL_DMUL(x3, s1c));
        return (float)RGBL_DADD(s, RGBL_DMUL(x7, s1));
    } else {
        const double sg = neg_cos ? -1.0 : 1.0;
        const double c0 = sg * 0x1p0, c1c = sg * -0x1.ffffffd0c621cp-2, c2c = sg * 0x1.55553e1068f19p-5,
                     c3c = sg * -0x1.6c087e89a359dp-10, c4c = sg * 0x1.99343027bf8c3p-16;
        const double x4 = RGBL_DMUL(x2, x2);
        const double c2 = RGBL_DADD(c3c, RGBL_DMUL(x2, c4c));
        const double c1 = RGBL_DADD(c0, RGBL_DMUL(x2, c1c));
        const double x6 = RGBL_DMUL(x4, x2);
        const double c = RGBL_DADD(c1, RGBL_DMUL(x4, c2c));
        return (float)RGBL_DADD(c, RGBL_DMUL(x6, c2));
    }
}

RGBL_HD void glibc_sincosf(float y, float* sin_out, float* cos_out) {
    double x = (double)y;
    if (f32_top12(y) < f32_top12(0x1.921FB6p-1f)) {
        const double s = RGBL_DMUL(x, x);
        if (f32_top12(y) < f32_top12(0x1p-12f)) { *sin_out = y; *cos_out = 1.0f; return; }
        *sin_out = sincosf_poly(x, s, false, 0);
        *cos_out = sincosf_poly(x, s, false, 1);
        return;
    }
    const double hpi_inv = 0x1.45F306DC9C883p+23, hpi = 0x1.921FB54442D18p0;
    const double r = RGBL_DMUL(x, hpi_inv);
    const int n = ((int32_t)r + 0x800000) >> 24;
    x = RGBL_DSUB(x, RGBL_DMUL((double)n, hpi));
    const int q = n & 3;
    const double sgn = (q == 1 || q == 2) ? -1.0 : 1.0;     // sign[] = {1,-1,-1,1}
    const bool second = (n & 2) != 0;
    const double xs = RGBL_DMUL(x, sgn), x2 = RGBL_DMUL(x, x);
    *sin_out = sincosf_poly(xs, x2, second, n);
    *cos_out = sincosf_poly(xs, x2, second, n ^ 1);
}

// FAST-9/16 arc strength K: the largest t such that the pixel is a corner for every threshold < t,
// i.e. max over the 16 contiguous 9-arcs of min(v - r) (bright) and of min(r - v) (dark); cv score = K-1.
// r[k] = ring intensities in OpenCV's ring order (SURVEY A.3), v = centre.
// Formulated on the raw intensities (K = max(v - min_arc max r, max_arc min r - v)) so that no negated
// value ever feeds a 3-input min/max: ptxas 12.9 for sm_100a was observed to drop the negation when it
// fuses max(max(a, -b), c) into VIMNMX3 (first GPU run of this kernel returned K = max(d)).
RGBL_HD int fast_arc_strength16(int v, const int r[16]) {
    int m2[16], M2[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) { m2[s] = min(r[s], r[(s + 1) & 15]); M2[s] = max(r[s], r[(s + 1) & 15]); }
    int m4[16], M4[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) { m4[s] = min(m2[s], m2[(s + 2) & 15]); M4[s] = max(M2[s], M2[(s + 2) & 15]); }
    int lo = 255, hi = 0;
#pragma unroll
    for (int s = 0; s < 16; ++s) {
        const int m8 = min(m4[s], m4[(s + 4) & 15]), M8 = max(M4[s], M4[(s + 4) & 15]);
        const int m9 = min(m8, r[(s + 8) & 15]), M9 = max(M8, r[(s + 8) & 15]);
        lo = min(lo, M9);      // darkest "all-below" bound: arc whose maximum is smallest
        hi = max(hi, m9);      // brightest "all-above" bound: arc whose minimum is largest
    }
    const int kb = v - lo, kd = hi - v;
    return kb > kd ? kb : kd;
}

#if defined(__CUDACC__)
// Sophus::SE3f point action (so3.hpp:358-366, se3.hpp:321-324), float32, no FMA.
__device__ __forceinline__ void se3f_rotate(const float* T, const float p[3], float out[3]) {
    const float qx = T[0], qy = T[1], qz = T[2], qw = T[3];
    float uv[3] = {__fsub_rn(__fmul_rn(qy, p[2]), __fmul_rn(qz, p[1])), __fsub_rn(__fmul_rn(qz, p[0]), __fmul_rn(qx, p[2])),
                   __fsub_rn(__fmul_rn(qx, p[1]), __fmul_rn(qy, p[0]))};
    uv[0] = __fadd_rn(uv[0], uv[0]); uv[1] = __fadd_rn(uv[1], uv[1]); uv[2] = __fadd_rn(uv[2], uv[2]);
    const float c[3] = {__fsub_rn(__fmul_rn(qy, uv[2]), __fmul_rn(qz, uv[1])), __fsub_rn(__fmul_rn(qz, uv[0]), __fmul_rn(qx, uv[2])),
                        __fsub_rn(__fmul_rn(qx, uv[1]), __fmul_rn(qy, uv[0]))};
#pragma unroll
    for (int i = 0; i < 3; ++i) out[i] = __fadd_rn(__fadd_rn(p[i], __fmul_rn(qw, uv[i])), c[i]);
}


// Eigen 3.3 (the reference's Eigen: Ubuntu 20.04 libeigen3-dev) adds the terms of a fixed-size dot product / squared norm / product
// coefficient with its unrolled scalar reduction (Core/Redux.h, redux_novec_unroller: halves, recursively).  Pinned against the
// reference's own code over a stand-in Eigen with the same rule (tests/test_oracle_tracking_ref.py).
__device__ __forceinline__ float eig_sum3(float a, float b, float c) { return __fadd_rn(a, __fadd_rn(b, c)); }
__device__ __forceinline__ float eig_sum4(float a, float b, float c, float d) { return __fadd_rn(__fadd_rn(a, b), __fadd_rn(c, d)); }

// Sophus::SE3f::inverse() (se3.hpp:208-211): invR = SO3f(conjugate), whose quaternion constructor normalises in float
// (so3.hpp:229-231, 481-487, 297-303: coeffs /= norm), translation invR * (t * -1).  qinv = (x, y, z, w), tinv = 3 floats.
__device__ __forceinline__ void se3f_inverse(const float* T, float qinv[4], float tinv[3]) {
    qinv[0] = -T[0]; qinv[1] = -T[1]; qinv[2] = -T[2]; qinv[3] = T[3];
    const float length = sqrtf(eig_sum4(__fmul_rn(qinv[0], qinv[0]), __fmul_rn(qinv[1], qinv[1]), __fmul_rn(qinv[2], qinv[2]), __fmul_rn(qinv[3], qinv[3])));
#pragma unroll
    for (int i = 0; i < 4; ++i) qinv[i] = __fdiv_rn(qinv[i], length);
    const float nt[3] = {__fmul_rn(T[4], -1.f), __fmul_rn(T[5], -1.f), __fmul_rn(T[6], -1.f)};
    se3f_rotate(qinv, nt, tinv);
}

// Sophus::SE3f * SE3f (Thirdparty/Sophus/sophus/se3.hpp:304-308): (Ra Rb, ta + Ra tb).  SO3f * SO3f is the Hamilton product written out in
// so3.hpp:325-339, evaluated left to right in float32; its result goes through the SO3f(quaternion) constructor, which normalises
// (so3.hpp:481-487, 297-303: coeffs /= norm).  Poses are (qx, qy, qz, qw, tx, ty, tz); out may not alias A or B.
__device__ __forceinline__ void se3f_mul(const float* A, const float* B, float* out) {
    const float ax = A[0], ay = A[1], az = A[2], aw = A[3], bx = B[0], by = B[1], bz = B[2], bw = B[3];
    const float w = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(aw, bw), __fmul_rn(ax, bx)), __fmul_rn(ay, by)), __fmul_rn(az, bz));
    const float x = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bx), __fmul_rn(ax, bw)), __fmul_rn(ay, bz)), __fmul_rn(az, by));
    const float y = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, by), __fmul_rn(ay, bw)), __fmul_rn(az, bx)), __fmul_rn(ax, bz));
    const float z = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bz), __fmul_rn(az, bw)), __fmul_rn(ax, by)), __fmul_rn(ay, bx));
    const float length = sqrtf(eig_sum4(__fmul_rn(x, x), __fmul_rn(y, y), __fmul_rn(z, z), __fmul_rn(w, w)));
    out[0] = __fdiv_rn(x, length); out[1] = __fdiv_rn(y, length); out[2] = __fdiv_rn(z, length); out[3] = __fdiv_rn(w, length);
    float r[3];
    se3f_rotate(A, B + 4, r);
    out[4] = __fadd_rn(A[4], r[0]); out[5] = __fadd_rn(A[5], r[1]); out[6] = __fadd_rn(A[6], r[2]);
}

// Tracking::TrackWithMotionModel's initial pose mVelocity * mLastFrame.GetPose() (src/Tracking.cc:2904) with the constant-velocity model
// mVelocity = Tcw(last) * Tcw(prev)^-1 (src/Tracking.cc:2243-2245).  prev == nullptr (no velocity yet): the last pose itself.
__device__ __forceinline__ void predict_pose(const float* prev, const float* last, float* pred) {
    if (!prev) {
#pragma unroll
        for (int i = 0; i < 7; ++i) pred[i] = last[i];
        return;
    }
    float inv[7], vel[7];
    se3f_inverse(prev, inv, inv + 4);
    se3f_mul(last, inv, vel);
    se3f_mul(vel, last, pred);
}

// Eigen QuaternionBase::toRotationMatrix (Geometry/Quaternion.h), float32, row-major R[9]
__device__ __forceinline__ void quatf_to_matrix(const float q[4], float R[9]) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    const float tx = __fmul_rn(2.f, x), ty = __fmul_rn(2.f, y), tz = __fmul_rn(2.f, z);
    const float twx = __fmul_rn(tx, w), twy = __fmul_rn(ty, w), twz = __fmul_rn(tz, w);
    const float txx = __fmul_rn(tx, x), txy = __fmul_rn(ty, x), txz = __fmul_rn(tz, x);
    const float tyy = __fmul_rn(ty, y), tyz = __fmul_rn(tz, y), tzz = __fmul_rn(tz, z);
    R[0] = __fsub_rn(1.f, __fadd_rn(tyy, tzz)); R[1] = __fsub_rn(txy, twz); R[2] = __fadd_rn(txz, twy);
    R[3] = __fadd_rn(txy, twz); R[4] = __fsub_rn(1.f, __fadd_rn(txx, tzz)); R[5] = __fsub_rn(tyz, twx);
    R[6] = __fsub_rn(txz, twy); R[7] = __fadd_rn(tyz, twx); R[8] = __fsub_rn(1.f, __fadd_rn(txx, tyy));
}

// Programmatic dependent launch (PDL): the kernels of the resident tracking chain are launched with the programmatic-stream-serialization
// attribute, so a kernel's CTAs are scheduled while its predecessor still runs and wait HERE until the predecessor's grid has completed
// and its memory is visible; the predecessor releases them early with pdl_trigger().  What is gained is the launch latency between two
// dependent kernels (a frame is a chain of 7).  Both are no-ops for a kernel launched the ordinary way.  Rule: pdl_wait() is the first
// statement of every chain kernel, unconditionally (a CTA that returned without waiting would let the NEXT kernel overtake).
__device__ __forceinline__ void pdl_wait() {
#ifndef RGBL_CUDA_EMU
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_trigger() {
#ifndef RGBL_CUDA_EMU
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}

// barrier of the first `nthreads` threads of a CTA (a multiple of 32; named barrier 1), for phases that only a few warps take part in
__device__ __forceinline__ void team_sync(int nthreads) {
#ifdef RGBL_CUDA_EMU
    emu::named_barrier(nthreads);
#else
    asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
#endif
}

// ---- Frame::isInFrustum (src/Frame.cc:602-664, Nleft == -1) + MapPoint::PredictScale (src/MapPoint.cc:531-545) for one map point.
// Float32, Eigen 3.3's reduction order for mRcw * P, norm() and dot(); pinned against the reference's own function body
// (tests/test_oracle_tracking_ref.py::test_is_in_frustum_and_search_local).
struct FrustumOut { uint8_t in_view; float px, py, pxr, depth, view_cos; int level; };
template <class FrameT, class PrmT>
__device__ __forceinline__ FrustumOut frustum_point(const FrameT& f, const PrmT& prm, const float P[3], const float* Pn, float mf_min, float mf_max) {
    FrustumOut o; o.in_view = 0; o.px = -1.f; o.py = -1.f; o.pxr = 0.f; o.depth = 0.f; o.view_cos = 0.f; o.level = 0;
    float Pc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        Pc[r] = __fadd_rn(eig_sum3(__fmul_rn(prm.Rcw[3 * r], P[0]), __fmul_rn(prm.Rcw[3 * r + 1], P[1]), __fmul_rn(prm.Rcw[3 * r + 2], P[2])), prm.tcw[r]);
    const float pc_dist = sqrtf(eig_sum3(__fmul_rn(Pc[0], Pc[0]), __fmul_rn(Pc[1], Pc[1]), __fmul_rn(Pc[2], Pc[2])));
    const float z = Pc[2];
    const float invz = __fdiv_rn(1.0f, z);
    bool ok = !(z < 0.0f);
    const float u = __fadd_rn(__fdiv_rn(__fmul_rn(f.fx, Pc[0]), Pc[2]), f.cx);
    const float v = __fadd_rn(__fdiv_rn(__fmul_rn(f.fy, Pc[1]), Pc[2]), f.cy);
    if (ok && (u < f.min_x || u > f.max_x)) ok = false;
    if (ok && (v < f.min_y || v > f.max_y)) ok = false;
    if (ok) {
        o.px = u; o.py = v;
        const float PO[3] = {__fsub_rn(P[0], prm.Ow[0]), __fsub_rn(P[1], prm.Ow[1]), __fsub_rn(P[2], prm.Ow[2])};
        const float dist = sqrtf(eig_sum3(__fmul_rn(PO[0], PO[0]), __fmul_rn(PO[1], PO[1]), __fmul_rn(PO[2], PO[2])));
        if (!(dist < __fmul_rn(0.8f, mf_min) || dist > __fmul_rn(1.2f, mf_max))) {
            const float vc = __fdiv_rn(eig_sum3(__fmul_rn(PO[0], Pn[0]), __fmul_rn(PO[1], Pn[1]), __fmul_rn(PO[2], Pn[2])), dist);
            if (!(vc < prm.cos_limit)) {
                const float ratio = __fdiv_rn(mf_max, dist);
                const float lg = (float)log((double)ratio);          // correctly-rounded stand-in for glibc logf
                int ns = (int)ceilf(__fdiv_rn(lg, f.log_scale_factor));
                if (ns < 0) ns = 0; else if (ns >= f.n_levels) ns = f.n_levels - 1;
                o.in_view = 1; o.pxr = __fsub_rn(u, __fmul_rn(f.bf, invz)); o.depth = pc_dist; o.level = ns; o.view_cos = vc;
            }
        }
    }
    return o;
}

// ---- resident tracking chain: the previous frame's LiDAR-depth keypoints as map points -----------------------------------
// Frame::UnprojectStereo (src/Frame.cc:1137-1150: x3D = mRwc * x3Dc + mOw, with mRwc / mOw from Frame::UpdatePoseMatrices
// :562-569) with the frame's estimated pose, the bForward / bBackward test of SearchByProjection (src/ORBmatcher.cc:1686-1693)
// and the per-point fields the search reads.  Shared by chain_prep_kernel and the tail of pose_optimize_kernel (which prepares
// the next frame's search as soon as the pose is known: one launch less).
struct ChainPrepDev {
    const rgbl_keypoint* kps; const float* depth; const int* n_ptr;      // kps == nullptr: disabled
    float fx, fy, cx, cy, mb; int mono, cap;
    uint8_t* valid; float* xw; int* octave; float* angle; uint8_t* obs_pos; int* flags; uint8_t* state_clear;
    const float* prev_pose;          // pose of the frame BEFORE the one being prepared (nullptr: no velocity yet)
    float* pred_pose;                // out: the motion model's pose for the next frame = where its search projects and its optimisation starts
};

// one thread: the next frame's predicted pose and the bForward / bBackward flags of its search (last_pose = the pose of the frame being prepared)
__device__ __forceinline__ void chain_prep_motion(const ChainPrepDev& cp, const float* last_pose) {
    float cur_pose[7];
    predict_pose(cp.prev_pose, last_pose, cur_pose);
#pragma unroll
    for (int i = 0; i < 7; ++i) cp.pred_pose[i] = cur_pose[i];
    // tlc = Tlw * (Tcw^-1).translation()
    float cinv[4], twc[3], r[3];
    se3f_inverse(cur_pose, cinv, twc);
    se3f_rotate(last_pose, twc, r);
    const float tlc_z = __fadd_rn(r[2], last_pose[6]);
    cp.flags[0] = (tlc_z > cp.mb && !cp.mono) ? 1 : 0;
    cp.flags[1] = (-tlc_z > cp.mb && !cp.mono) ? 1 : 0;
}

// Rwc (row-major) and Ow of a pose, once per CTA / caller (Frame::UpdatePoseMatrices)
__device__ __forceinline__ void chain_pose_matrices(const float* pose, float Rwc[9], float Ow[3]) {
    float qinv[4];
    se3f_inverse(pose, qinv, Ow);
    quatf_to_matrix(qinv, Rwc);
}

__device__ __forceinline__ void chain_prep_item(const ChainPrepDev& cp, const float Rwc[9], const float Ow[3], int i) {
    if (cp.state_clear) cp.state_clear[i] = 0;           // feature states of the search that follows (saves a memset node)
    uint8_t v = 0;
    if (i < *cp.n_ptr) {
        const float z = cp.depth[i];
        const rgbl_keypoint kp = cp.kps[i];
        cp.octave[i] = kp.octave; cp.angle[i] = kp.angle; cp.obs_pos[i] = 1;
        if (z > 0.f) {
            const float invfx = __fdiv_rn(1.0f, cp.fx), invfy = __fdiv_rn(1.0f, cp.fy);
            const float pc[3] = {__fmul_rn(__fmul_rn(__fsub_rn(kp.x, cp.cx), z), invfx), __fmul_rn(__fmul_rn(__fsub_rn(kp.y, cp.cy), z), invfy), z};
#pragma unroll
            for (int r = 0; r < 3; ++r)
                cp.xw[3 * i + r] = __fadd_rn(eig_sum3(__fmul_rn(Rwc[3 * r], pc[0]), __fmul_rn(Rwc[3 * r + 1], pc[1]), __fmul_rn(Rwc[3 * r + 2], pc[2])), Ow[r]);
            v = 1;
        }
    }
    cp.valid[i] = v;
}
#endif  // __CUDACC__

}  // namespace rgbl
#endif
