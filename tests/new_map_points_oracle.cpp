// ORACLE (test infrastructure, NOT product code): CPU restatement of LocalMapping::CreateNewMapPoints (src/LocalMapping.cc,
// Nleft == -1, no IMU, mbMonocular false) over the neighbours the caller passes, one neighbour at a time with has_mp1 carried
// here, as the reference does it.  Its search is oracle/mapping_oracle.cpp's orc_search_for_triangulation, passed in as a
// function pointer so that this file needs no link step against the oracle library.
//   GeometricTools::Triangulate        src/GeometricTools.cc, over Eigen 3.4 JacobiSVD<Matrix4f> (SVD/JacobiSVD.h,
//                                      Jacobi/RealSvd2x2.h, Jacobi/Jacobi.h) restated below
//   KeyFrame::UnprojectStereo          src/KeyFrame.cc
//   Pinhole::unprojectEig / project    src/CameraModels/Pinhole.cpp
//   Sophus SE3f / SO3f                 Thirdparty/Sophus/sophus/se3.hpp, so3.hpp (GetPose's rotation matrix, GetCameraCenter, mRwc)
// Float32 throughout, Eigen 3.3's reduction order for 3-term sums (a + (b + c)), no FMA (built with -ffp-contract=off).
// PARITY UNPINNED against the reference's own build: its Eigen version is not pinned and Eigen is not available to this build.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct KeyPoint { float x, y, size, angle, response; int octave, class_id; };
struct View {                       // = rgbl_keyframe_view
    int32_t n; const uint8_t* desc; const KeyPoint* keys; const KeyPoint* keys_un; const float* uright; const float* depth; const uint8_t* has_mp;
    int32_t n_nodes; const uint32_t* node_ids; const int32_t* node_start; const int32_t* node_feat; float Tcw[7];
};
typedef int (*SearchFn)(int, const uint8_t*, const void*, const uint8_t*, const float*, int, const uint32_t*, const int*, const int*, int, const uint8_t*,
                        const void*, const uint8_t*, const float*, int, const uint32_t*, const int*, const int*, const float*, const float*, const float*,
                        const float*, int, int, int, int32_t*);

inline float sum3(float a, float b, float c) { return a + (b + c); }
inline float sum4(float a, float b, float c, float d) { return (a + b) + (c + d); }
inline float dot3(const float* a, const float* b) { return sum3(a[0] * b[0], a[1] * b[1], a[2] * b[2]); }

// Eigen QuaternionBase::toRotationMatrix, row-major
void quat_to_matrix(const float* q, float R[9]) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z, twx = tx * w, twy = ty * w, twz = tz * w;
    const float txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.f - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.f - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.f - (txx + tyy);
}

// SO3f action: Eigen's _transformVector (uv = 2 q.vec x p; p + w uv + q.vec x uv)
void quat_rotate(const float* q, const float p[3], float out[3]) {
    float uv[3] = {q[1] * p[2] - q[2] * p[1], q[2] * p[0] - q[0] * p[2], q[0] * p[1] - q[1] * p[0]};
    for (float& u : uv) u = u + u;
    const float c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
    for (int i = 0; i < 3; ++i) out[i] = (p[i] + q[3] * uv[i]) + c[i];
}

// mTwc = mTcw.inverse(): the normalised conjugate quaternion (-> mRwc) and the camera centre (GetCameraCenter)
void pose_inverse(const float* T, float Rwc[9], float Ow[3]) {
    float q[4] = {-T[0], -T[1], -T[2], T[3]};
    const float len = std::sqrt(sum4(q[0] * q[0], q[1] * q[1], q[2] * q[2], q[3] * q[3]));
    for (float& v : q) v = v / len;
    const float nt[3] = {T[4] * -1.f, T[5] * -1.f, T[6] * -1.f};
    quat_rotate(q, nt, Ow);
    quat_to_matrix(q, Rwc);
}

// apply_rotation_in_the_plane(x, y, (c, s)) over len entries with strides: x' = c x + s y, y' = -s x + c y
void rotate_plane(float* x, float* y, int stride, float c, float s, int len = 4) {
    if (c == 1.f && s == 0.f) return;
    for (int k = 0; k < len; ++k) {
        const float xi = x[k * stride], yi = y[k * stride];
        x[k * stride] = c * xi + s * yi;
        y[k * stride] = -s * xi + c * yi;
    }
}

// Eigen 3.4 JacobiSVD<Matrix4f>(A, ComputeFullV), square: no preconditioner; -> column 3 of V after the descending sort.
// false for a non-finite A (Eigen: InvalidInput), or after 64 sweeps without convergence (Eigen has no limit).
bool jacobi_svd4_null(const float A[4][4], float v3[4]) {
    float scale = 0.f;
    for (int i = 0; i < 4; ++i) for (int k = 0; k < 4; ++k) { if (!std::isfinite(A[i][k])) return false; scale = std::max(scale, std::fabs(A[i][k])); }
    if (scale == 0.f) scale = 1.f;
    float W[4][4], V[4][4];
    for (int i = 0; i < 4; ++i) for (int k = 0; k < 4; ++k) { W[i][k] = A[i][k] / scale; V[i][k] = i == k ? 1.f : 0.f; }
    const float precision = 2.f * FLT_EPSILON, consider_zero = FLT_MIN;
    float max_diag = 0.f;
    for (int i = 0; i < 4; ++i) max_diag = std::max(max_diag, std::fabs(W[i][i]));
    bool finished = false;
    for (int sweep = 0; sweep < 64 && !finished; ++sweep) {
        finished = true;
        for (int p = 1; p < 4; ++p) {
            for (int q = 0; q < p; ++q) {
                const float threshold = std::max(consider_zero, precision * max_diag);
                if (!(std::fabs(W[p][q]) > threshold || std::fabs(W[q][p]) > threshold)) continue;
                finished = false;
                // real_2x2_jacobi_svd(W, p, q, &j_left, &j_right)
                float m[2][2] = {{W[p][p], W[p][q]}, {W[q][p], W[q][q]}};
                const float t = m[0][0] + m[1][1], d = m[1][0] - m[0][1];
                float c1, s1;
                if (std::fabs(d) < FLT_MIN) { s1 = 0.f; c1 = 1.f; }
                else { const float u = t / d, tmp = std::sqrt(1.f + u * u); s1 = 1.f / tmp; c1 = u / tmp; }
                rotate_plane(&m[0][0], &m[1][0], 1, c1, s1, 2);            // m.applyOnTheLeft(0, 1, rot1)
                float cr, sr;                                              // makeJacobi(m(0,0), m(0,1), m(1,1))
                const float x = m[0][0], y = m[0][1], z = m[1][1], deno = 2.f * std::fabs(y);
                if (deno < FLT_MIN) { cr = 1.f; sr = 0.f; }
                else {
                    const float tau = (x - z) / deno, w = std::sqrt(tau * tau + 1.f);
                    const float tt = tau > 0.f ? 1.f / (tau + w) : 1.f / (tau - w);
                    const float sign_t = tt > 0.f ? 1.f : -1.f, n = 1.f / std::sqrt(tt * tt + 1.f);
                    sr = -sign_t * (y / std::fabs(y)) * std::fabs(tt) * n;
                    cr = n;
                }
                const float cl = c1 * cr - s1 * -sr, sl = c1 * -sr + s1 * cr;   // rot1 * j_right.transpose()
                rotate_plane(&W[p][0], &W[q][0], 1, cl, sl);               // W.applyOnTheLeft(p, q, j_left)
                rotate_plane(&W[0][p], &W[0][q], 4, cr, -sr);              // W.applyOnTheRight(p, q, j_right)
                rotate_plane(&V[0][p], &V[0][q], 4, cr, -sr);              // V.applyOnTheRight(p, q, j_right)
                max_diag = std::max(max_diag, std::max(std::fabs(W[p][p]), std::fabs(W[q][q])));
            }
        }
    }
    if (!finished) return false;
    float sv[4];
    for (int i = 0; i < 4; ++i) sv[i] = std::fabs(W[i][i]) * scale;
    for (int i = 0; i < 4; ++i) {
        int pos = i;
        for (int k = i + 1; k < 4; ++k) if (sv[k] > sv[pos]) pos = k;
        if (sv[pos] == 0.f) break;
        if (pos != i) { std::swap(sv[i], sv[pos]); for (int r = 0; r < 4; ++r) std::swap(V[r][i], V[r][pos]); }
    }
    for (int r = 0; r < 4; ++r) v3[r] = V[r][3];
    return true;
}

}  // namespace

extern "C" {

// Route and result codes of one candidate match, written to the optional trace (one entry per match of every pair, in pair order,
// ascending idx1): route 0 = neither (low parallax, no stereo), 1 = Triangulate, 2 = UnprojectStereo of key frame 1, 3 = of
// key frame 2; result 0 = created, else the first failed check.
enum { R_OK = 0, R_LOW_PARALLAX, R_SVD_W0, R_NO_DEPTH, R_BEHIND1, R_BEHIND2, R_REPROJ1, R_REPROJ2, R_DIST0, R_FAR, R_SCALE, R_SVD_FAIL };

int orc_create_new_map_points(void* search_fn, const View* kf1, int np, const View* kf2, const float* F12, const float* ep, float fx, float fy, float cx, float cy,
                              float bf, int n_levels, const float* sf, const float* sg, float th_far, int check_orientation, int coarse,
                              int32_t* created_start, int32_t* out_idx1, int32_t* out_idx2, float* out_x3d, int cap, int32_t* n_matches,
                              int32_t* trace /* nullable: [np * kf1->n][6] = pair, idx1, idx2, route, result, stereo flags */, int32_t* n_trace) {
    (void)n_levels;
    SearchFn search = reinterpret_cast<SearchFn>(search_fn);
    const int n1 = kf1->n;
    std::vector<uint8_t> has_mp1(kf1->has_mp, kf1->has_mp + n1);
    std::vector<int32_t> match(std::max(n1, 1));
    float Rcw1[9], Rwc1s[9], Ow1[3];
    quat_to_matrix(kf1->Tcw, Rcw1); pose_inverse(kf1->Tcw, Rwc1s, Ow1);
    const float* tcw1 = kf1->Tcw + 4;
    const float mb = bf / fx, invfx = 1.0f / fx, invfy = 1.0f / fy, ratio_factor = 1.5f * sf[1];
    int created = 0, nt = 0;
    created_start[0] = 0;
    for (int j = 0; j < np; ++j) {
        const View& v2 = kf2[j];
        const int nm = search(n1, kf1->desc, kf1->keys_un, has_mp1.data(), kf1->uright, kf1->n_nodes, kf1->node_ids, kf1->node_start, kf1->node_feat,
                              v2.n, v2.desc, v2.keys_un, v2.has_mp, v2.uright, v2.n_nodes, v2.node_ids, v2.node_start, v2.node_feat, F12 + 9 * j, ep + 2 * j,
                              sf, sg, 0, coarse, check_orientation, match.data());
        if (n_matches) n_matches[j] = nm;
        float Rcw2[9], Rwc2s[9], Ow2[3];
        quat_to_matrix(v2.Tcw, Rcw2); pose_inverse(v2.Tcw, Rwc2s, Ow2);
        const float* tcw2 = v2.Tcw + 4;
        for (int idx1 = 0; idx1 < n1; ++idx1) {                    // vMatchedPairs: ascending idx1
            const int idx2 = match[idx1];
            if (idx2 < 0) continue;
            const KeyPoint& kp1 = kf1->keys_un[idx1];
            const KeyPoint& kp2 = v2.keys_un[idx2];
            const float kp1_ur = kf1->uright[idx1], kp2_ur = v2.uright[idx2];
            const bool bStereo1 = kp1_ur >= 0, bStereo2 = kp2_ur >= 0;
            const float xn1[3] = {(kp1.x - cx) / fx, (kp1.y - cy) / fy, 1.f};
            const float xn2[3] = {(kp2.x - cx) / fx, (kp2.y - cy) / fy, 1.f};
            float ray1[3], ray2[3];
            for (int r = 0; r < 3; ++r) {
                ray1[r] = sum3(Rcw1[r] * xn1[0], Rcw1[3 + r] * xn1[1], Rcw1[6 + r] * xn1[2]);
                ray2[r] = sum3(Rcw2[r] * xn2[0], Rcw2[3 + r] * xn2[1], Rcw2[6 + r] * xn2[2]);
            }
            const float cosParallaxRays = dot3(ray1, ray2) / (std::sqrt(dot3(ray1, ray1)) * std::sqrt(dot3(ray2, ray2)));
            float cosParallaxStereo = cosParallaxRays + 1;
            float cosParallaxStereo1 = cosParallaxStereo, cosParallaxStereo2 = cosParallaxStereo;
            if (bStereo1) cosParallaxStereo1 = (float)std::cos(2 * std::atan2((double)(mb / 2), (double)kf1->depth[idx1]));
            else if (bStereo2) cosParallaxStereo2 = (float)std::cos(2 * std::atan2((double)(mb / 2), (double)v2.depth[idx2]));
            cosParallaxStereo = std::min(cosParallaxStereo1, cosParallaxStereo2);
            float x3D[3];
            int route = 0, result = R_OK;
            if (cosParallaxRays < cosParallaxStereo && cosParallaxRays > 0 && (bStereo1 || bStereo2 || cosParallaxRays < 0.9998)) {
                route = 1;
                float A[4][4];
                for (int k = 0; k < 4; ++k) {                      // Tc1w / Tc2w as 3 x 4 [R | t]
                    const float a0 = k < 3 ? Rcw1[k] : tcw1[0], a1 = k < 3 ? Rcw1[3 + k] : tcw1[1], a2 = k < 3 ? Rcw1[6 + k] : tcw1[2];
                    const float b0 = k < 3 ? Rcw2[k] : tcw2[0], b1 = k < 3 ? Rcw2[3 + k] : tcw2[1], b2 = k < 3 ? Rcw2[6 + k] : tcw2[2];
                    A[0][k] = xn1[0] * a2 - a0; A[1][k] = xn1[1] * a2 - a1; A[2][k] = xn2[0] * b2 - b0; A[3][k] = xn2[1] * b2 - b1;
                }
                float v[4];
                if (!jacobi_svd4_null(A, v)) result = R_SVD_FAIL;
                else if (v[3] == 0) result = R_SVD_W0;
                else { x3D[0] = v[0] / v[3]; x3D[1] = v[1] / v[3]; x3D[2] = v[2] / v[3]; }
            } else if (bStereo1 && cosParallaxStereo1 < cosParallaxStereo2) {
                route = 2;
                const float z = kf1->depth[idx1];
                if (z > 0) {
                    const float xc[3] = {(kf1->keys[idx1].x - cx) * z * invfx, (kf1->keys[idx1].y - cy) * z * invfy, z};
                    for (int r = 0; r < 3; ++r) x3D[r] = dot3(Rwc1s + 3 * r, xc) + Ow1[r];
                } else result = R_NO_DEPTH;
            } else if (bStereo2 && cosParallaxStereo2 < cosParallaxStereo1) {
                route = 3;
                const float z = v2.depth[idx2];
                if (z > 0) {
                    const float xc[3] = {(v2.keys[idx2].x - cx) * z * invfx, (v2.keys[idx2].y - cy) * z * invfy, z};
                    for (int r = 0; r < 3; ++r) x3D[r] = dot3(Rwc2s + 3 * r, xc) + Ow2[r];
                } else result = R_NO_DEPTH;
            } else {
                result = R_LOW_PARALLAX;
            }
            if (result == R_OK) {
                const float z1 = dot3(Rcw1 + 6, x3D) + tcw1[2], z2 = dot3(Rcw2 + 6, x3D) + tcw2[2];
                if (z1 <= 0) result = R_BEHIND1;
                else if (z2 <= 0) result = R_BEHIND2;
                else {
                    auto reproj_ok = [&](const float* Rcw, const float* tcw, float z, const KeyPoint& kp, bool st, float ur) {
                        const float sigmaSquare = sg[kp.octave];
                        const float x = dot3(Rcw, x3D) + tcw[0], y = dot3(Rcw + 3, x3D) + tcw[1];
                        const float invz = 1.0 / z;
                        if (!st) {
                            const float u = fx * x / z + cx, v = fy * y / z + cy;     // Pinhole::project
                            const float errX = u - kp.x, errY = v - kp.y;
                            return !((errX * errX + errY * errY) > 5.991 * sigmaSquare);
                        }
                        const float u = fx * x * invz + cx, u_r = u - bf * invz, v = fy * y * invz + cy;
                        const float errX = u - kp.x, errY = v - kp.y, errX_r = u_r - ur;
                        return !((errX * errX + errY * errY + errX_r * errX_r) > 7.8 * sigmaSquare);
                    };
                    if (!reproj_ok(Rcw1, tcw1, z1, kp1, bStereo1, kp1_ur)) result = R_REPROJ1;
                    else if (!reproj_ok(Rcw2, tcw2, z2, kp2, bStereo2, kp2_ur)) result = R_REPROJ2;
                    else {
                        const float n1v[3] = {x3D[0] - Ow1[0], x3D[1] - Ow1[1], x3D[2] - Ow1[2]};
                        const float n2v[3] = {x3D[0] - Ow2[0], x3D[1] - Ow2[1], x3D[2] - Ow2[2]};
                        const float dist1 = std::sqrt(dot3(n1v, n1v)), dist2 = std::sqrt(dot3(n2v, n2v));
                        if (dist1 == 0 || dist2 == 0) result = R_DIST0;
                        else if (th_far > 0 && (dist1 >= th_far || dist2 >= th_far)) result = R_FAR;
                        else {
                            const float ratioDist = dist2 / dist1, ratioOctave = sf[kp1.octave] / sf[kp2.octave];
                            if (ratioDist * ratio_factor < ratioOctave || ratioDist > ratioOctave * ratio_factor) result = R_SCALE;
                        }
                    }
                }
            }
            if (trace) {
                int32_t* t = trace + 6 * nt;
                t[0] = j; t[1] = idx1; t[2] = idx2; t[3] = route; t[4] = result; t[5] = (bStereo1 ? 1 : 0) | (bStereo2 ? 2 : 0);
            }
            ++nt;
            if (result != R_OK) continue;
            if (created >= cap) return -3;                          // RGBL_E_CAPACITY
            out_idx1[created] = idx1; out_idx2[created] = idx2;
            for (int r = 0; r < 3; ++r) out_x3d[3 * created + r] = x3D[r];
            ++created;
            has_mp1[idx1] = 1;                                      // pKF1->AddMapPoint: later neighbours skip this feature
        }
        created_start[j + 1] = created;
    }
    if (n_trace) *n_trace = nt;
    return 0;
}

}  // extern "C"
