// ORACLE (test infrastructure): cv::undistortPoints(src, dst, K, D, noArray(), K) for CV_32FC2 points, the call of
// Frame::UndistortKeyPoints and Frame::ComputeImageBounds (src/Frame.cc:837-899), restated from OpenCV's cvUndistortPointsInternal
// (calib3d/src/undistort.dispatch.cpp): the camera matrix and distortion converted to double, ifx = 1./fx, the default criterion
// TermCriteria(MAX_ITER, 5), the icdist < 0 guard, then the projection with RR = P * I.  The tilt compensation of that function is the
// identity for k[12] = k[13] = 0 and is left out.  Compiled with -ffp-contract=off; pinned against python-cv2 in
// tests/test_oracle_undistort.py.
#include <algorithm>
#include <cstdint>

namespace {

void undistort_one(const double A[4], const double k[14], float px, float py, float* ox, float* oy) {
    const double fx = A[0], fy = A[1], cx = A[2], cy = A[3];
    const double ifx = 1. / fx, ify = 1. / fy;
    // RR = P * R with P = K (3x3) and R = I
    const double RR[3][3] = {{fx, 0., cx}, {0., fy, cy}, {0., 0., 1.}};
    double x = px, y = py;
    const double u = x, v = y;
    x = (x - cx) * ifx;
    y = (y - cy) * ify;
    const double x0 = x, y0 = y;
    for (int j = 0; j < 5; j++) {
        double r2 = x * x + y * y;
        double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
        if (icdist < 0) {
            x = (u - cx) * ifx;
            y = (v - cy) * ify;
            break;
        }
        double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
        double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
        x = (x0 - deltaX) * icdist;
        y = (y0 - deltaY) * icdist;
    }
    double xx = RR[0][0] * x + RR[0][1] * y + RR[0][2];
    double yy = RR[1][0] * x + RR[1][1] * y + RR[1][2];
    double ww = 1. / (RR[2][0] * x + RR[2][1] * y + RR[2][2]);
    *ox = (float)(xx * ww);
    *oy = (float)(yy * ww);
}

void load(const float K[4], const float* dist, int n_dist, double A[4], double k[14]) {
    for (int i = 0; i < 4; ++i) A[i] = K[i];
    for (int i = 0; i < 14; ++i) k[i] = i < n_dist ? (double)dist[i] : 0.;
}

}  // namespace

extern "C" {

// xy: n x 2 float (x, y) -> out: n x 2.  K = (fx, fy, cx, cy); dist: n_dist (4, 5, 8 or 12) coefficients in OpenCV's order (14, the tilted
// sensor model, is not restated).
int orc_undistort_points(const float* xy, int n, const float K[4], const float* dist, int n_dist, float* out) {
    if (n_dist != 4 && n_dist != 5 && n_dist != 8 && n_dist != 12) return -1;
    double A[4], k[14];
    load(K, dist, n_dist, A, k);
    for (int i = 0; i < n; ++i) undistort_one(A, k, xy[2 * i], xy[2 * i + 1], &out[2 * i], &out[2 * i + 1]);
    return 0;
}

// Frame::ComputeImageBounds (src/Frame.cc:871-899) of a W x H image -> mnMinX, mnMaxX, mnMinY, mnMaxY
int orc_image_bounds(int W, int H, const float K[4], const float* dist, int n_dist, float* bounds) {
    if (n_dist < 4) return -1;
    if (dist[0] != 0.f) {
        const float c[8] = {0.f, 0.f, (float)W, 0.f, 0.f, (float)H, (float)W, (float)H};
        float m[8];
        const int rc = orc_undistort_points(c, 4, K, dist, n_dist, m);
        if (rc) return rc;
        bounds[0] = std::min(m[0], m[4]);
        bounds[1] = std::max(m[2], m[6]);
        bounds[2] = std::min(m[1], m[3]);
        bounds[3] = std::max(m[5], m[7]);
    } else {
        bounds[0] = 0.f; bounds[1] = (float)W; bounds[2] = 0.f; bounds[3] = (float)H;
    }
    return 0;
}

}  // extern "C"
