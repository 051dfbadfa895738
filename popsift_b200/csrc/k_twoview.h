// The math of ps_two_view_config_batch (include/popsift_b200_twoview.h), in double: the unit rays and Kabsch's rotation
// of step 3, the pure-rotation test, the calibrated homography, its normalisation and its decomposition into (R, t, n)
// with the n_z > 0 pruning of step 4, and the triangulation angle of step 6.  One definition for the kernel
// (k_twoview.cu) and the host check (tests/cpp/twoview_math_check.cpp).
#pragma once
#include "k_pose_solve.h"

namespace psb {

constexpr double kTvNoParallax = 1e-9;     // sigma1 - sigma3 <= this times sigma2: the homography has no parallax
// the configurations, PS_TV_* of the header (k_twoview.cu checks that they agree)
constexpr int kTvDegenerate = 0, kTvGeneral = 1, kTvPlanar = 2, kTvPanoramic = 3, kTvUncalibrated = 4;

// (x, y, 1) / |(x, y, 1)|
PSV_HD void tv_ray(double x, double y, double* a)
{
    const double k = 1.0 / sqrt(x * x + y * y + 1.0);
    a[0] = x * k; a[1] = y * k; a[2] = k;
}

// B += b a^T (row-major)
PSV_HD void tv_outer_acc(const double* b, const double* a, double* B)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) B[3 * i + j] += b[i] * a[j];
}

// Kabsch: the rotation R0 = U V^T of B = U S V^T (pose_svd: det U = det V = +1), which maximises tr(R^T B); false when B
// has rank < 2
PSV_HD bool tv_kabsch(const double (&B)[9], double* R0)
{
    double U[3][3], V[3][3];
    if (!pose_svd(B, U, V)) return false;
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) R0[3 * a + b] = U[0][a] * V[0][b] + U[1][a] * V[1][b] + U[2][a] * V[2][b];
    return true;
}

// step 3's rotation test of one row: w = R0 (x^_l, y^_l, 1); w_z > 0 and the squared pixel transfer error in the right
// image below thr2
PSV_HD bool tv_rotation_ok(const double* R0, const PCam& K, double xl, double yl, double xr_px, double yr_px, double thr2)
{
    const double w0 = R0[0] * xl + R0[1] * yl + R0[2], w1 = R0[3] * xl + R0[4] * yl + R0[5], w2 = R0[6] * xl + R0[7] * yl + R0[8];
    if (!(w2 > 0.0)) return false;
    const double du = K.fxr * (w0 / w2) + K.cxr - xr_px, dv = K.fyr * (w1 / w2) + K.cyr - yr_px;
    return du * du + dv * dv < thr2;
}

// H_c = K_r^-1 H K_l (H in pixels, left to right)
PSV_HD void tv_h_calibrated(const double* H, const PCam& K, double* Hc)
{
    double M[9];
    for (int r = 0; r < 3; ++r) {
        M[3 * r] = H[3 * r] * K.fxl;
        M[3 * r + 1] = H[3 * r + 1] * K.fyl;
        M[3 * r + 2] = H[3 * r] * K.cxl + H[3 * r + 1] * K.cyl + H[3 * r + 2];
    }
    for (int c = 0; c < 3; ++c) {
        Hc[c] = (M[c] - K.cxr * M[6 + c]) / K.fxr;
        Hc[3 + c] = (M[3 + c] - K.cyr * M[6 + c]) / K.fyr;
        Hc[6 + c] = M[6 + c];
    }
}

// singular values s[0] >= s[1] >= s[2] of H (square roots of the eigenvalues of H^T H by pose_jacobi3, negative
// eigenvalues taken as 0) and the right singular vectors V[k], each signed so that its first entry of largest magnitude is
// positive; false when not finite
PSV_HD bool tv_h_svd(const double* H, double* s, double (&V)[3][3])
{
    double S[9], Q[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) S[3 * a + b] = H[a] * H[b] + H[3 + a] * H[3 + b] + H[6 + a] * H[6 + b];
    pose_jacobi3(S, Q);
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2 - i; ++j)
            if (S[4 * o[j + 1]] > S[4 * o[j]]) { const int t = o[j]; o[j] = o[j + 1]; o[j + 1] = t; }
    for (int k = 0; k < 3; ++k) {
        s[k] = sqrt(fmax(S[4 * o[k]], 0.0));
        int m = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(Q[3 * r + o[k]]) > fabs(Q[3 * m + o[k]])) m = r;
        const double sg = Q[3 * m + o[k]] < 0.0 ? -1.0 : 1.0;
        for (int r = 0; r < 3; ++r) V[k][r] = sg * Q[3 * r + o[k]];
    }
    return isfinite(s[0]) && isfinite(s[1]) && isfinite(s[2]);
}

// H divided by its middle singular value; false when that is not finite and > 0
PSV_HD bool tv_h_normalise(const double* H, double* Hn)
{
    double s[3], V[3][3];
    if (!tv_h_svd(H, s, V) || !(s[1] > 0.0)) return false;
    for (int j = 0; j < 9; ++j) Hn[j] = H[j] / s[1];
    return true;
}

// x_r^T H x_l of a calibrated row
PSV_HD double tv_h_side(const double* H, double xl, double yl, double xr, double yr)
{
    const double u = H[0] * xl + H[1] * yl + H[2], v = H[3] * xl + H[4] * yl + H[5], w = H[6] * xl + H[7] * yl + H[8];
    return xr * u + yr * v + w;
}

// The four (R, t, n) with H = R + t n^T, |n| = 1, of a normalised, signed H (Ma-Soatto-Kosecka-Sastry 5.3): with v1, v2,
// v3 the right singular vectors (tv_h_svd) and s1 >= s2 >= s3,
//   u+- = (sqrt(s2^2 - s3^2) v1 +- sqrt(s1^2 - s2^2) v3) / sqrt(s1^2 - s3^2),
//   U = [v2, u, v2 x u], W = [H v2, H u, H v2 x H u], R = W U^T, n = v2 x u, t = (H - R) n,
// in order (u+, n, t), (u-, n, t), (u+, -n, -t), (u-, -n, -t).  Returns 4; 0 when s1 - s3 <= kTvNoParallax s2 (no
// parallax: H is a rotation); -1 when the SVD fails.
PSV_HD int tv_h_decompose(const double* H, double (&R)[4][9], double (&t)[4][3], double (&n)[4][3])
{
    double s[3], V[3][3];
    if (!tv_h_svd(H, s, V)) return -1;
    if (!(s[0] - s[2] > kTvNoParallax * s[1])) return 0;
    const double d13 = s[0] * s[0] - s[2] * s[2];
    const double a = sqrt(fmax(s[1] * s[1] - s[2] * s[2], 0.0) / d13), b = sqrt(fmax(s[0] * s[0] - s[1] * s[1], 0.0) / d13);
    double Hv2[3];
    for (int r = 0; r < 3; ++r) Hv2[r] = H[3 * r] * V[1][0] + H[3 * r + 1] * V[1][1] + H[3 * r + 2] * V[1][2];
    for (int k = 0; k < 2; ++k) {
        const double sg = k == 0 ? 1.0 : -1.0;
        double u[3], Hu[3], vu[3], Hvu[3];
        for (int r = 0; r < 3; ++r) u[r] = a * V[0][r] + sg * b * V[2][r];
        for (int r = 0; r < 3; ++r) Hu[r] = H[3 * r] * u[0] + H[3 * r + 1] * u[1] + H[3 * r + 2] * u[2];
        pose_cross(V[1], u, vu);
        pose_cross(Hv2, Hu, Hvu);
        // R = W U^T = Hv2 v2^T + Hu u^T + Hvu vu^T
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R[k][3 * i + j] = Hv2[i] * V[1][j] + Hu[i] * u[j] + Hvu[i] * vu[j];
        for (int r = 0; r < 3; ++r) n[k][r] = vu[r];
        for (int i = 0; i < 3; ++i) {
            double v = 0.0;
            for (int j = 0; j < 3; ++j) v += (H[3 * i + j] - R[k][3 * i + j]) * vu[j];
            t[k][i] = v;
        }
        for (int j = 0; j < 9; ++j) R[k + 2][j] = R[k][j];
        for (int r = 0; r < 3; ++r) { n[k + 2][r] = -n[k][r]; t[k + 2][r] = -t[k][r]; }
    }
    return 4;
}

// the candidates with n_z > 0 in order: their indices in keep, their number returned
PSV_HD int tv_prune(const double (&n)[4][3], int (&keep)[4])
{
    int m = 0;
    for (int k = 0; k < 4; ++k)
        if (n[k][2] > 0.0) keep[m++] = k;
    return m;
}

// the angle at X between the rays from the left centre (0) and from the right centre c = -R^T t, degrees
PSV_HD double tv_angle(const double* X, const double* R, const double* t)
{
    const double c[3] = {-(R[0] * t[0] + R[3] * t[1] + R[6] * t[2]), -(R[1] * t[0] + R[4] * t[1] + R[7] * t[2]),
                         -(R[2] * t[0] + R[5] * t[1] + R[8] * t[2])};
    const double v[3] = {X[0] - c[0], X[1] - c[1], X[2] - c[2]};
    double w[3];
    pose_cross(X, v, w);
    const double cr = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), dt = X[0] * v[0] + X[1] * v[1] + X[2] * v[2];
    return atan2(cr, dt) * (180.0 / 3.141592653589793);
}

// step 2: the configuration from the counts, kTvPlanar standing for "planar or panoramic: step 3"; allow_h = false
// classifies as if planar_or_panoramic were false
PSV_HD int tv_classify(int n_e, int n_f, int n_h, int min_inliers, double min_ef_ratio, double max_h_ratio, bool allow_h = true)
{
    const bool calibrated = n_e >= min_inliers && (double)n_e >= min_ef_ratio * (double)n_f;
    const double m = calibrated ? (double)n_e : (double)n_f;
    const bool hp = allow_h && n_h >= min_inliers && (double)n_h > max_h_ratio * m;
    if (hp) return kTvPlanar;
    if (calibrated) return kTvGeneral;
    return n_f >= min_inliers ? kTvUncalibrated : kTvDegenerate;
}

} // namespace psb
