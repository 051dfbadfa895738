// The per-observation math of ps_triangulate_tracks (include/popsift_b200_triangulate.h), in double: camera centres, ray
// directions, the hypothesis point (pose_two_rays of k_pose_solve.h), the pixel residual and its Jacobian, and the 3 x 3
// Gauss-Newton step.  One definition for the kernels (k_triangulate.cu) and the host check
// (tests/cpp/triangulate_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_pose_solve.h"

namespace psb {

// one set's camera: the pose X_cam = R X + t, its centre C = -R^T t, and the pinhole intrinsics
struct TriCam {
    double R[9], t[3], C[3];
    double fx, fy, cx, cy;
};

PSV_HD void tri_centre(const double* R, const double* t, double* C)
{
    for (int k = 0; k < 3; ++k) C[k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);
}

// the unit direction R^T ((x - cx) / fx, (y - cy) / fy, 1) / |.| of pixel (x, y); false when it is zero or not finite
PSV_HD bool tri_direction(const TriCam& K, double x, double y, double* d)
{
    const double xn = (x - K.cx) / K.fx, yn = (y - K.cy) / K.fy;
    for (int k = 0; k < 3; ++k) d[k] = K.R[k] * xn + K.R[3 + k] * yn + K.R[6 + k];
    return pose_unit(d);
}

// The hypothesis of two rays C_a + s_a d_a, C_b + s_b d_b: pose_two_rays with t = C_a - C_b, then the midpoint
// X = ((C_a + s_a d_a) + (C_b + s_b d_b)) / 2.  Valid when pose_two_rays holds and d_a.d_b <= cos_min.
PSV_HD bool tri_hypothesis(const double* Ca, const double* da, const double* Cb, const double* db, double cos_min, double* X)
{
    const double w[3] = {Ca[0] - Cb[0], Ca[1] - Cb[1], Ca[2] - Cb[2]};
    double sa, sb;
    if (!pose_two_rays(da, db, w, sa, sb)) return false;
    if (!(da[0] * db[0] + da[1] * db[1] + da[2] * db[2] <= cos_min)) return false;
    for (int k = 0; k < 3; ++k) X[k] = 0.5 * ((Ca[k] + sa * da[k]) + (Cb[k] + sb * db[k]));
    return true;
}

// The pixel residual of pixel (x, y) under X: X_c = R X + t, false unless z = X_c[2] > 0; iz = 1 / z,
// e_x = fx (X_c[0] iz) + cx - x, e_y = fy (X_c[1] iz) + cy - y.  Jx / Jy (optional): d e_x / dX, d e_y / dX.  Xc_out
// (optional): X_c, written whether or not z > 0 (bundle adjustment's pose Jacobian, k_bundle.h).
PSV_HD bool tri_residual(const TriCam& K, const double* X, double x, double y, double& ex, double& ey, double* Jx = nullptr,
                         double* Jy = nullptr, double* Xc_out = nullptr)
{
    double Xc[3];
    for (int r = 0; r < 3; ++r) Xc[r] = K.R[3 * r] * X[0] + K.R[3 * r + 1] * X[1] + K.R[3 * r + 2] * X[2] + K.t[r];
    if (Xc_out)
        for (int r = 0; r < 3; ++r) Xc_out[r] = Xc[r];
    if (!(Xc[2] > 0.0)) return false;
    const double iz = 1.0 / Xc[2];
    const double p = Xc[0] * iz, q = Xc[1] * iz;
    ex = K.fx * p + K.cx - x;
    ey = K.fy * q + K.cy - y;
    if (Jx) {
        for (int k = 0; k < 3; ++k) {
            Jx[k] = K.fx * ((K.R[k] - p * K.R[6 + k]) * iz);
            Jy[k] = K.fy * ((K.R[3 + k] - q * K.R[6 + k]) * iz);
        }
    }
    return true;
}

// e2 = e_x^2 + e_y^2 of pixel (x, y) under X; false (e2 untouched) when X is not in front of the camera
PSV_HD bool tri_error2(const TriCam& K, const double* X, double x, double y, double& e2)
{
    double ex, ey;
    if (!tri_residual(K, X, x, y, ex, ey)) return false;
    e2 = ex * ex + ey * ey;
    return true;
}

// The Gauss-Newton step of S = (J^T J as 00, 01, 02, 11, 12, 22; -J^T e): dX = (J^T J)^-1 (-J^T e) by Cramer's rule;
// false when the determinant is not finite and > 0
PSV_HD bool tri_step(const double* S, double* dX)
{
    const double a = S[0], b = S[1], c = S[2], d = S[3], e = S[4], f = S[5], g0 = S[6], g1 = S[7], g2 = S[8];
    const double m0 = d * f - e * e, m1 = b * f - e * c, m2 = b * e - d * c;
    const double det = a * m0 - b * m1 + c * m2;
    if (!(det > 0.0) || !isfinite(det)) return false;
    dX[0] = (g0 * m0 - b * (g1 * f - e * g2) + c * (g1 * e - d * g2)) / det;
    dX[1] = (a * (g1 * f - e * g2) - g0 * m1 + c * (b * g2 - g1 * c)) / det;
    dX[2] = (a * (d * g2 - g1 * e) - b * (b * g2 - g1 * c) + g0 * m2) / det;
    return true;
}

} // namespace psb
