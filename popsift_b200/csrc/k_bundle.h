// The per-observation math of ps_bundle_adjust (include/popsift_b200_bundle.h), in double, built on k_triangulate.h: the
// robust loss and its IRLS weight, the residual's pose and point Jacobians, Rodrigues' formula and the pose update, the
// 6 x 6 Cholesky factorisation and solve of the preconditioner, and the 3 x 3 symmetric inverse of the point blocks.  One
// definition for the kernels (k_bundle.cu) and the host check (tests/cpp/bundle_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_triangulate.h"

namespace psb {

enum { BA_LOSS_SQUARED = 0, BA_LOSS_HUBER = 1, BA_LOSS_CAUCHY = 2 };   // PS_LOSS_*

// rho(z) and its IRLS weight w = rho'(z) for z = |e|^2 / s^2 >= 0
PSV_HD void ba_loss(int loss, double z, double& rho, double& w)
{
    if (loss == BA_LOSS_HUBER) {
        if (z <= 1.0) { rho = z; w = 1.0; }
        else { const double r = sqrt(z); rho = 2.0 * r - 1.0; w = 1.0 / r; }
    } else if (loss == BA_LOSS_CAUCHY) {
        rho = log1p(z);
        w = 1.0 / (1.0 + z);
    } else {
        rho = z;
        w = 1.0;
    }
}

// The residual e of pixel (x, y) under X (tri_residual) and its Jacobians, false when z <= 0.  Jc (2 x 6, row-major):
// d e / d(omega, dt) of the update R <- Exp(omega) R, t <- t + dt at 0; with a = d e_r / dX_c = f_r iz (unit_r - (p, q)_r
// e_z) and v = X_c - t (= R X): d e_r / d omega = v x a, d e_r / d dt = a.  Jp (2 x 3): d e / dX.
PSV_HD bool ba_jacobian(const TriCam& K, const double* X, double x, double y, double* e, double* Jc, double* Jp)
{
    double Xc[3];
    if (!tri_residual(K, X, x, y, e[0], e[1], Jp, Jp + 3, Xc)) return false;
    const double iz = 1.0 / Xc[2];
    const double p = Xc[0] * iz, q = Xc[1] * iz;
    const double v[3] = {Xc[0] - K.t[0], Xc[1] - K.t[1], Xc[2] - K.t[2]};
    const double a[2][3] = {{K.fx * iz, 0.0, -(K.fx * p) * iz}, {0.0, K.fy * iz, -(K.fy * q) * iz}};
    for (int r = 0; r < 2; ++r) {
        double* J = Jc + 6 * r;
        J[0] = v[1] * a[r][2] - v[2] * a[r][1];
        J[1] = v[2] * a[r][0] - v[0] * a[r][2];
        J[2] = v[0] * a[r][1] - v[1] * a[r][0];
        J[3] = a[r][0];
        J[4] = a[r][1];
        J[5] = a[r][2];
    }
    return true;
}

// Exp(omega) by Rodrigues: theta2 = omega.omega; A = sin(theta) / theta and B = (1 - cos(theta)) / theta2, or their series
// 1 - theta2 / 6 and 1 / 2 - theta2 / 24 when theta2 < 1e-16; E = I + A [omega]x + B (omega omega^T - theta2 I), row-major
PSV_HD void ba_rodrigues(const double* w, double* E)
{
    const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    double A, B;
    if (th2 < 1e-16) {
        A = 1.0 - th2 / 6.0;
        B = 0.5 - th2 / 24.0;
    } else {
        const double th = sqrt(th2);
        A = sin(th) / th;
        B = (1.0 - cos(th)) / th2;
    }
    const double W[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) E[3 * i + j] = (i == j ? 1.0 : 0.0) + A * W[3 * i + j] + B * (w[i] * w[j] - (i == j ? th2 : 0.0));
}

// the pose update: Rn = Exp(d[0..2]) R (row-major products in k order), tn = t + d[3..5]
PSV_HD void ba_pose_update(const double* R, const double* t, const double* d, double* Rn, double* tn)
{
    double E[9];
    ba_rodrigues(d, E);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rn[3 * i + j] = E[3 * i] * R[j] + E[3 * i + 1] * R[3 + j] + E[3 * i + 2] * R[6 + j];
    for (int k = 0; k < 3; ++k) tn[k] = t[k] + d[3 + k];
}

// Cholesky A = L L^T of a symmetric 6 x 6 (row-major, the lower triangle read); L row-major lower.  False when a pivot is
// not finite and > 0.
PSV_HD bool ba_chol6(const double* A, double* L)
{
    for (int k = 0; k < 36; ++k) L[k] = 0.0;
    for (int j = 0; j < 6; ++j) {
        double d = A[6 * j + j];
        for (int k = 0; k < j; ++k) d -= L[6 * j + k] * L[6 * j + k];
        if (!(d > 0.0) || !isfinite(d)) return false;
        const double s = sqrt(d);
        L[6 * j + j] = s;
        for (int i = j + 1; i < 6; ++i) {
            double v = A[6 * i + j];
            for (int k = 0; k < j; ++k) v -= L[6 * i + k] * L[6 * j + k];
            L[6 * i + j] = v / s;
        }
    }
    return true;
}

// x = (L L^T)^-1 b: forward, then backward substitution
PSV_HD void ba_chol6_solve(const double* L, const double* b, double* x)
{
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double v = b[i];
        for (int k = 0; k < i; ++k) v -= L[6 * i + k] * y[k];
        y[i] = v / L[6 * i + i];
    }
    for (int i = 5; i >= 0; --i) {
        double v = y[i];
        for (int k = i + 1; k < 6; ++k) v -= L[6 * k + i] * x[k];
        x[i] = v / L[6 * i + i];
    }
}

// The inverse of a symmetric 3 x 3 (00, 01, 02, 11, 12, 22) by its adjugate, in the same order; false when the
// determinant is not finite and > 0
PSV_HD bool ba_inv3(const double* S, double* I)
{
    const double a = S[0], b = S[1], c = S[2], d = S[3], e = S[4], f = S[5];
    const double m0 = d * f - e * e, m1 = b * f - e * c, m2 = b * e - d * c;
    const double det = a * m0 - b * m1 + c * m2;
    if (!(det > 0.0) || !isfinite(det)) return false;
    I[0] = m0 / det;
    I[1] = -m1 / det;
    I[2] = m2 / det;
    I[3] = (a * f - c * c) / det;
    I[4] = -(a * e - b * c) / det;
    I[5] = (a * d - b * b) / det;
    return true;
}

// y = S x for a symmetric 3 x 3 in ba_inv3's order
PSV_HD void ba_sym3_mul(const double* S, const double* x, double* y)
{
    y[0] = S[0] * x[0] + S[1] * x[1] + S[2] * x[2];
    y[1] = S[1] * x[0] + S[3] * x[1] + S[4] * x[2];
    y[2] = S[2] * x[0] + S[4] * x[1] + S[5] * x[2];
}

// Marquardt's damping of a diagonal entry: d + lambda * min(max(d, 1e-6), 1e32)
PSV_HD double ba_damp(double d, double lambda)
{
    return d + lambda * fmin(fmax(d, 1e-6), 1e32);
}

} // namespace psb
