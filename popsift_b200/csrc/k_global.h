// The per-edge math of ps_rotation_averaging and ps_global_positioning (include/popsift_b200_global.h), in double: the
// rotation logarithm, the projection of a float rotation onto SO(3), the pair residual Log(R_r^T R_p R_l), the update R <- R Exp(x) (ba_rodrigues of k_bundle.h), and an
// observation's scale d and residual v - d (X - c).  One definition for the kernels (k_global.cu), the host start of
// rotation averaging and the host check (tests/cpp/global_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_bundle.h"

namespace psb {

// C = A B, row-major 3 x 3, each entry summed in k order
PSV_HD void gl_mul(const double* A, const double* B, double* C)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// C = A^T B
PSV_HD void gl_mul_tn(const double* A, const double* B, double* C)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}

// Log of a rotation (row-major) as a rotation vector.  c = (tr M - 1) / 2 clamped to [-1, 1], s = the axial vector of
// (M - M^T) / 2, theta = atan2(|s|, c).  For c > -0.99: w = (theta / |s|) s, or (1 + |s|^2 / 6) s when |s| < 1e-8.  Near
// pi (c <= -0.99) the axis comes from the symmetric part B = (M + M^T) / 2 = c I + (1 - c) a a^T: k the largest diagonal
// entry of B, a_k = sqrt((B_kk - c) / (1 - c)), a_j = B_jk / ((1 - c) a_k), its sign chosen so that a.s >= 0; w = theta a.
PSV_HD void gl_log(const double* M, double* w)
{
    double c = 0.5 * ((M[0] + M[4] + M[8]) - 1.0);
    c = fmin(1.0, fmax(-1.0, c));
    const double s[3] = {0.5 * (M[7] - M[5]), 0.5 * (M[2] - M[6]), 0.5 * (M[3] - M[1])};
    const double sn = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
    const double th = atan2(sn, c);
    if (c > -0.99) {
        const double f = sn < 1e-8 ? 1.0 + sn * sn / 6.0 : th / sn;
        for (int k = 0; k < 3; ++k) w[k] = f * s[k];
        return;
    }
    const double B[9] = {M[0], 0.5 * (M[1] + M[3]), 0.5 * (M[2] + M[6]), 0.5 * (M[1] + M[3]), M[4], 0.5 * (M[5] + M[7]),
                         0.5 * (M[2] + M[6]), 0.5 * (M[5] + M[7]), M[8]};
    int k = 0;
    if (B[4] > B[3 * k + k]) k = 1;
    if (B[8] > B[3 * k + k]) k = 2;
    const double omc = 1.0 - c;
    double a[3];
    a[k] = sqrt(fmax(0.0, (B[3 * k + k] - c) / omc));
    for (int j = 0; j < 3; ++j)
        if (j != k) a[j] = B[3 * j + k] / (omc * a[k]);
    const double sg = a[0] * s[0] + a[1] * s[1] + a[2] * s[2] < 0.0 ? -1.0 : 1.0;
    for (int j = 0; j < 3; ++j) w[j] = th * (sg * a[j]);
}

// The rotation nearest a float matrix by a unit-quaternion round trip (Shepperd's branch on the largest of tr, m00, m11,
// m22; q normalised in double), so rotations chained from float records stay orthonormal to double precision
PSV_HD void gl_orthonormal(const float* m, double* R)
{
    const double a[9] = {m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8]};
    const double tr = a[0] + a[4] + a[8];
    double w, x, y, z;
    if (tr > 0.0) {
        const double s = 2.0 * sqrt(tr + 1.0);
        w = 0.25 * s; x = (a[7] - a[5]) / s; y = (a[2] - a[6]) / s; z = (a[3] - a[1]) / s;
    } else if (a[0] > a[4] && a[0] > a[8]) {
        const double s = 2.0 * sqrt(1.0 + a[0] - a[4] - a[8]);
        w = (a[7] - a[5]) / s; x = 0.25 * s; y = (a[1] + a[3]) / s; z = (a[2] + a[6]) / s;
    } else if (a[4] > a[8]) {
        const double s = 2.0 * sqrt(1.0 + a[4] - a[0] - a[8]);
        w = (a[2] - a[6]) / s; x = (a[1] + a[3]) / s; y = 0.25 * s; z = (a[5] + a[7]) / s;
    } else {
        const double s = 2.0 * sqrt(1.0 + a[8] - a[0] - a[4]);
        w = (a[3] - a[1]) / s; x = (a[2] + a[6]) / s; y = (a[5] + a[7]) / s; z = 0.25 * s;
    }
    const double n = sqrt(w * w + x * x + y * y + z * z);
    w /= n; x /= n; y /= n; z /= n;
    R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - z * w); R[2] = 2.0 * (x * z + y * w);
    R[3] = 2.0 * (x * y + z * w); R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - x * w);
    R[6] = 2.0 * (x * z - y * w); R[7] = 2.0 * (y * z + x * w); R[8] = 1.0 - 2.0 * (x * x + y * y);
}

// the pair residual r = Log(R_r^T (R_p R_l))
PSV_HD void gl_pair_residual(const double* Rl, const double* Rr, const double* Rp, double* r)
{
    double A[9], M[9];
    gl_mul(Rp, Rl, A);
    gl_mul_tn(Rr, A, M);
    gl_log(M, r);
}

// the rotation update Rn = R Exp(x)
PSV_HD void gl_rot_update(const double* R, const double* x, double* Rn)
{
    double E[9];
    ba_rodrigues(x, E);
    gl_mul(R, E, Rn);
}

// One observation of global positioning: u = X - c, d = max(0, v.u) / (u.u) (0 when u.u is not > 0), e = v - d u.
// Returns |e|^2.
PSV_HD double gl_obs(const double* v, const double* X, const double* c, double& d, double* e)
{
    const double u[3] = {X[0] - c[0], X[1] - c[1], X[2] - c[2]};
    const double uu = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
    const double vu = v[0] * u[0] + v[1] * u[1] + v[2] * u[2];
    d = uu > 0.0 ? fmax(0.0, vu) / uu : 0.0;
    for (int k = 0; k < 3; ++k) e[k] = v[k] - d * u[k];
    return e[0] * e[0] + e[1] * e[1] + e[2] * e[2];
}

} // namespace psb
