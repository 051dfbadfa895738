// The calibrated two-view math of ps_relative_pose_batch (include/popsift_b200_pose.h), in double: the five-point solver,
// the 3 x 3 SVD behind the essential-matrix projection and the pose decomposition, the triangulation / cheirality rule,
// the calibration of the rows and the pixel F.
// One definition for the kernels (k_pose.cu) and the host check (tests/cpp/pose_solver_check.cpp).  Arrays indexed at
// run time live in local memory on the device.
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_verify_sample.h"   // PSV_HD

namespace psb {

constexpr int kPoseSlots = 10;               // hypotheses per sample: at most ten real solutions
constexpr double kPoseNullTol = 1e-10;       // 5 x 9 pivot: below this times the largest entry, the sample gives nothing
constexpr double kPoseElimTol = 1e-12;       // 10 x 20 pivot: below this times the largest entry, the sample gives nothing

// One pair's intrinsics in double (left, right) and the squared calibrated threshold (ps_relative_pose_batch's rule 1)
struct PCam { double fxl, fyl, cxl, cyl, fxr, fyr, cxr, cyr; float t2, pad; };

// host: the PCam of cameras l, r (ps_camera) at `threshold` pixels: f = (fx_l + fy_l + fx_r + fy_r) / 4 in double,
// t2 = (float)((threshold / f)^2)
template <class Cam>
inline PCam pose_cam(const Cam& l, const Cam& r, float threshold)
{
    const double fbar = ((double)l.fx + (double)l.fy + (double)r.fx + (double)r.fy) / 4.0;
    const double ts = (double)threshold / fbar;
    return {l.fx, l.fy, l.cx, l.cy, r.fx, r.fy, r.cx, r.cy, (float)(ts * ts), 0.0f};
}

// rule 1: a pixel row (x_l, y_l, x_r, y_r) in calibrated coordinates, x^ = (x - cx) / fx in double, rounded once
PSV_HD void pose_calibrate(const PCam& K, float xl, float yl, float xr, float yr, float* c)
{
    c[0] = (float)(((double)xl - K.cxl) / K.fxl);
    c[1] = (float)(((double)yl - K.cyl) / K.fyl);
    c[2] = (float)(((double)xr - K.cxr) / K.fxr);
    c[3] = (float)(((double)yr - K.cyr) / K.fyr);
}

// ---- polynomials in (x, y, z) of E = x X + y Y + z Z + W ----
// linear: [x, y, z, 1]; quadratic: [x^2, xy, y^2, xz, yz, z^2, x, y, z, 1]; cubic (the elimination order):
//   0 x^3  1 y^3  2 x^2y  3 xy^2  4 x^2z  5 x^2  6 y^2z  7 y^2  8 xyz  9 xy | 10 xz^2  11 xz  12 x  13 yz^2  14 yz  15 y
//   16 z^3  17 z^2  18 z  19 1

PSV_HD void pose_mul11(const double (&a)[4], const double (&b)[4], double (&q)[10])
{
    q[0] = a[0] * b[0];
    q[1] = a[0] * b[1] + a[1] * b[0];
    q[2] = a[1] * b[1];
    q[3] = a[0] * b[2] + a[2] * b[0];
    q[4] = a[1] * b[2] + a[2] * b[1];
    q[5] = a[2] * b[2];
    q[6] = a[0] * b[3] + a[3] * b[0];
    q[7] = a[1] * b[3] + a[3] * b[1];
    q[8] = a[2] * b[3] + a[3] * b[2];
    q[9] = a[3] * b[3];
}

// c += q * a (quadratic times linear)
PSV_HD void pose_mul21_acc(const double (&q)[10], const double (&a)[4], double (&c)[20])
{
    const double x = a[0], y = a[1], z = a[2], o = a[3];
    c[0] += q[0] * x;                                   // x^3
    c[1] += q[2] * y;                                   // y^3
    c[2] += q[0] * y + q[1] * x;                        // x^2 y
    c[3] += q[1] * y + q[2] * x;                        // x y^2
    c[4] += q[0] * z + q[3] * x;                        // x^2 z
    c[5] += q[0] * o + q[6] * x;                        // x^2
    c[6] += q[2] * z + q[4] * y;                        // y^2 z
    c[7] += q[2] * o + q[7] * y;                        // y^2
    c[8] += q[1] * z + q[3] * y + q[4] * x;             // x y z
    c[9] += q[1] * o + q[6] * y + q[7] * x;             // x y
    c[10] += q[3] * z + q[5] * x;                       // x z^2
    c[11] += q[3] * o + q[6] * z + q[8] * x;            // x z
    c[12] += q[6] * o + q[9] * x;                       // x
    c[13] += q[4] * z + q[5] * y;                       // y z^2
    c[14] += q[4] * o + q[7] * z + q[8] * y;            // y z
    c[15] += q[7] * o + q[9] * y;                       // y
    c[16] += q[5] * z;                                  // z^3
    c[17] += q[5] * o + q[8] * z;                       // z^2
    c[18] += q[8] * o + q[9] * z;                       // z
    c[19] += q[9] * o;                                  // 1
}

PSV_HD double pose_peval(const double* c, int d, double x)
{
    double v = c[d];
    for (int i = d - 1; i >= 0; --i) v = v * x + c[i];
    return v;
}

// the root of q (degree k, monotone on [lo, hi], q(lo) negative when lo_neg, q(hi) of the other sign): Newton steps
// kept inside the bracket, a bisection where a step would leave it or would not halve the step before (rtsafe)
PSV_HD double pose_bracket_root(const double* q, int k, double lo, double hi, bool lo_neg)
{
    double x = 0.5 * (lo + hi), dx = hi - lo, dxold = dx;
    for (int it = 0; it < 200; ++it) {
        double f = q[k], g = 0.0;
        for (int i = k - 1; i >= 0; --i) { g = g * x + f; f = f * x + q[i]; }
        if (f == 0.0) return x;
        if ((f < 0.0) == lo_neg) lo = x; else hi = x;
        const double xn = x - f / g;
        dxold = dx;
        if (!(g != 0.0) || !(xn > lo && xn < hi) || fabs(2.0 * f) > fabs(dxold * g)) {
            dx = 0.5 * (hi - lo);
            x = lo + dx;
        } else {
            dx = f / g;
            x = xn;
        }
        if (fabs(dx) <= 2.2e-16 * fabs(x) || !(hi - lo > 2.2e-16 * fmax(fabs(lo), fabs(hi)))) return x;
    }
    return x;
}

// Real roots of c[0] + c[1] z + .. + c[d] z^d, ascending; returns their number.  Isolation by the derivative chain: the
// roots of p^(m + 1) split the real line into intervals on which p^(m) is monotone, so each holds at most one root of
// p^(m), present exactly when the signs at its ends differ; the outer ends are -B and B with B Fujiwara's bound
// 2 max(|c[d-1] / c[d]|, |c[d-2] / c[d]|^(1/2), .., |c[0] / (2 c[d])|^(1/d)) of p, which bounds every root of every
// derivative (Gauss-Lucas).  A root of even multiplicity is not found.
PSV_HD int pose_real_roots(const double (&c)[11], double (&r)[10])
{
    int d = 10;
    while (d > 0 && c[d] == 0.0) --d;
    if (d == 0) return 0;
    double B = 0.0;
    for (int i = 0; i < d; ++i) B = fmax(B, pow(fabs(c[i] / c[d]) * (i == 0 ? 0.5 : 1.0), 1.0 / (d - i)));
    B *= 2.0;
    if (!isfinite(B) || !(B > 0.0)) return 0;
    double prev[10];
    int np = 0;
    for (int k = 1; k <= d; ++k) {
        // q = p^(d - k), degree k: q_i = c[i + m] (i + m)! / i!, m = d - k
        const int m = d - k;
        double q[11];
        for (int i = 0; i <= k; ++i) {
            double f = c[i + m];
            for (int j = i + 1; j <= i + m; ++j) f *= (double)j;
            q[i] = f;
        }
        int nr = 0;
        double cur[10];
        double a = -B, fa = pose_peval(q, k, a);
        for (int e = 0; e <= np; ++e) {
            const double b = e < np ? prev[e] : B;
            const double fb = pose_peval(q, k, b);
            if (b > a) {
                if (fa == 0.0) {
                    if (nr == 0 || cur[nr - 1] != a) cur[nr++] = a;
                } else if ((fa < 0.0) != (fb < 0.0) && fb != 0.0) {
                    cur[nr++] = pose_bracket_root(q, k, a, b, fa < 0.0);
                }
            }
            a = b; fa = fb;
        }
        if (fa == 0.0 && (nr == 0 || cur[nr - 1] != a) && nr < 10) cur[nr++] = a;
        for (int i = 0; i < nr; ++i) prev[i] = cur[i];
        np = nr;
    }
    for (int i = 0; i < np; ++i) r[i] = prev[i];
    return np;
}

// polynomial product, ascending coefficients: c (degree da + db) = a * b
PSV_HD void pose_pmul(const double* a, int da, const double* b, int db, double* c)
{
    for (int i = 0; i <= da + db; ++i) c[i] = 0.0;
    for (int i = 0; i <= da; ++i)
        for (int j = 0; j <= db; ++j) c[i + j] += a[i] * b[j];
}

// Gauss-Newton polish of a solution (x, y, z) on the ten reduced cubics M (rows of [I | G], the monomial order above):
// two steps, each kept only when it lowers the sum of squared residuals
PSV_HD double pose_cubic_residual(const double (&M)[10][20], double x, double y, double z, double (*J)[3], double* f)
{
    const double mono[20] = {x * x * x, y * y * y, x * x * y, x * y * y, x * x * z, x * x, y * y * z, y * y, x * y * z, x * y,
                             x * z * z, x * z, x, y * z * z, y * z, y, z * z * z, z * z, z, 1.0};
    const double dx[20] = {3 * x * x, 0, 2 * x * y, y * y, 2 * x * z, 2 * x, 0, 0, y * z, y, z * z, z, 1, 0, 0, 0, 0, 0, 0, 0};
    const double dy[20] = {0, 3 * y * y, x * x, 2 * x * y, 0, 0, 2 * y * z, 2 * y, x * z, x, 0, 0, 0, z * z, z, 1, 0, 0, 0, 0};
    const double dz[20] = {0, 0, 0, 0, x * x, 0, y * y, 0, x * y, 0, 2 * x * z, x, 0, 2 * y * z, y, 0, 3 * z * z, 2 * z, 1, 0};
    double ss = 0.0;
    for (int r = 0; r < 10; ++r) {
        double v = 0.0, a = 0.0, b = 0.0, c = 0.0;
        for (int k = 0; k < 20; ++k) { v += M[r][k] * mono[k]; a += M[r][k] * dx[k]; b += M[r][k] * dy[k]; c += M[r][k] * dz[k]; }
        if (f) { f[r] = v; J[r][0] = a; J[r][1] = b; J[r][2] = c; }
        ss += v * v;
    }
    return ss;
}

PSV_HD void pose_polish(const double (&M)[10][20], double& x, double& y, double& z)
{
    for (int it = 0; it < 2; ++it) {
        double J[10][3], f[10];
        const double ss = pose_cubic_residual(M, x, y, z, J, f);
        if (!(ss > 0.0)) return;
        double A[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
        for (int r = 0; r < 10; ++r)
            for (int a = 0; a < 3; ++a) {
                g[a] -= J[r][a] * f[r];
                for (int b = 0; b < 3; ++b) A[3 * a + b] += J[r][a] * J[r][b];
            }
        const double det = A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
        if (!(fabs(det) > 0.0) || !isfinite(det)) return;
        const double d0 = (g[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (g[1] * A[8] - A[5] * g[2]) + A[2] * (g[1] * A[7] - A[4] * g[2])) / det;
        const double d1 = (A[0] * (g[1] * A[8] - A[5] * g[2]) - g[0] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * g[2] - g[1] * A[6])) / det;
        const double d2 = (A[0] * (A[4] * g[2] - g[1] * A[7]) - A[1] * (A[3] * g[2] - g[1] * A[6]) + g[0] * (A[3] * A[7] - A[4] * A[6])) / det;
        const double xn = x + d0, yn = y + d1, zn = z + d2;
        if (!isfinite(xn) || !isfinite(yn) || !isfinite(zn)) return;
        if (!(pose_cubic_residual(M, xn, yn, zn, nullptr, nullptr) < ss)) return;
        x = xn; y = yn; z = zn;
    }
}

// Five-point solver (Nister's elimination): calibrated rows p[j] = (x_l, y_l, x_r, y_r).  Writes up to ten essential
// matrices (row-major, x_r^T E x_l = 0, unnormalised) in ascending z and returns their number; 0 when the sample gives none.
//   1. the 5 x 9 epipolar system, Gauss-Jordan with partial pivoting in column order; four free columns, else nothing;
//      the null vectors of the free columns in order (a free column 1, the others 0), orthonormalised by modified
//      Gram-Schmidt in that order, are X, Y, Z, W;
//   2. the ten cubics det E = 0 (row 9) and 2 E E^T E - tr(E E^T) E = 0 (rows 0..8, row-major) in 20 monomials;
//   3. Gauss-Jordan with partial pivoting on the first ten columns: [I | G];
//   4. k = <e> - z <f>, l = <g> - z <h>, m = <i> - z <j> (rows 4..9) are linear in (x, y, 1) with coefficients in z of
//      degree 3, 3, 4; det of that 3 x 3 is the degree-10 polynomial, whose real roots are z;
//   5. (x, y, 1) spans the null space of the 3 x 3 at z: the largest of the three row cross products; then two
//      Gauss-Newton steps on the ten reduced cubics polish (x, y, z), each kept only when it lowers the residual.  A root whose x, y
//      or E is not finite, or whose E is zero, is skipped: the solutions are numbered without it.
// `sol_z` (optional) receives the roots.
PSV_HD int pose_five_point(const double (&p)[5][4], double (&Es)[kPoseSlots][9], double* sol_z = nullptr)
{
    double A[5][9];
    double sc = 0.0;
    for (int j = 0; j < 5; ++j) {
        const double x = p[j][0], y = p[j][1], xr = p[j][2], yr = p[j][3];
        const double row[9] = {xr * x, xr * y, xr, yr * x, yr * y, yr, x, y, 1.0};
        for (int c = 0; c < 9; ++c) { A[j][c] = row[c]; sc = fmax(sc, fabs(row[c])); }
    }
    int piv[5], fr[4];
    int row = 0, nfree = 0;
    for (int col = 0; col < 9; ++col) {
        int best = -1;
        double bv = kPoseNullTol * sc;
        for (int r = row; r < 5; ++r) {
            const double v = fabs(A[r][col]);
            if (v > bv) { bv = v; best = r; }
        }
        if (best < 0) {
            if (nfree < 4) fr[nfree] = col;
            ++nfree;
            continue;
        }
        if (best != row)
            for (int c = 0; c < 9; ++c) { const double t = A[row][c]; A[row][c] = A[best][c]; A[best][c] = t; }
        const double inv = 1.0 / A[row][col];
        for (int c = 0; c < 9; ++c) A[row][c] *= inv;
        for (int r = 0; r < 5; ++r) {
            if (r == row) continue;
            const double f = A[r][col];
            if (f != 0.0)
                for (int c = 0; c < 9; ++c) A[r][c] -= f * A[row][c];
        }
        piv[row] = col;
        ++row;
    }
    if (row != 5 || nfree != 4) return 0;
    // E[e] as a linear polynomial [x, y, z, 1]: basis k's entry e
    double L[9][4];
    for (int e = 0; e < 9; ++e)
        for (int k = 0; k < 4; ++k) L[e][k] = e == fr[k] ? 1.0 : 0.0;
    for (int r = 0; r < 5; ++r)
        for (int k = 0; k < 4; ++k) L[piv[r]][k] = -A[r][fr[k]];
    // orthonormal basis of the null space (modified Gram-Schmidt in basis order): the cubics below are far better
    // conditioned than on the raw vectors
    for (int k = 0; k < 4; ++k) {
        for (int j = 0; j < k; ++j) {
            double d = 0.0;
            for (int e = 0; e < 9; ++e) d += L[e][k] * L[e][j];
            for (int e = 0; e < 9; ++e) L[e][k] -= d * L[e][j];
        }
        double nn = 0.0;
        for (int e = 0; e < 9; ++e) nn += L[e][k] * L[e][k];
        const double inv = 1.0 / sqrt(nn);
        for (int e = 0; e < 9; ++e) L[e][k] *= inv;
    }
    // the ten cubics
    double M[10][20];
    for (int i = 0; i < 10; ++i)
        for (int c = 0; c < 20; ++c) M[i][c] = 0.0;
    {
        double q[10];
        // det E by the first row: E0 (E4 E8 - E5 E7) - E1 (E3 E8 - E5 E6) + E2 (E3 E7 - E4 E6)
        const int cof[3][5] = {{0, 4, 8, 5, 7}, {1, 3, 8, 5, 6}, {2, 3, 7, 4, 6}};
        for (int k = 0; k < 3; ++k) {
            double q1[10], q2[10];
            pose_mul11(L[cof[k][1]], L[cof[k][2]], q1);
            pose_mul11(L[cof[k][3]], L[cof[k][4]], q2);
            const double sg = k == 1 ? -1.0 : 1.0;
            for (int i = 0; i < 10; ++i) q[i] = sg * (q1[i] - q2[i]);
            pose_mul21_acc(q, L[cof[k][0]], M[9]);
        }
        // EE^T (symmetric, quadratic) and its trace
        double S[9][10], tr[10];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                for (int u = 0; u < 10; ++u) S[3 * i + j][u] = 0.0;
                for (int k = 0; k < 3; ++k) {
                    pose_mul11(L[3 * i + k], L[3 * j + k], q);
                    for (int u = 0; u < 10; ++u) S[3 * i + j][u] += q[u];
                }
            }
        for (int u = 0; u < 10; ++u) tr[u] = S[0][u] + S[4][u] + S[8][u];
        // 2 (EE^T) E - tr E, entry (i, j) = sum_k 2 S_ik E_kj - tr E_ij
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                for (int k = 0; k < 3; ++k) {
                    for (int u = 0; u < 10; ++u) q[u] = 2.0 * S[3 * i + k][u];
                    pose_mul21_acc(q, L[3 * k + j], M[3 * i + j]);
                }
                for (int u = 0; u < 10; ++u) q[u] = -tr[u];
                pose_mul21_acc(q, L[3 * i + j], M[3 * i + j]);
            }
    }
    double msc = 0.0;
    for (int i = 0; i < 10; ++i)
        for (int c = 0; c < 20; ++c) msc = fmax(msc, fabs(M[i][c]));
    if (!(msc > 0.0) || !isfinite(msc)) return 0;
    for (int col = 0; col < 10; ++col) {
        int best = -1;
        double bv = kPoseElimTol * msc;
        for (int r = col; r < 10; ++r) {
            const double v = fabs(M[r][col]);
            if (v > bv) { bv = v; best = r; }
        }
        if (best < 0) return 0;
        if (best != col)
            for (int c = col; c < 20; ++c) { const double t = M[col][c]; M[col][c] = M[best][c]; M[best][c] = t; }
        const double inv = 1.0 / M[col][col];
        for (int c = col; c < 20; ++c) M[col][c] *= inv;
        for (int r = 0; r < 10; ++r) {
            if (r == col) continue;
            const double f = M[r][col];
            if (f != 0.0)
                for (int c = col; c < 20; ++c) M[r][c] -= f * M[col][c];
        }
    }
    // B(z): rows k, l, m; columns the coefficients of x (degree 3), y (3) and 1 (4), ascending in z
    double Bx[3][4], By[3][4], B1[3][5];
    for (int k = 0; k < 3; ++k) {
        const double* ge = &M[4 + 2 * k][10];
        const double* gf = &M[5 + 2 * k][10];
        Bx[k][0] = ge[2]; Bx[k][1] = ge[1] - gf[2]; Bx[k][2] = ge[0] - gf[1]; Bx[k][3] = -gf[0];
        By[k][0] = ge[5]; By[k][1] = ge[4] - gf[5]; By[k][2] = ge[3] - gf[4]; By[k][3] = -gf[3];
        B1[k][0] = ge[9]; B1[k][1] = ge[8] - gf[9]; B1[k][2] = ge[7] - gf[8]; B1[k][3] = ge[6] - gf[7]; B1[k][4] = -gf[6];
    }
    // det = Bx0 (By1 B12 - B11 By2) - By0 (Bx1 B12 - B11 Bx2) + B10 (Bx1 By2 - By1 Bx2)
    double poly[11];
    for (int i = 0; i < 11; ++i) poly[i] = 0.0;
    {
        double t1[8], t2[8], m7[7], c10[11];
        pose_pmul(By[1], 3, B1[2], 4, t1); pose_pmul(B1[1], 4, By[2], 3, t2);
        for (int i = 0; i < 8; ++i) t1[i] -= t2[i];
        pose_pmul(Bx[0], 3, t1, 7, c10);
        for (int i = 0; i < 11; ++i) poly[i] += c10[i];
        pose_pmul(Bx[1], 3, B1[2], 4, t1); pose_pmul(B1[1], 4, Bx[2], 3, t2);
        for (int i = 0; i < 8; ++i) t1[i] -= t2[i];
        pose_pmul(By[0], 3, t1, 7, c10);
        for (int i = 0; i < 11; ++i) poly[i] -= c10[i];
        pose_pmul(Bx[1], 3, By[2], 3, m7); pose_pmul(By[1], 3, Bx[2], 3, t1);
        for (int i = 0; i < 7; ++i) m7[i] -= t1[i];
        pose_pmul(B1[0], 4, m7, 6, c10);
        for (int i = 0; i < 11; ++i) poly[i] += c10[i];
    }
    double zs[10];
    const int nz = pose_real_roots(poly, zs);
    int n = 0;
    for (int s = 0; s < nz; ++s) {
        const double z = zs[s];
        double R[3][3];
        for (int k = 0; k < 3; ++k) {
            R[k][0] = pose_peval(Bx[k], 3, z);
            R[k][1] = pose_peval(By[k], 3, z);
            R[k][2] = pose_peval(B1[k], 4, z);
        }
        double best[3] = {0.0, 0.0, 0.0}, bn = -1.0;
        for (int k = 0; k < 3; ++k) {
            const double* a = R[k == 2 ? 1 : 0];
            const double* b = R[k == 0 ? 1 : 2];
            const double v[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
            const double nn = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
            if (nn > bn) { bn = nn; best[0] = v[0]; best[1] = v[1]; best[2] = v[2]; }
        }
        if (!(fabs(best[2]) > 0.0)) continue;
        double x = best[0] / best[2], y = best[1] / best[2];
        if (!isfinite(x) || !isfinite(y)) continue;
        double zz = z;
        pose_polish(M, x, y, zz);
        double nn = 0.0;
        for (int e = 0; e < 9; ++e) {
            Es[n][e] = x * L[e][0] + y * L[e][1] + zz * L[e][2] + L[e][3];
            nn += Es[n][e] * Es[n][e];
        }
        if (!(nn > 0.0) || !isfinite(nn)) continue;     // not a solution: the next root takes this slot
        if (sol_z) sol_z[n] = zz;
        ++n;
    }
    return n;
}

// ---- 3 x 3 SVD for essential matrices ----

// eigenvectors of the symmetric 3 x 3 S by cyclic Jacobi (fixed 12 sweeps): columns of V, eigenvalues on S's diagonal
PSV_HD void pose_jacobi3(double (&S)[9], double (&V)[9])
{
    for (int k = 0; k < 9; ++k) V[k] = (k % 4 == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 12; ++sweep) {
        for (int k = 0; k < 3; ++k) {
            const int p = k == 2 ? 1 : 0, q = k == 0 ? 1 : 2;
            const double apq = S[3 * p + q];
            if (fabs(apq) < 1e-300) continue;
            const double th = (S[4 * q] - S[4 * p]) / (2.0 * apq);
            const double t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
            const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
            for (int r = 0; r < 3; ++r) {
                const double a = S[3 * r + p], b = S[3 * r + q];
                S[3 * r + p] = c * a - s * b; S[3 * r + q] = s * a + c * b;
            }
            for (int r = 0; r < 3; ++r) {
                const double a = S[3 * p + r], b = S[3 * q + r];
                S[3 * p + r] = c * a - s * b; S[3 * q + r] = s * a + c * b;
                const double va = V[3 * r + p], vb = V[3 * r + q];
                V[3 * r + p] = c * va - s * vb; V[3 * r + q] = s * va + c * vb;
            }
        }
    }
}

PSV_HD void pose_cross(const double* a, const double* b, double* c)
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

PSV_HD bool pose_unit(double* v)
{
    const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    if (!(n > 0.0) || !isfinite(n)) return false;
    v[0] /= n; v[1] /= n; v[2] /= n;
    return true;
}

// E = U diag(s1, s2, s3) V^T with det U = det V = +1: v1, v2 the eigenvectors of E^T E of the two largest eigenvalues,
// v3 = v1 x v2; u1 = E v1 / |E v1|, u2 = the unit part of E v2 orthogonal to u1, u3 = u1 x u2.  U[k], V[k] are the
// k-th singular vectors.  False when E has rank < 2.
PSV_HD bool pose_svd(const double (&E)[9], double (&U)[3][3], double (&V)[3][3])
{
    double S[9], Q[9];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) S[3 * a + b] = E[a] * E[b] + E[3 + a] * E[3 + b] + E[6 + a] * E[6 + b];
    pose_jacobi3(S, Q);
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2 - i; ++j)
            if (S[4 * o[j + 1]] > S[4 * o[j]]) { const int t = o[j]; o[j] = o[j + 1]; o[j + 1] = t; }
    for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 3; ++r) V[k][r] = Q[3 * r + o[k]];
    pose_cross(V[0], V[1], V[2]);
    if (!pose_unit(V[2])) return false;
    for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 3; ++r) U[k][r] = E[3 * r] * V[k][0] + E[3 * r + 1] * V[k][1] + E[3 * r + 2] * V[k][2];
    if (!pose_unit(U[0])) return false;
    const double d = U[0][0] * U[1][0] + U[0][1] * U[1][1] + U[0][2] * U[1][2];
    for (int r = 0; r < 3; ++r) U[1][r] -= d * U[0][r];
    if (!pose_unit(U[1])) return false;
    pose_cross(U[0], U[1], U[2]);
    return true;
}

// the four (R, t) of E in the header's order: (U W V^T, +u3), (U W V^T, -u3), (U W^T V^T, +u3), (U W^T V^T, -u3)
PSV_HD void pose_candidates(const double (&U)[3][3], const double (&V)[3][3], double (&R)[4][9], double (&t)[4][3])
{
    // U W V^T = -u1 v2^T + u2 v1^T + u3 v3^T; U W^T V^T = u1 v2^T - u2 v1^T + u3 v3^T
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            const double s = U[1][a] * V[0][b] - U[0][a] * V[1][b], w = U[2][a] * V[2][b];
            R[0][3 * a + b] = R[1][3 * a + b] = s + w;
            R[2][3 * a + b] = R[3][3 * a + b] = w - s;
        }
    for (int r = 0; r < 3; ++r) {
        t[0][r] = t[2][r] = U[2][r];
        t[1][r] = t[3][r] = -U[2][r];
    }
}

// The two-ray rule of triangulation: (d_l, d_r) minimising |d_l a + t - d_r b|^2 by the 2 x 2 normal equations (Cramer),
// for rays d_l a from t and d_r b from the origin.  True when det = (a.a)(b.b) - (a.b)^2 > 1e-12 (a.a)(b.b), d_l > 0 and
// d_r > 0.  Shared by ps_relative_pose_batch (pose_front) and ps_triangulate_tracks (k_triangulate.cu).
PSV_HD bool pose_two_rays(const double* a, const double* b, const double* t, double& dl, double& dr)
{
    const double aa = a[0] * a[0] + a[1] * a[1] + a[2] * a[2], bb = b[0] * b[0] + b[1] * b[1] + b[2] * b[2];
    const double ab = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
    const double at = a[0] * t[0] + a[1] * t[1] + a[2] * t[2], bt = b[0] * t[0] + b[1] * t[1] + b[2] * t[2];
    const double det = aa * bb - ab * ab;
    if (!(det > 1e-12 * (aa * bb))) return false;
    dl = (ab * bt - at * bb) / det;
    dr = (aa * bt - ab * at) / det;
    return dl > 0.0 && dr > 0.0;
}

// Triangulation of one calibrated row under (R, t), X_r = R X_l + t: pose_two_rays with a = R (x_l, y_l, 1), b = (x_r,
// y_r, 1) (b's unit third entry enters every product exactly).  In front when it holds.  *X (optional) = the midpoint
// (d_l x_l + R^T (d_r b - t)) / 2 in the left frame.
PSV_HD bool pose_front(const double* R, const double* t, double xl, double yl, double xr, double yr, double* X = nullptr)
{
    const double a[3] = {R[0] * xl + R[1] * yl + R[2], R[3] * xl + R[4] * yl + R[5], R[6] * xl + R[7] * yl + R[8]};
    const double b[3] = {xr, yr, 1.0};
    double dl, dr;
    if (!pose_two_rays(a, b, t, dl, dr)) return false;
    if (X) {
        const double c0 = dr * xr - t[0], c1 = dr * yr - t[1], c2 = dr - t[2];
        X[0] = 0.5 * (dl * xl + R[0] * c0 + R[3] * c1 + R[6] * c2);
        X[1] = 0.5 * (dl * yl + R[1] * c0 + R[4] * c1 + R[7] * c2);
        X[2] = 0.5 * (dl + R[2] * c0 + R[5] * c1 + R[8] * c2);
    }
    return true;
}

// [t]x R / sqrt(2) (|t| = 1, R a rotation: Frobenius norm 1)
PSV_HD void pose_essential(const double* R, const double* t, double* E)
{
    const double k = 0.7071067811865476;
    for (int c = 0; c < 3; ++c) {
        E[c] = k * (t[1] * R[6 + c] - t[2] * R[3 + c]);
        E[3 + c] = k * (t[2] * R[c] - t[0] * R[6 + c]);
        E[6 + c] = k * (t[0] * R[3 + c] - t[1] * R[c]);
    }
}

// Frobenius norm 1 and the first entry of largest magnitude positive (ps_verify_batch's F scaling); false (and zeros)
// when E is zero or not finite
PSV_HD bool pose_scale(const double* m, double* out)
{
    double nn = 0.0;
    for (int j = 0; j < 9; ++j) nn += m[j] * m[j];
    const double n = sqrt(nn);
    if (!(n > 0.0) || !isfinite(n)) {
        for (int j = 0; j < 9; ++j) out[j] = 0.0;
        return false;
    }
    double rb = m[0];
    for (int j = 1; j < 9; ++j) if (fabs(m[j]) > fabs(rb)) rb = m[j];
    const double k = (rb < 0.0 ? -1.0 : 1.0) / n;
    for (int j = 0; j < 9; ++j) out[j] = m[j] * k;
    return true;
}

// F = K_r^-T E K_l^-1 (double), scaled like ps_verify_batch's F
PSV_HD void pose_pixels(const double* E, const PCam& K, double* F)
{
    double M[9], N[9];
    for (int r = 0; r < 3; ++r) {
        M[3 * r] = E[3 * r] / K.fxl;
        M[3 * r + 1] = E[3 * r + 1] / K.fyl;
        M[3 * r + 2] = E[3 * r + 2] - (K.cxl / K.fxl) * E[3 * r] - (K.cyl / K.fyl) * E[3 * r + 1];
    }
    for (int c = 0; c < 3; ++c) {
        N[c] = M[c] / K.fxr;
        N[3 + c] = M[3 + c] / K.fyr;
        N[6 + c] = M[6 + c] - (K.cxr / K.fxr) * M[c] - (K.cyr / K.fyr) * M[3 + c];
    }
    pose_scale(N, F);
}

} // namespace psb
