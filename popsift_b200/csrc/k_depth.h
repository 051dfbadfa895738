// The per-pixel math of ps_depth_maps and ps_depth_filter (include/popsift_b200_depth.h): the plane-induced warp, the NCC
// from the five window sums, the best-K aggregation, the sub-plane parabola and the consistency test.  One definition for
// the kernels (k_depth.cu) and the host check (tests/cpp/depth_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_verify_sample.h"   // PSV_HD

namespace psb {

// One (reference, source) pair's homography: (u, v, w) = H (x, y, 1) + iota b, H = K_s R_s R_r^T K_r^-1 and
// b = K_s (t_s - R_s R_r^T t_r), both computed in double on the host (step 3 of ps_depth_maps)
template <class T>
PSV_HD bool dp_warp(const T* H, const T* b, T x, T y, T iota, T w_s, T h_s, T& u, T& v)
{
    const T hx = (H[0] * x + H[1] * y + H[2]) + iota * b[0];
    const T hy = (H[3] * x + H[4] * y + H[5]) + iota * b[1];
    const T hz = (H[6] * x + H[7] * y + H[8]) + iota * b[2];
    if (!(hz > T(0))) return false;
    u = hx / hz;
    v = hy / hz;
    return u >= T(0) && u <= w_s - T(1) && v >= T(0) && v <= h_s - T(1);
}

// The homography of step 3 from the two cameras (fx, fy, cx, cy) and poses (R row-major, t), in double
PSV_HD void dp_homography(const double* Kr, const double* Rr, const double* tr, const double* Ks, const double* Rs,
                          const double* ts, double* H, double* b)
{
    double Rrel[9], trel[3], M[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rrel[3 * i + j] = Rs[3 * i] * Rr[3 * j] + Rs[3 * i + 1] * Rr[3 * j + 1] + Rs[3 * i + 2] * Rr[3 * j + 2];
    for (int i = 0; i < 3; ++i) trel[i] = ts[i] - (Rrel[3 * i] * tr[0] + Rrel[3 * i + 1] * tr[1] + Rrel[3 * i + 2] * tr[2]);
    // M = Rrel K_r^-1: K_r^-1 (x, y, 1) = ((x - cx) / fx, (y - cy) / fy, 1)
    for (int i = 0; i < 3; ++i) {
        M[3 * i] = Rrel[3 * i] / Kr[0];
        M[3 * i + 1] = Rrel[3 * i + 1] / Kr[1];
        M[3 * i + 2] = Rrel[3 * i + 2] - Rrel[3 * i] * Kr[2] / Kr[0] - Rrel[3 * i + 1] * Kr[3] / Kr[1];
    }
    // rows of K_s applied: (fx m0 + cx m2, fy m1 + cy m2, m2)
    for (int j = 0; j < 3; ++j) {
        H[j] = Ks[0] * M[j] + Ks[2] * M[6 + j];
        H[3 + j] = Ks[1] * M[3 + j] + Ks[3] * M[6 + j];
        H[6 + j] = M[6 + j];
    }
    b[0] = Ks[0] * trel[0] + Ks[2] * trel[2];
    b[1] = Ks[1] * trel[1] + Ks[3] * trel[2];
    b[2] = trel[2];
}

// Step 5: the NCC cost of one source from the window sums; false when the source is not valid for the pixel.  The sums
// may be taken over values shifted by a constant (the device uses I - 128): var_r, var_s and m AB - A B do not change.
PSV_HD bool dp_ncc(double m, double A, double AA, double B, double BB, double AB, double floor_m2, double& c)
{
    const double vr = m * AA - A * A, vs = m * BB - B * B;
    if (!(vr > floor_m2) || !(vs > floor_m2)) return false;
    const double r = (m * AB - A * B) / sqrt(vr * vs);
    c = fmin(fmax(1.0 - r, 0.0), 2.0);
    return true;
}

// Step 6 on the device: c inserted into the ascending list a[0 .. K - 1] (+inf where empty)
template <int K>
PSV_HD void dp_insert(float (&a)[K], float c)
{
#pragma unroll
    for (int j = 0; j < K; ++j) {
        const float lo = fminf(a[j], c);
        c = fmaxf(a[j], c);
        a[j] = lo;
    }
}

// Step 6: the mean of the min(top_k, nv) smallest of the ascending a[0 .. K - 1] (top_k <= K), summed in ascending order;
// +inf when nv < min_sources
template <class T, int K>
PSV_HD T dp_mean(const T (&a)[K], int nv, int top_k, int min_sources)
{
    if (nv < min_sources || nv == 0) return (T)INFINITY;
    const int kk = nv < top_k ? nv : top_k;
    T s = 0;
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (j < kk) s += a[j];
    return s / (T)kk;
}

// Step 8: the sub-plane offset delta of the winner k of n planes
template <class T>
PSV_HD T dp_parabola(T cm, T c0, T cp, int k, int n)
{
    if (!(k > 0 && k < n - 1) || !isfinite(cm) || !isfinite(cp)) return T(0);
    const T den = cm - T(2) * c0 + cp;
    if (!(den > T(0))) return T(0);
    const T d = (cm - cp) / (T(2) * den);
    return d < T(-0.5) ? T(-0.5) : (d > T(0.5) ? T(0.5) : d);
}

// a camera for the filter: K (fx, fy, cx, cy), the pose and the image size
struct DpCam {
    double K[4], R[9], t[3];
    int32_t w, h;
};

// the world point of pixel (x, y) at depth D: R^T (D K^-1 (x, y, 1) - t)
PSV_HD void dp_backproject(const DpCam& c, double x, double y, double D, double* X)
{
    const double p[3] = {D * (x - c.K[2]) / c.K[0] - c.t[0], D * (y - c.K[3]) / c.K[1] - c.t[1], D - c.t[2]};
    for (int k = 0; k < 3; ++k) X[k] = c.R[k] * p[0] + c.R[3 + k] * p[1] + c.R[6 + k] * p[2];
}

PSV_HD void dp_to_camera(const DpCam& c, const double* X, double* Xc)
{
    for (int r = 0; r < 3; ++r) Xc[r] = c.R[3 * r] * X[0] + c.R[3 * r + 1] * X[1] + c.R[3 * r + 2] * X[2] + c.t[r];
}

// The first half of ps_depth_filter's test (its step 1): the source pixel (qx, qy) that pixel (x, y) of r at depth D
// lands on, and the depth zs of that point in s; false when it is behind s or outside its image
PSV_HD bool dp_lookup(const DpCam& r, const DpCam& s, double x, double y, double D, int& qx, int& qy, double& zs)
{
    double X[3], Xs[3];
    dp_backproject(r, x, y, D, X);
    dp_to_camera(s, X, Xs);
    if (!(Xs[2] > 0.0)) return false;
    const double u = s.K[0] * Xs[0] / Xs[2] + s.K[2], v = s.K[1] * Xs[1] / Xs[2] + s.K[3];
    if (!(u >= 0.0 && u <= s.w - 1.0 && v >= 0.0 && v <= s.h - 1.0)) return false;
    qx = (int)floor(u + 0.5);
    qy = (int)floor(v + 0.5);
    zs = Xs[2];
    return true;
}

// Steps 2 and 3: source pixel (qx, qy) at depth Dq > 0 projected back into r against pixel (x, y); zs as dp_lookup gave it
PSV_HD bool dp_consistent(const DpCam& r, const DpCam& s, double x, double y, int qx, int qy, double zs, double Dq,
                          double max_reproj, double max_diff)
{
    double X[3], Xr[3];
    dp_backproject(s, (double)qx, (double)qy, Dq, X);
    dp_to_camera(r, X, Xr);
    if (!(Xr[2] > 0.0)) return false;
    const double ex = r.K[0] * Xr[0] / Xr[2] + r.K[2] - x, ey = r.K[1] * Xr[1] / Xr[2] + r.K[3] - y;
    return sqrt(ex * ex + ey * ey) <= max_reproj && fabs(zs - Dq) <= max_diff * Dq;
}

} // namespace psb
