// The eligibility test of guided matching (include/popsift_b200_guided.h): may right keypoint (X, Y) match left keypoint
// (x, y) under a pair's homography or fundamental matrix?  One definition for the kernels (k_match.cu, k_match_u8.cu) and
// the host check (tests/cpp/guided_mask.cpp).  Every operation is rounded explicitly (one fma is one rounding), so the
// host and the device agree bit for bit.
//
//   t2 = t * t                                                        (float32, t the threshold in pixels)
//   homography  (u, v, w) = H (x, y, 1)                               per row
//               du = fma(-X, w, u), dv = fma(-Y, w, v)
//               eligible when fma(du, du, dv * dv) < t2 * (w * w)
//   fundamental (a0, a1, a2) = F (x, y, 1), ra = fma(a0, a0, a1 * a1)  per row
//               b0 = fma(F00, X, fma(F10, Y, F20)), b1 = fma(F01, X, fma(F11, Y, F21)), cb = fma(b0, b0, b1 * b1)
//                                                                     per column
//               e = fma(X, a0, fma(Y, a1, a2))
//               eligible when e * e < t2 * (ra + cb)
//   with H x = (fma(m0, x, fma(m1, y, m2)), fma(m3, x, fma(m4, y, m5)), fma(m6, x, fma(m7, y, m8))).
// The comparison is strict: a zero model makes nothing eligible (0 < 0 is false), and so does any NaN.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PSG_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define PSG_HD inline
#endif

namespace psb {

enum { kGuidedH = 0, kGuidedF = 1 };      // = PS_GEOM_HOMOGRAPHY / PS_GEOM_FUNDAMENTAL

PSG_HD float g_fma(float a, float b, float c)
{
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return std::fmaf(a, b, c);
#endif
}
PSG_HD float g_mul(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
PSG_HD float g_add(float a, float b)
{
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// the per-row part: H -> (u, v, w, t2 w^2); F -> (a0, a1, a2, ra)
struct GuidedRow { float p0, p1, p2, p3; };

template <int MODEL>
PSG_HD GuidedRow guided_row(const float (&m)[9], float t2, float x, float y)
{
    GuidedRow r;
    r.p0 = g_fma(m[0], x, g_fma(m[1], y, m[2]));
    r.p1 = g_fma(m[3], x, g_fma(m[4], y, m[5]));
    r.p2 = g_fma(m[6], x, g_fma(m[7], y, m[8]));
    if (MODEL == kGuidedH) r.p3 = g_mul(t2, g_mul(r.p2, r.p2));
    else r.p3 = g_fma(r.p0, r.p0, g_mul(r.p1, r.p1));
    return r;
}

// the per-column part of F: cb = b0^2 + b1^2 (unused under H)
template <int MODEL>
PSG_HD float guided_col(const float (&m)[9], float X, float Y)
{
    if (MODEL == kGuidedH) return 0.0f;
    const float b0 = g_fma(m[0], X, g_fma(m[3], Y, m[6]));
    const float b1 = g_fma(m[1], X, g_fma(m[4], Y, m[7]));
    return g_fma(b0, b0, g_mul(b1, b1));
}

template <int MODEL>
PSG_HD bool guided_ok(const GuidedRow& r, float cb, float t2, float X, float Y)
{
    if (MODEL == kGuidedH) {
        const float du = g_fma(-X, r.p2, r.p0), dv = g_fma(-Y, r.p2, r.p1);
        return g_fma(du, du, g_mul(dv, dv)) < r.p3;
    } else {
        const float e = g_fma(X, r.p0, g_fma(Y, r.p1, r.p2));
        return g_mul(e, e) < g_mul(t2, g_add(r.p3, cb));
    }
}

// the whole test for one (left point, right point)
template <int MODEL>
PSG_HD bool guided_eligible(const float (&m)[9], float t2, float x, float y, float X, float Y)
{
    return guided_ok<MODEL>(guided_row<MODEL>(m, t2, x, y), guided_col<MODEL>(m, X, Y), t2, X, Y);
}

} // namespace psb
