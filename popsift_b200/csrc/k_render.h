// The per-element math of ps_mesh_render and ps_mesh_texture (include/popsift_b200_render.h): the projection, the edge
// functions, the perspective-correct depth, the z-buffer key, the visibility probe, the facing test, the texel's clamped
// barycentrics and the bilinear sample.  One definition for the kernels (k_render.cu) and the host check
// (tests/cpp/render_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "k_verify_sample.h"   // PSV_HD

namespace psb {

// one view of ps_mesh_render (144 bytes): K = (fx, fy, cx, cy), the pose, the z-buffer offset of its first pixel and its size
struct RdView {
    double K[4], R[9], t[3];
    int64_t off;
    int32_t w, h;
};

// one view of ps_mesh_texture (184 bytes): as RdView with the camera centre, the image and the depth map
struct TxView {
    double K[4], R[9], t[3], c[3];
    const uint8_t* img;
    const float* depth;
    int64_t pitch;
    int32_t w, h;
};

// render step 1: X_c = R X + t, each row ((R_r0 X + R_r1 Y) + R_r2 Z) + t_r, and p; false unless X_c is finite with
// z >= z_near and p is finite
PSV_HD bool rd_project(const double* K, const double* R, const double* t, const double* X, double z_near, double* p, double& z)
{
    double Xc[3];
    for (int r = 0; r < 3; ++r) Xc[r] = R[3 * r] * X[0] + R[3 * r + 1] * X[1] + R[3 * r + 2] * X[2] + t[r];
    if (!(isfinite(Xc[0]) && isfinite(Xc[1]) && isfinite(Xc[2]) && Xc[2] >= z_near)) return false;
    p[0] = K[0] * Xc[0] / Xc[2] + K[2];
    p[1] = K[1] * Xc[1] / Xc[2] + K[3];
    z = Xc[2];
    return isfinite(p[0]) && isfinite(p[1]);
}

// render step 2: E(a, b; x, y) = (b_x - a_x)(y - a_y) - (b_y - a_y)(x - a_x)
PSV_HD double rd_edge(const double* a, const double* b, double x, double y)
{
    return (b[0] - a[0]) * (y - a[1]) - (b[1] - a[1]) * (x - a[0]);
}

// render steps 2-3: A and the candidate box [x0, x1] x [y0, y1] clamped to the w x h image; false when the triangle is not
// drawn (A zero or not finite, or an empty box)
PSV_HD bool rd_setup(const double (*p)[2], int w, int h, double& A, int* box)
{
    A = rd_edge(p[0], p[1], p[2][0], p[2][1]);
    if (!(isfinite(A) && A != 0.0)) return false;
    const double lx = fmax(ceil(fmin(fmin(p[0][0], p[1][0]), p[2][0])), 0.0);
    const double hx = fmin(floor(fmax(fmax(p[0][0], p[1][0]), p[2][0])), (double)(w - 1));
    const double ly = fmax(ceil(fmin(fmin(p[0][1], p[1][1]), p[2][1])), 0.0);
    const double hy = fmin(floor(fmax(fmax(p[0][1], p[1][1]), p[2][1])), (double)(h - 1));
    if (!(lx <= hx && ly <= hy)) return false;
    box[0] = (int)lx;
    box[1] = (int)hx;
    box[2] = (int)ly;
    box[3] = (int)hy;
    return true;
}

// render steps 3-4 at pixel (x, y): true when covered, with the depth rounded to float
PSV_HD bool rd_cover(const double (*p)[2], const double* z, double A, int x, int y, float& zf)
{
    const double fx = (double)x, fy = (double)y;
    const double E0 = rd_edge(p[1], p[2], fx, fy), E1 = rd_edge(p[2], p[0], fx, fy), E2 = rd_edge(p[0], p[1], fx, fy);
    if (A > 0.0 ? !(E0 >= 0.0 && E1 >= 0.0 && E2 >= 0.0) : !(E0 <= 0.0 && E1 <= 0.0 && E2 <= 0.0)) return false;
    const double l0 = E0 / A, l1 = E1 / A, l2 = E2 / A;
    zf = (float)(1.0 / (l0 / z[0] + l1 / z[1] + l2 / z[2]));
    return true;
}

// render step 5: the z-buffer key; every key of a covered pixel is below kEmptyKey (the bits of a NaN)
constexpr unsigned long long kEmptyKey = ~0ull;

PSV_HD unsigned long long rd_key(float z, int m)
{
    uint32_t b;
    memcpy(&b, &z, 4);
    return (unsigned long long)b << 32 | (unsigned long long)(uint32_t)m;
}

// texture step 1: centroid and normal of a triangle
PSV_HD void tx_frame(const double* V0, const double* V1, const double* V2, double* C, double* n)
{
    double a[3], b[3];
    for (int k = 0; k < 3; ++k) {
        C[k] = (V0[k] + V1[k] + V2[k]) / 3.0;
        a[k] = V1[k] - V0[k];
        b[k] = V2[k] - V0[k];
    }
    n[0] = a[1] * b[2] - a[2] * b[1];
    n[1] = a[2] * b[0] - a[0] * b[2];
    n[2] = a[0] * b[1] - a[1] * b[0];
}

// texture step 2, facing: n.d > 0 and n.d >= (min_cos |n|) |d| with d = c - C
PSV_HD bool tx_facing(const double* n, const double* C, const double* c, float min_cos)
{
    const double d[3] = {c[0] - C[0], c[1] - C[1], c[2] - C[2]};
    const double nd = n[0] * d[0] + n[1] * d[1] + n[2] * d[2];
    const double nn = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]), dd = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    return nd > 0.0 && nd >= (double)min_cos * nn * dd;
}

// texture step 2, visibility of one probe P in view V: projects, nearest pixel inside, not occluded (tol1 = 1 + depth_tol)
PSV_HD bool tx_probe(const TxView& V, const double* P, double z_near, double tol1, double* p)
{
    double z;
    if (!rd_project(V.K, V.R, V.t, P, z_near, p, z)) return false;
    const double qx = floor(p[0] + 0.5), qy = floor(p[1] + 0.5);
    if (!(qx >= 0.0 && qx < (double)V.w && qy >= 0.0 && qy < (double)V.h)) return false;
#ifdef __CUDA_ARCH__
    const float D = __ldg(V.depth + (size_t)qy * V.w + (size_t)qx);
#else
    const float D = V.depth[(size_t)qy * V.w + (size_t)qx];
#endif
    return !(D > 0.0f && z > (double)D * tol1);
}

// texture step 5: the clamped (u, v) of texel (i, j) of a cell (b = 1)
PSV_HD void tx_uv(int i, int j, int cell, double& u, double& v)
{
    const double s = (double)(cell - 2);
    u = fmax(((double)i + 0.5 - 1.0) / s, 0.0);
    v = fmax(((double)j + 0.5 - 1.0) / s, 0.0);
    if (u + v > 1.0) {
        u = fmin(fmax((u - v + 1.0) / 2.0, 0.0), 1.0);
        v = 1.0 - u;
    }
}

// texture step 6: the bilinear sample of a w x h image at (x, y), clamped to [0, w - 1] x [0, h - 1]
PSV_HD double tx_bilinear(const uint8_t* img, int64_t pitch, int w, int h, double x, double y)
{
    x = fmin(fmax(x, 0.0), (double)(w - 1));
    y = fmin(fmax(y, 0.0), (double)(h - 1));
    const int fx = (int)floor(x), fy = (int)floor(y);
    const int u0 = fx < w - 2 ? fx : w - 2, v0 = fy < h - 2 ? fy : h - 2;
    const double a = x - (double)u0, c = y - (double)v0;
    const uint8_t* r0 = img + (size_t)v0 * pitch + u0;
    const uint8_t* r1 = r0 + pitch;
#ifdef __CUDA_ARCH__
    const double I00 = __ldg(r0), I10 = __ldg(r0 + 1), I01 = __ldg(r1), I11 = __ldg(r1 + 1);
#else
    const double I00 = r0[0], I10 = r0[1], I01 = r1[0], I11 = r1[1];
#endif
    return (1.0 - c) * ((1.0 - a) * I00 + a * I10) + c * ((1.0 - a) * I01 + a * I11);
}

// texture step 6: floor(S + 1/2) clamped to 0 .. 255, NaN to 0
PSV_HD uint8_t tx_round(double S)
{
    return (uint8_t)fmin(fmax(floor(S + 0.5), 0.0), 255.0);
}

} // namespace psb
