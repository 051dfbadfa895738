// The per-voxel math of ps_tsdf_integrate and ps_tsdf_mesh (include/popsift_b200_mesh.h): the grid point, the projection,
// the truncated signed distance, the running averages, the Kuhn split and its triangle table, and the edge vertex.  One
// definition for the kernels (k_mesh.cu) and the host check (tests/cpp/mesh_math_check.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#include "k_verify_sample.h"   // PSV_HD

namespace psb {

// one view of ps_tsdf_integrate (168 bytes): K = (fx, fy, cx, cy), the pose, the image, its maps and its size
struct TsView {
    double K[4], R[9], t[3];
    const uint8_t* img;
    const float* depth;
    const uint8_t* ncons;
    int64_t pitch;
    int32_t w, h;
};

// X_g = origin + voxel (i, j, k), in double
PSV_HD void ts_point(const double* origin, double voxel, int i, int j, int k, double* X)
{
    X[0] = origin[0] + voxel * (double)i;
    X[1] = origin[1] + voxel * (double)j;
    X[2] = origin[2] + voxel * (double)k;
}

// step 1: X_c = R X + t, each row ((R_r0 X + R_r1 Y) + R_r2 Z) + t_r
PSV_HD void ts_to_camera(const double* R, const double* t, const double* X, double* Xc)
{
    for (int r = 0; r < 3; ++r) Xc[r] = R[3 * r] * X[0] + R[3 * r + 1] * X[1] + R[3 * r + 2] * X[2] + t[r];
}

// step 2: the pixel q of a camera-frame point; false when it is not in front or q is outside the w x h image
PSV_HD bool ts_pixel(const double* K, int w, int h, const double* Xc, int& qx, int& qy)
{
    if (!(Xc[2] > 0.0)) return false;
    const double u = K[0] * Xc[0] / Xc[2] + K[2], v = K[1] * Xc[1] / Xc[2] + K[3];
    const double fu = floor(u + 0.5), fv = floor(v + 0.5);
    if (!(fu >= 0.0 && fu < (double)w && fv >= 0.0 && fv < (double)h)) return false;
    qx = (int)fu;
    qy = (int)fv;
    return true;
}

// steps 4 and 5: tau of depth D at camera depth z; false when the point lies more than trunc behind the surface
PSV_HD bool ts_tau(float D, double z, float trunc, float& tau)
{
    const double sdf = (double)D - z;
    if (sdf < -(double)trunc) return false;
    tau = (float)fmin(1.0, sdf / (double)trunc);
    return true;
}

// step 6
PSV_HD void ts_update(float& T, float& W, float& G, float tau, float grey)
{
    const float Wn = W + 1.0f;
    T = (T * W + tau) / Wn;
    G = (G * W + grey) / Wn;
    W = Wn;
}

// The frustum test of one block corner: bit 0 in front (z > 0), bits 1-4 beyond the left, right, top or bottom edge by
// more than one pixel.  The projection of a box in front of the camera is the hull of its corners' projections, so when
// the AND of the 8 corners' codes has bit 0 and one of bits 1-4, no grid point of the box reaches step 3; the margin of a
// pixel covers the rounding of the per-point projection.
PSV_HD unsigned ts_corner_code(const TsView& V, const double* X)
{
    double Xc[3];
    ts_to_camera(V.R, V.t, X, Xc);
    if (!(Xc[2] > 0.0)) return 0u;
    const double u = V.K[0] * Xc[0] / Xc[2] + V.K[2], v = V.K[1] * Xc[1] / Xc[2] + V.K[3];
    return 1u | (u < -1.5 ? 2u : 0u) | (u > (double)V.w + 0.5 ? 4u : 0u) | (v < -1.5 ? 8u : 0u) | (v > (double)V.h + 0.5 ? 16u : 0u);
}

PSV_HD bool ts_block_unseen(unsigned code_and) { return (code_and & 1u) && (code_and & 30u); }

// ---- extraction

// the tables live in constant memory on the device; a function that reads them is device-only in the kernels' build and
// inline in the host check's
#ifdef __CUDACC__
#define TS_TABLE __constant__
#define TS_TABLE_FN __device__ __forceinline__
#else
#define TS_TABLE
#define TS_TABLE_FN inline
#endif

// corner codes of the 6 Kuhn tetrahedra (step 2 of ps_tsdf_mesh)
TS_TABLE constexpr uint8_t kKuhnTet[6][4] = {{0, 1, 3, 7}, {0, 5, 1, 7}, {0, 3, 2, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 6, 4, 7}};

// step 4 as a table: per tetrahedron and case (bit m: local corner m inside), the triangles (0, 1 or 2) and their
// corners as edges, lower corner << 3 | direction code; tests/mesh_oracle.py generates the same table from the rule
TS_TABLE constexpr uint8_t kTetTriCount[16] = {0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0};

TS_TABLE constexpr uint8_t kTetTri[6][16][2][3] = {
    {{{0, 0, 0}, {0, 0, 0}}, {{1, 3, 7}, {0, 0, 0}}, {{1, 14, 10}, {0, 0, 0}}, {{3, 7, 14}, {3, 14, 10}}, {{3, 10, 28}, {0, 0, 0}}, {{1, 28, 7}, {1, 10, 28}}, {{1, 14, 28}, {1, 28, 3}}, {{7, 14, 28}, {0, 0, 0}}, {{7, 28, 14}, {0, 0, 0}}, {{1, 3, 28}, {1, 28, 14}}, {{1, 28, 10}, {1, 7, 28}}, {{3, 28, 10}, {0, 0, 0}}, {{3, 10, 14}, {3, 14, 7}}, {{1, 10, 14}, {0, 0, 0}}, {{1, 7, 3}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
    {{{0, 0, 0}, {0, 0, 0}}, {{5, 1, 7}, {0, 0, 0}}, {{5, 42, 12}, {0, 0, 0}}, {{1, 7, 42}, {1, 42, 12}}, {{1, 12, 14}, {0, 0, 0}}, {{5, 14, 7}, {5, 12, 14}}, {{5, 42, 14}, {5, 14, 1}}, {{7, 42, 14}, {0, 0, 0}}, {{7, 14, 42}, {0, 0, 0}}, {{5, 1, 14}, {5, 14, 42}}, {{5, 14, 12}, {5, 7, 14}}, {{1, 14, 12}, {0, 0, 0}}, {{1, 12, 42}, {1, 42, 7}}, {{5, 12, 42}, {0, 0, 0}}, {{5, 7, 1}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
    {{{0, 0, 0}, {0, 0, 0}}, {{3, 2, 7}, {0, 0, 0}}, {{3, 28, 17}, {0, 0, 0}}, {{2, 7, 28}, {2, 28, 17}}, {{2, 17, 21}, {0, 0, 0}}, {{3, 21, 7}, {3, 17, 21}}, {{3, 28, 21}, {3, 21, 2}}, {{7, 28, 21}, {0, 0, 0}}, {{7, 21, 28}, {0, 0, 0}}, {{3, 2, 21}, {3, 21, 28}}, {{3, 21, 17}, {3, 7, 21}}, {{2, 21, 17}, {0, 0, 0}}, {{2, 17, 28}, {2, 28, 7}}, {{3, 17, 28}, {0, 0, 0}}, {{3, 7, 2}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
    {{{0, 0, 0}, {0, 0, 0}}, {{2, 6, 7}, {0, 0, 0}}, {{2, 21, 20}, {0, 0, 0}}, {{6, 7, 21}, {6, 21, 20}}, {{6, 20, 49}, {0, 0, 0}}, {{2, 49, 7}, {2, 20, 49}}, {{2, 21, 49}, {2, 49, 6}}, {{7, 21, 49}, {0, 0, 0}}, {{7, 49, 21}, {0, 0, 0}}, {{2, 6, 49}, {2, 49, 21}}, {{2, 49, 20}, {2, 7, 49}}, {{6, 49, 20}, {0, 0, 0}}, {{6, 20, 21}, {6, 21, 7}}, {{2, 20, 21}, {0, 0, 0}}, {{2, 7, 6}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
    {{{0, 0, 0}, {0, 0, 0}}, {{4, 5, 7}, {0, 0, 0}}, {{4, 35, 33}, {0, 0, 0}}, {{5, 7, 35}, {5, 35, 33}}, {{5, 33, 42}, {0, 0, 0}}, {{4, 42, 7}, {4, 33, 42}}, {{4, 35, 42}, {4, 42, 5}}, {{7, 35, 42}, {0, 0, 0}}, {{7, 42, 35}, {0, 0, 0}}, {{4, 5, 42}, {4, 42, 35}}, {{4, 42, 33}, {4, 7, 42}}, {{5, 42, 33}, {0, 0, 0}}, {{5, 33, 35}, {5, 35, 7}}, {{4, 33, 35}, {0, 0, 0}}, {{4, 7, 5}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
    {{{0, 0, 0}, {0, 0, 0}}, {{6, 4, 7}, {0, 0, 0}}, {{6, 49, 34}, {0, 0, 0}}, {{4, 7, 49}, {4, 49, 34}}, {{4, 34, 35}, {0, 0, 0}}, {{6, 35, 7}, {6, 34, 35}}, {{6, 49, 35}, {6, 35, 4}}, {{7, 49, 35}, {0, 0, 0}}, {{7, 35, 49}, {0, 0, 0}}, {{6, 4, 35}, {6, 35, 49}}, {{6, 35, 34}, {6, 7, 35}}, {{4, 35, 34}, {0, 0, 0}}, {{4, 34, 49}, {4, 49, 7}}, {{6, 34, 49}, {0, 0, 0}}, {{6, 7, 4}, {0, 0, 0}}, {{0, 0, 0}, {0, 0, 0}}},
};

// the 19 edges of a split cell (step 3), lower corner << 3 | direction: a & d == 0, in (d, a) order
TS_TABLE constexpr uint8_t kCellEdge[19] = {1, 17, 33, 49, 2, 10, 34, 42, 3, 35, 4, 12, 20, 28, 5, 21, 6, 14, 7};

// the case of tetrahedron t in a cell whose inside corners are the bits of mask
TS_TABLE_FN int ts_tet_case(int t, unsigned mask)
{
    int c = 0;
    for (int m = 0; m < 4; ++m) c |= (int)((mask >> kKuhnTet[t][m]) & 1u) << m;
    return c;
}

// the edges with a sign change (all of them used by a triangle) and the triangles of a cell
TS_TABLE_FN void ts_cell_counts(unsigned mask, int& n_edges, int& n_tris)
{
    n_edges = 0;
    for (int e = 0; e < 19; ++e) {
        const int a = kCellEdge[e] >> 3, b = a + (kCellEdge[e] & 7);
        n_edges += (int)(((mask >> a) ^ (mask >> b)) & 1u);
    }
    n_tris = 0;
    for (int t = 0; t < 6; ++t) n_tris += kTetTriCount[ts_tet_case(t, mask)];
}

// step 5: the vertex of the edge from lower corner (ax, ay, az) in direction d; o, h: origin and voxel rounded to float
PSV_HD void ts_vertex(const float* o, float h, int ax, int ay, int az, int d, float Ta, float Tb, float Ga, float Gb, float* X,
                      float& grey)
{
    const float s = Ta / (Ta - Tb);
    X[0] = o[0] + h * ((float)ax + s * (float)(d & 1));
    X[1] = o[1] + h * ((float)ay + s * (float)((d >> 1) & 1));
    X[2] = o[2] + h * ((float)az + s * (float)((d >> 2) & 1));
    grey = Ga + s * (Gb - Ga);
}

} // namespace psb
