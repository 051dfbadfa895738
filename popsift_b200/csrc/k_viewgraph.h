// The cycle error of ps_view_graph_filter (include/popsift_b200_viewgraph.h), in double.  One definition for the
// enumeration kernel (k_viewgraph.cu) and the host check (tests/cpp/viewgraph_math_check.cpp).
#pragma once
#include "k_global.h"

namespace psb {

constexpr double kVgDeg = 3.141592653589793 / 180.0;

// R(x->y) of a pair: its rotation R_p, transposed when the pair is stored as (y, x)
PSV_HD void vg_directed(const double* Rp, bool transposed, double* R)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[3 * i + j] = transposed ? Rp[3 * j + i] : Rp[3 * i + j];
}

// The cycle error of the triangle a < b < c in degrees: |Log(R(c->a) (R(b->c) R(a->b)))|.  Rab, Rbc, Rca are the rotations
// of the pairs joining (a, b), (b, c) and (c, a) as stored; t_ab is true when the first is stored as (b, a), t_bc when the
// second is stored as (c, b), t_ca when the third is stored as (a, c).
PSV_HD double vg_cycle_error(const double* Rab, bool t_ab, const double* Rbc, bool t_bc, const double* Rca, bool t_ca)
{
    double A[9], B[9], C[9], BA[9], M[9], w[3];
    vg_directed(Rab, t_ab, A);
    vg_directed(Rbc, t_bc, B);
    vg_directed(Rca, t_ca, C);
    gl_mul(B, A, BA);
    gl_mul(C, BA, M);
    gl_log(M, w);
    return sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]) / kVgDeg;
}

} // namespace psb
