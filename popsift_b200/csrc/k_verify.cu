// Geometric verification of matched pairs, hand-written for sm_90a: the correspondence gather of ps_match_correspondences
// and the batched RANSAC of ps_verify_batch (contract in include/popsift_b200.h).
//
// ps_match_correspondences: corr_gather_kernel, one CTA per pair.  Each row is tested on its own (accept, dedup rule
// against the three rows before it); an order-preserving block scan (warp ballots + a prefix over the warps) compacts
// the kept rows, so no atomic decides the output order.
//
// ps_verify_batch, one workspace (workspace.h), all launches on one stream:
//   1. verify_normalize_kernel  one CTA per pair: centroids and the common scale in double (fixed-order reductions), then
//                               the pair's points as normalised float4 rows and the normalised squared threshold.
//   2. verify_solve_kernel      one lane per minimal sample, in double: the sample hash (k_verify_sample.h), the 4-point
//                               DLT or the 7-point method; writes each hypothesis's normalised float model and count
//                               0 (valid) or -1 (invalid).
//   3. verify_score_kernel      the hot path.  Work items (pair, 128 samples, chunk of correspondences), so a pair of
//                               200 000 correspondences and 10 000 pairs of 200 both fill the SMs.  The chunk streams
//                               through shared memory in tiles (cp.async.bulk + mbarrier, two buffers) read as broadcast
//                               LDS.128; each lane counts its hypotheses' inliers in registers (FP32 CUDA cores, K = 3
//                               contractions), then adds the count to the hypothesis's total (integer atomics: the sum
//                               does not depend on the order).
//   4. verify_select_kernel     one CTA per pair: the winner by (count desc, h asc), the refit (9x9 normal matrix in
//                               double, fixed order; smallest eigenvector by warp-parallel Jacobi; for F the rank-2 step),
//                               the output model in pixels, the mask and its sum.
//   5. verify_taps_kernel       (taps only) every hypothesis's count and pixel model.
#include "k_verify_common.h"
#include "k_verify_sample.h"
#include "ps_internal.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace psb {

namespace {

// ---- correspondence gather -------------------------------------------------------------------------------------------

struct CorrPair {
    const ps_feature* feat_l; const int32_t* rev_l;
    const ps_feature* feat_r; const int32_t* rev_r;
    long long row0;      // first match row / output row of the pair
    int n_l, n_r;
};

constexpr int kGatherThreads = 256;

__device__ __forceinline__ bool corr_keep(const CorrPair& P, const int32_t* m, int i)
{
    const int32_t* row = m + 3 * (P.row0 + i);
    const int best = row[0];
    if (row[2] != 1 || P.n_r <= 0 || best < 0 || best >= P.n_r) return false;
    const int fl = P.rev_l[i], fr = P.rev_r[best];
#pragma unroll
    for (int d = 1; d <= 3; ++d) {
        const int j = i - d;
        if (j < 0) break;
        const int32_t* rj = m + 3 * (P.row0 + j);
        if (rj[2] == 1 && rj[0] >= 0 && rj[0] < P.n_r && P.rev_l[j] == fl && P.rev_r[rj[0]] == fr) return false;
    }
    return true;
}

__global__ void __launch_bounds__(kGatherThreads) corr_gather_kernel(const CorrPair* __restrict__ pairs, const int32_t* __restrict__ match,
                                                                     float4* __restrict__ corr, int32_t* __restrict__ src,
                                                                     int32_t* __restrict__ counts)
{
    const CorrPair P = pairs[blockIdx.x];
    __shared__ int warp_tot[kGatherThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;
    for (int i0 = 0; i0 < P.n_l; i0 += kGatherThreads) {
        const int i = i0 + (int)threadIdx.x;
        const bool keep = i < P.n_l && corr_keep(P, match, i);
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kGatherThreads / 32; ++w) {
            before += w < warp ? warp_tot[w] : 0;
            total += warp_tot[w];
        }
        if (keep) {
            const int o = base + before + __popc(bal & ((1u << lane) - 1u));
            const ps_feature& fl = P.feat_l[P.rev_l[i]];
            const ps_feature& fr = P.feat_r[P.rev_r[match[3 * (P.row0 + i)]]];
            corr[P.row0 + o] = make_float4(fl.xpos, fl.ypos, fr.xpos, fr.ypos);
            src[P.row0 + o] = i;
        }
        base += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[blockIdx.x] = base;
}

// ---- RANSAC ----------------------------------------------------------------------------------------------------------

struct VXform { double cxl, cyl, cxr, cyr, s; float t2, pad; };   // normalised point = s (x - c); t2 = (s t)^2
struct VSolveItem { int pair, s0; };
struct VScoreItem { int pair, s0, c0, c1; };

constexpr int kNormThreads = 256;
constexpr int kSolveThreads = 64;

__global__ void __launch_bounds__(kNormThreads) verify_normalize_kernel(const VPair* __restrict__ pairs, const float4* __restrict__ corr,
                                                                        float4* __restrict__ pts, VXform* __restrict__ xf, double thr)
{
    __shared__ double red[33];
    const VPair P = pairs[blockIdx.x];
    const float4* c = corr + P.start;
    double sx = 0, sy = 0, sxr = 0, syr = 0;
    for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
        const float4 v = c[i];
        sx += v.x; sy += v.y; sxr += v.z; syr += v.w;
    }
    const double inv_n = P.n > 0 ? 1.0 / P.n : 0.0;
    const double cxl = block_sum_d(sx, red) * inv_n, cyl = block_sum_d(sy, red) * inv_n;
    const double cxr = block_sum_d(sxr, red) * inv_n, cyr = block_sum_d(syr, red) * inv_n;
    double sd = 0;
    for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
        const float4 v = c[i];
        sd += sqrt((v.x - cxl) * (v.x - cxl) + (v.y - cyl) * (v.y - cyl)) + sqrt((v.z - cxr) * (v.z - cxr) + (v.w - cyr) * (v.w - cyr));
    }
    const double d = block_sum_d(sd, red) * 0.5 * inv_n;
    const double s = d > 0.0 ? sqrt(2.0) / d : 1.0;
    for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
        const float4 v = c[i];
        pts[P.start + i] = make_float4((float)(s * (v.x - cxl)), (float)(s * (v.y - cyl)), (float)(s * (v.z - cxr)), (float)(s * (v.w - cyr)));
    }
    if (threadIdx.x == 0) xf[blockIdx.x] = VXform{cxl, cyl, cxr, cyr, s, (float)((s * thr) * (s * thr)), 0.0f};
}

// ---- minimal solvers (double, one lane per sample) ----

__device__ __forceinline__ double cross2(double ax, double ay, double bx, double by, double cx, double cy)
{
    return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

__device__ __forceinline__ double det3(const double (&m)[9])
{
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

__device__ __forceinline__ void adj3(const double (&m)[9], double (&a)[9])
{
    a[0] = m[4] * m[8] - m[5] * m[7]; a[1] = m[2] * m[7] - m[1] * m[8]; a[2] = m[1] * m[5] - m[2] * m[4];
    a[3] = m[5] * m[6] - m[3] * m[8]; a[4] = m[0] * m[8] - m[2] * m[6]; a[5] = m[2] * m[3] - m[0] * m[5];
    a[6] = m[3] * m[7] - m[4] * m[6]; a[7] = m[1] * m[6] - m[0] * m[7]; a[8] = m[0] * m[4] - m[1] * m[3];
}

// the projective basis map of four points: columns lambda_j p_j with [p0 p1 p2] lambda = p3
__device__ __forceinline__ void basis4(const double (&x)[4], const double (&y)[4], double (&B)[9])
{
    const double M[9] = {x[0], x[1], x[2], y[0], y[1], y[2], 1.0, 1.0, 1.0};
    double A[9];
    adj3(M, A);
    const double l0 = A[0] * x[3] + A[1] * y[3] + A[2], l1 = A[3] * x[3] + A[4] * y[3] + A[5], l2 = A[6] * x[3] + A[7] * y[3] + A[8];
    B[0] = l0 * x[0]; B[1] = l1 * x[1]; B[2] = l2 * x[2];
    B[3] = l0 * y[0]; B[4] = l1 * y[1]; B[5] = l2 * y[2];
    B[6] = l0;        B[7] = l1;        B[8] = l2;
}

__device__ __forceinline__ bool store_model(const double (&m)[9], float* out)
{
    double nn = 0.0;
#pragma unroll
    for (int j = 0; j < 9; ++j) nn += m[j] * m[j];
    if (!(nn > 0.0) || !isfinite(nn)) return false;
    const double r = 1.0 / sqrt(nn);
#pragma unroll
    for (int j = 0; j < 9; ++j) out[j] = (float)(m[j] * r);
    return true;
}

// 4-point homography in normalised coordinates: H = B_r adj(B_l) (the DLT's unique solution for four points in general
// position); false when three points are collinear in either image
__device__ __forceinline__ bool solve_h4(const float4 (&p)[4], double (&H)[9])
{
    double xl[4], yl[4], xr[4], yr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { xl[j] = p[j].x; yl[j] = p[j].y; xr[j] = p[j].z; yr[j] = p[j].w; }
    constexpr double eps = 1e-7;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const int a = t == 0 ? 1 : 0, b = t <= 1 ? 2 : 1, c = t <= 2 ? 3 : 2;   // the triple without point t
        if (fabs(cross2(xl[a], yl[a], xl[b], yl[b], xl[c], yl[c])) < eps) return false;
        if (fabs(cross2(xr[a], yr[a], xr[b], yr[b], xr[c], yr[c])) < eps) return false;
    }
    double Bl[9], Br[9], Al[9];
    basis4(xl, yl, Bl);
    basis4(xr, yr, Br);
    adj3(Bl, Al);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) H[3 * r + c] = Br[3 * r] * Al[c] + Br[3 * r + 1] * Al[3 + c] + Br[3 * r + 2] * Al[6 + c];
    return true;
}

// real roots of a l^3 + b l^2 + c l + d, ascending; returns their number
__device__ __forceinline__ int cubic_roots(double a, double b, double c, double d, double (&r)[3])
{
    const double sc = fmax(fmax(fabs(a), fabs(b)), fmax(fabs(c), fabs(d)));
    int n = 0;
    r[0] = r[1] = r[2] = 0.0;
    if (!(sc > 0.0)) return 0;
    if (fabs(a) <= 1e-12 * sc) {
        if (fabs(b) <= 1e-12 * sc) {
            if (fabs(c) <= 1e-12 * sc) return 0;
            r[0] = -d / c;
            return 1;
        }
        const double disc = c * c - 4.0 * b * d;
        if (disc < 0.0) return 0;
        const double q = -0.5 * (c + copysign(sqrt(disc), c));
        r[0] = q / b;
        r[1] = q != 0.0 ? d / q : r[0];
        n = 2;
    } else {
        const double B = b / a, C = c / a, D = d / a;
        const double p = C - B * B / 3.0, q = 2.0 * B * B * B / 27.0 - B * C / 3.0 + D;
        const double disc = q * q / 4.0 + p * p * p / 27.0;
        if (disc > 0.0) {
            const double sq = sqrt(disc);
            r[0] = cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq) - B / 3.0;
            n = 1;
        } else if (p == 0.0) {
            r[0] = r[1] = r[2] = -B / 3.0;
            n = 3;
        } else {
            const double m = 2.0 * sqrt(-p / 3.0);
            const double arg = fmin(1.0, fmax(-1.0, 3.0 * q / (p * m)));
            // th = acos(arg) / 3 in [0, pi / 3]; sincospi needs no argument reduction table (no local memory)
            double sn, cs;
            sincospi(acos(arg) / (3.0 * 3.141592653589793), &sn, &cs);
            r[0] = m * cs - B / 3.0;
            r[1] = m * (-0.5 * cs + 0.8660254037844386 * sn) - B / 3.0;     // cos(th - 2 pi / 3)
            r[2] = m * (-0.5 * cs - 0.8660254037844386 * sn) - B / 3.0;     // cos(th - 4 pi / 3)
            n = 3;
        }
        // two Newton steps on the original polynomial (unused entries are polished too and ignored)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
#pragma unroll
            for (int it = 0; it < 2; ++it) {
                const double x = r[j];
                const double f = ((a * x + b) * x + c) * x + d, g = (3.0 * a * x + 2.0 * b) * x + c;
                if (g != 0.0) r[j] = x - f / g;
            }
        }
    }
    // ascending (compare-swap network; unused entries stay at the end)
    if (n >= 2 && r[1] < r[0]) { const double t = r[0]; r[0] = r[1]; r[1] = t; }
    if (n == 3) {
        if (r[2] < r[1]) { const double t = r[1]; r[1] = r[2]; r[2] = t; }
        if (r[1] < r[0]) { const double t = r[0]; r[0] = r[1]; r[1] = t; }
    }
    return n;
}

__device__ __forceinline__ double det_mix(const double (&f1)[9], const double (&f2)[9], double l)
{
    double m[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) m[j] = f2[j] + l * (f1[j] - f2[j]);
    return det3(m);
}

// 7-point method: null space of the 7 x 9 system by Gauss-Jordan elimination with partial pivoting (column order; the
// matrix lives in shared memory, column-strided per lane), F1 / F2 from the two free columns, then the cubic det = 0.
// Returns the number of real roots (0: failed solve); models[j] are F = l_j F1 + (1 - l_j) F2, ascending l_j.
__device__ __forceinline__ int solve_f7(const float4 (&p)[7], double* A, double* N, int* piv, double (&F)[3][9])
{
    const int T = kSolveThreads, t = threadIdx.x;
#define AE(r, c) A[((r) * 9 + (c)) * T + t]
    double sc = 0.0;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
        const double x = p[j].x, y = p[j].y, xr = p[j].z, yr = p[j].w;
        const double row[9] = {xr * x, xr * y, xr, yr * x, yr * y, yr, x, y, 1.0};
#pragma unroll
        for (int c = 0; c < 9; ++c) { AE(j, c) = row[c]; sc = fmax(sc, fabs(row[c])); }
    }
    int row = 0, nfree = 0, fa = -1, fb = -1;
    for (int col = 0; col < 9; ++col) {
        int best = -1;
        double bv = 1e-10 * sc;
        for (int r = row; r < 7; ++r) {
            const double v = fabs(AE(r, col));
            if (v > bv) { bv = v; best = r; }
        }
        if (best < 0) {
            if (nfree == 0) fa = col; else if (nfree == 1) fb = col;
            ++nfree;
            continue;
        }
        if (best != row)
            for (int c = 0; c < 9; ++c) { const double tmp = AE(row, c); AE(row, c) = AE(best, c); AE(best, c) = tmp; }
        const double inv = 1.0 / AE(row, col);
        for (int c = 0; c < 9; ++c) AE(row, c) *= inv;
        for (int r = 0; r < 7; ++r) {
            if (r == row) continue;
            const double f = AE(r, col);
            if (f != 0.0)
                for (int c = 0; c < 9; ++c) AE(r, c) -= f * AE(row, c);
        }
        piv[row * T + t] = col;
        ++row;
    }
    if (row != 7 || nfree != 2) return 0;
    // null vectors: x_f = 1 for one free column, 0 for the other, x_piv(r) = -A[r][f]
    for (int c = 0; c < 9; ++c) { N[c * T + t] = 0.0; N[(9 + c) * T + t] = 0.0; }
    N[fa * T + t] = 1.0;
    N[(9 + fb) * T + t] = 1.0;
    for (int r = 0; r < 7; ++r) {
        const int pc = piv[r * T + t];
        N[pc * T + t] = -AE(r, fa);
        N[(9 + pc) * T + t] = -AE(r, fb);
    }
#undef AE
    double f1[9], f2[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) { f1[c] = N[c * T + t]; f2[c] = N[(9 + c) * T + t]; }
    // det(F2 + l (F1 - F2)) = a l^3 + b l^2 + c l + d from its values at 0, 1, -1, 2
    const double d0 = det_mix(f1, f2, 0.0), d1 = det_mix(f1, f2, 1.0), dm = det_mix(f1, f2, -1.0), d2 = det_mix(f1, f2, 2.0);
    const double b = 0.5 * (d1 + dm) - d0;
    const double a = (d2 - 4.0 * b - d0 - (d1 - dm)) / 6.0;
    const double c = 0.5 * (d1 - dm) - a;
    double r[3];
    const int n = cubic_roots(a, b, c, d0, r);
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int e = 0; e < 9; ++e) F[j][e] = r[j] * f1[e] + (1.0 - r[j]) * f2[e];
    return n;
}

template <int MODEL>
__global__ void __launch_bounds__(kSolveThreads) verify_solve_kernel(const VSolveItem* __restrict__ items, const VPair* __restrict__ pairs,
                                                                     const float4* __restrict__ pts, int n_samples, uint64_t seed,
                                                                     float* __restrict__ models, int32_t* __restrict__ counts)
{
    constexpr int M = MODEL == PS_GEOM_HOMOGRAPHY ? 4 : 7;
    constexpr int K = MODEL == PS_GEOM_HOMOGRAPHY ? 1 : 3;
    const VSolveItem it = items[blockIdx.x];
    const int s = it.s0 + (int)threadIdx.x;
    if (s >= n_samples) return;
    const VPair P = pairs[it.pair];
    const size_t h0 = ((size_t)it.pair * n_samples + s) * K;
    uint32_t idx[M];
    bool ok = P.n >= M && verify_sample<M>(seed, it.pair, s, (uint32_t)P.n, idx);
    float4 p[M];
#pragma unroll
    for (int j = 0; j < M; ++j) p[j] = ok ? pts[P.start + idx[j]] : make_float4(0.f, 0.f, 0.f, 0.f);
    bool valid[K];
    if constexpr (MODEL == PS_GEOM_HOMOGRAPHY) {
        double H[9];
        valid[0] = ok && solve_h4(p, H) && store_model(H, models + 9 * h0);
    } else {
        __shared__ double A[63 * kSolveThreads];
        __shared__ double N[18 * kSolveThreads];
        __shared__ int piv[7 * kSolveThreads];
        double F[3][9];
        const int n = ok ? solve_f7(p, A, N, piv, F) : 0;
#pragma unroll
        for (int j = 0; j < 3; ++j) valid[j] = j < n && store_model(F[j], models + 9 * (h0 + j));
    }
#pragma unroll
    for (int j = 0; j < K; ++j) counts[h0 + j] = valid[j] ? 0 : -1;
}

template <int MODEL>
__global__ void __launch_bounds__(kScoreThreads) verify_score_kernel(const VScoreItem* __restrict__ items, const VPair* __restrict__ pairs,
                                                                     const VXform* __restrict__ xf, const float4* __restrict__ pts,
                                                                     int n_samples, const float* __restrict__ models,
                                                                     int32_t* __restrict__ counts)
{
    constexpr int K = MODEL == PS_GEOM_HOMOGRAPHY ? 1 : 3;
    __shared__ __align__(128) float4 tile[2][kTile];
    __shared__ __align__(8) uint64_t bar[2];
    const VScoreItem it = items[blockIdx.x];
    const VPair P = pairs[it.pair];
    const float t2 = xf[it.pair].t2;
    const int s = it.s0 + (int)threadIdx.x;
    const size_t h0 = ((size_t)it.pair * n_samples + s) * K;
    float m[K][9];
    bool act[K];
    int cnt[K];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        act[j] = s < n_samples && counts[h0 + j] >= 0;
        cnt[j] = 0;
#pragma unroll
        for (int e = 0; e < 9; ++e) m[j][e] = act[j] ? models[9 * (h0 + j) + e] : 0.0f;
    }
    score_tiles<MODEL, K>(pts + P.start + it.c0, it.c1 - it.c0, m, t2, tile, bar, cnt);
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (act[j] && cnt[j]) atomicAdd(&counts[h0 + j], cnt[j]);
}

// ---- output model in pixels ----

// normalised model -> pixels (H = T_r^-1 Hn T_l, F = T_r^T Fn T_l with T = [s 0 -s cx; 0 s -s cy; 0 0 1]), then the
// output scaling of the header; all-zero when the model is zero or not finite
template <int MODEL>
__device__ __forceinline__ void to_pixels(const float (&mn)[9], const VXform& X, float* out)
{
    const double s = X.s;
    const double Tl[9] = {s, 0.0, -s * X.cxl, 0.0, s, -s * X.cyl, 0.0, 0.0, 1.0};
    double L[9];      // left factor: T_r^-1 (H) or T_r^T (F)
    if constexpr (MODEL == PS_GEOM_HOMOGRAPHY) {
        const double is = 1.0 / s;
        const double Li[9] = {is, 0.0, X.cxr, 0.0, is, X.cyr, 0.0, 0.0, 1.0};
#pragma unroll
        for (int j = 0; j < 9; ++j) L[j] = Li[j];
    } else {
        const double Lt[9] = {s, 0.0, 0.0, 0.0, s, 0.0, -s * X.cxr, -s * X.cyr, 1.0};
#pragma unroll
        for (int j = 0; j < 9; ++j) L[j] = Lt[j];
    }
    double MT[9], R[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) MT[3 * r + c] = (double)mn[3 * r] * Tl[c] + (double)mn[3 * r + 1] * Tl[3 + c] + (double)mn[3 * r + 2] * Tl[6 + c];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[3 * r + c] = L[3 * r] * MT[c] + L[3 * r + 1] * MT[3 + c] + L[3 * r + 2] * MT[6 + c];
    double nn = 0.0;
#pragma unroll
    for (int j = 0; j < 9; ++j) nn += R[j] * R[j];
    const double norm = sqrt(nn);
    double k = 0.0;
    if (norm > 0.0 && isfinite(norm)) {
        if constexpr (MODEL == PS_GEOM_HOMOGRAPHY) {
            k = fabs(R[8]) >= 1e-8 * norm ? 1.0 / R[8] : 1.0 / norm;
        } else {
            double rb = R[0];            // the first entry of largest magnitude
#pragma unroll
            for (int j = 1; j < 9; ++j) if (fabs(R[j]) > fabs(rb)) rb = R[j];
            k = (rb < 0.0 ? -1.0 : 1.0) / norm;
        }
    }
#pragma unroll
    for (int j = 0; j < 9; ++j) out[j] = (float)(R[j] * k);
}

template <int MODEL>
__global__ void verify_taps_kernel(const VXform* __restrict__ xf, const float* __restrict__ models, const int32_t* __restrict__ counts,
                                   long long n_hyp, int per_pair, int32_t* __restrict__ tap_counts, float* __restrict__ tap_models)
{
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_hyp) return;
    const int c = counts[h];
    tap_counts[h] = c;
    float mn[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) mn[e] = c >= 0 ? models[9 * h + e] : 0.0f;
    if (c >= 0) to_pixels<MODEL>(mn, xf[h / per_pair], tap_models + 9 * h);
    else
        for (int e = 0; e < 9; ++e) tap_models[9 * h + e] = 0.0f;
}

// ---- selection and refit ----

// smallest eigenvector of the symmetric 3 x 3 matrix S by cyclic Jacobi (fixed sweeps, one thread, static indices)
__device__ __forceinline__ void jacobi3_min(double (&S)[9], double (&v)[3])
{
    double V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int sweep = 0; sweep < 12; ++sweep) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int p = k == 2 ? 1 : 0, q = k == 0 ? 1 : 2;
            const double apq = S[3 * p + q];
            if (fabs(apq) < 1e-300) continue;
            const double th = (S[4 * q] - S[4 * p]) / (2.0 * apq);
            const double t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
            const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double a = S[3 * r + p], b = S[3 * r + q];
                S[3 * r + p] = c * a - s * b; S[3 * r + q] = s * a + c * b;
            }
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double a = S[3 * p + r], b = S[3 * q + r];
                S[3 * p + r] = c * a - s * b; S[3 * q + r] = s * a + c * b;
                const double va = V[3 * r + p], vb = V[3 * r + q];
                V[3 * r + p] = c * va - s * vb; V[3 * r + q] = s * va + c * vb;
            }
        }
    }
    const int m = (S[0] <= S[4] && S[0] <= S[8]) ? 0 : (S[4] <= S[8] ? 1 : 2);
#pragma unroll
    for (int r = 0; r < 3; ++r) v[r] = m == 0 ? V[3 * r] : m == 1 ? V[3 * r + 1] : V[3 * r + 2];
}

template <int MODEL>
__global__ void __launch_bounds__(kSelectThreads, 1) verify_select_kernel(const VPair* __restrict__ pairs, const VXform* __restrict__ xf,
                                                                       const float4* __restrict__ pts, int n_samples, int refine,
                                                                       const float* __restrict__ models, const int32_t* __restrict__ counts,
                                                                       float* __restrict__ out_models, int32_t* __restrict__ out_n,
                                                                       uint8_t* __restrict__ out_mask)
{
    constexpr int M = MODEL == PS_GEOM_HOMOGRAPHY ? 4 : 7;
    constexpr int K = MODEL == PS_GEOM_HOMOGRAPHY ? 1 : 3;
    constexpr int NW = kSelectThreads / 32;
    __shared__ int red_i[33];
    __shared__ int win_c[NW];
    __shared__ long long win_h[NW];
    __shared__ double Nsh[NW][45];
    __shared__ double A[81], V[81];
    __shared__ float model[9], refit[9];
    const int p = blockIdx.x;
    const VPair P = pairs[p];
    const VXform X = xf[p];
    const float4* q = pts + P.start;
    // winner: most inliers, ties to the smallest h
    const long long nh = (long long)K * n_samples, h0 = (long long)p * nh;
    int bc;
    long long bh;
    select_winner<NW>(counts + h0, nh, P.n >= M, win_c, win_h, bc, bh);
    if (bc < 0) {
        // no valid hypothesis (or too few correspondences): zero model, count, mask
        if (threadIdx.x < 9) out_models[9 * p + threadIdx.x] = 0.0f;
        if (threadIdx.x == 0) out_n[p] = 0;
        for (int i = threadIdx.x; i < P.n; i += kSelectThreads) out_mask[P.start + i] = 0;
        return;
    }
    if (threadIdx.x < 9) model[threadIdx.x] = models[9 * (h0 + bh) + threadIdx.x];
    __syncthreads();
    float mw[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) mw[e] = model[e];
    const int min_refit = MODEL == PS_GEOM_HOMOGRAPHY ? 4 : 8;
    if (refine && bc >= min_refit) {
        double r[9];
        refit_smallest<MODEL, NW>(mw, q, P.n, X.t2, Nsh, A, V, r);
        if (threadIdx.x == 0) {
            if constexpr (MODEL == PS_GEOM_FUNDAMENTAL) {
                // rank 2: F - (F v) v^T with v the right singular vector of the smallest singular value
                double S[9];
#pragma unroll
                for (int a = 0; a < 3; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) S[3 * a + b] = r[a] * r[b] + r[3 + a] * r[3 + b] + r[6 + a] * r[6 + b];
                double v[3];
                jacobi3_min(S, v);
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const double fv = r[3 * a] * v[0] + r[3 * a + 1] * v[1] + r[3 * a + 2] * v[2];
#pragma unroll
                    for (int b = 0; b < 3; ++b) r[3 * a + b] -= fv * v[b];
                }
            }
            if (!store_model(r, refit))
                for (int e = 0; e < 9; ++e) refit[e] = 0.0f;
        }
        __syncthreads();
        float mr[9];
#pragma unroll
        for (int e = 0; e < 9; ++e) mr[e] = refit[e];
        int c = 0;
        for (int i = threadIdx.x; i < P.n; i += kSelectThreads) c += inlier<MODEL>(mr, q[i], X.t2) ? 1 : 0;
        const int rc = block_sum_i(c, red_i);
        if (rc >= bc) {
#pragma unroll
            for (int e = 0; e < 9; ++e) mw[e] = mr[e];
        }
    }
    int c = 0;
    for (int i = threadIdx.x; i < P.n; i += kSelectThreads) {
        const bool in = inlier<MODEL>(mw, q[i], X.t2);
        out_mask[P.start + i] = in ? 1 : 0;
        c += in ? 1 : 0;
    }
    const int total = block_sum_i(c, red_i);
    if (threadIdx.x == 0) {
        out_n[p] = total;
        to_pixels<MODEL>(mw, X, out_models + 9 * p);
    }
}

template <int MODEL>
int launch_verify(const VPair* d_pairs, const VXform* d_xf, const float4* d_pts, const VSolveItem* d_solve, int n_solve,
                  const VScoreItem* d_score, int n_score, int n_pairs, const ps_verify_params& prm, float* hyp_models,
                  int32_t* hyp_counts, float* d_models, int32_t* d_n, uint8_t* d_mask, const ps_verify_taps* taps, cudaStream_t st)
{
    int launches = 0;
    verify_solve_kernel<MODEL><<<n_solve, kSolveThreads, 0, st>>>(d_solve, d_pairs, d_pts, prm.n_samples, prm.seed, hyp_models, hyp_counts);
    ++launches;
    if (n_score > 0) {
        verify_score_kernel<MODEL><<<n_score, kScoreThreads, 0, st>>>(d_score, d_pairs, d_xf, d_pts, prm.n_samples, hyp_models, hyp_counts);
        ++launches;
    }
    verify_select_kernel<MODEL><<<n_pairs, kSelectThreads, 0, st>>>(d_pairs, d_xf, d_pts, prm.n_samples, prm.refine, hyp_models,
                                                                    hyp_counts, d_models, d_n, d_mask);
    ++launches;
    if (taps) {
        constexpr int K = MODEL == PS_GEOM_HOMOGRAPHY ? 1 : 3;
        const long long n_hyp = (long long)n_pairs * K * prm.n_samples;
        verify_taps_kernel<MODEL><<<(unsigned)((n_hyp + 255) / 256), 256, 0, st>>>(d_xf, hyp_models, hyp_counts, n_hyp, K * prm.n_samples,
                                                                                   taps->d_counts, taps->d_models);
        ++launches;
    }
    return launches;
}

} // namespace

int run_match_correspondences(const ps_feature* const* feat, const int32_t* const* rev, const int32_t* n_desc, const int32_t* pairs,
                              int n_pairs, const int32_t* match, float* corr, int32_t* src, int32_t* n_corr, cudaStream_t st,
                              const char** err)
{
    *err = nullptr;
    std::vector<CorrPair> hp(n_pairs);
    long long row = 0;
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        hp[p] = {feat[l], rev[l], feat[r], rev[r], row, n_desc[l], n_desc[r]};
        row += n_desc[l];
    }
    Workspace ws(st, "cudaMallocFromPoolAsync failed (correspondences)", "correspondences: upload failed");
    const size_t o_pairs = ws.put(hp.data(), hp.size() * sizeof(CorrPair), 16);
    const size_t o_counts = ws.put(nullptr, (size_t)n_pairs * sizeof(int32_t), 16);
    if (!ws.alloc(err)) return -1;
    int32_t* d_counts = ws.at<int32_t>(o_counts);
    corr_gather_kernel<<<n_pairs, kGatherThreads, 0, st>>>(ws.at<const CorrPair>(o_pairs), match, reinterpret_cast<float4*>(corr), src, d_counts);
    if (cudaMemcpyAsync(n_corr, d_counts, (size_t)n_pairs * sizeof(int32_t), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return ws.fail("correspondences: count download failed", err);
    return 1;
}

int run_verify_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_verify_params& prm,
                     float* d_models, int32_t* d_n, uint8_t* d_mask, const ps_verify_taps* taps, cudaStream_t st, const char** err)
{
    *err = nullptr;
    const int K = prm.model == PS_GEOM_HOMOGRAPHY ? 1 : 3, M = prm.model == PS_GEOM_HOMOGRAPHY ? 4 : 7;
    const int ns = prm.n_samples;
    long long total_rows = 0;
    double work = 0.0;
    for (int p = 0; p < n_pairs; ++p) {
        total_rows = std::max(total_rows, (long long)corr_start[p] + n_corr[p]);
        if (n_corr[p] >= M) work += (double)((ns + kScoreThreads - 1) / kScoreThreads) * n_corr[p];
    }
    // correspondences per score item: about 16 items per SM over the whole call, at least two tiles
    const double per = std::ceil(work / (16.0 * sm_count()));
    const int chunk = (int)std::min<double>(1 << 30, std::max<double>(2 * kTile, std::ceil(per / kTile) * kTile));
    std::vector<VPair> vp(n_pairs);
    std::vector<VSolveItem> solve;
    std::vector<VScoreItem> score;
    for (int p = 0; p < n_pairs; ++p) {
        vp[p] = {corr_start[p], n_corr[p], 0};
        for (int s0 = 0; s0 < ns; s0 += kSolveThreads) solve.push_back({p, s0});
        if (n_corr[p] < M) continue;
        for (int c0 = 0; c0 < n_corr[p]; c0 += chunk)
            for (int s0 = 0; s0 < ns; s0 += kScoreThreads) score.push_back({p, s0, c0, (int)std::min<long long>((long long)c0 + chunk, n_corr[p])});
    }
    if (solve.size() > 0x7fffffffu || score.size() > 0x7fffffffu) { *err = "ps_verify_batch: too many work items"; return -1; }
    const size_t n_hyp = (size_t)n_pairs * K * ns;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (verify workspace)", "verify: plan upload failed");
    const size_t o_pairs = ws.put(vp.data(), vp.size() * sizeof(VPair)), o_solve = ws.put(solve.data(), solve.size() * sizeof(VSolveItem));
    const size_t o_score = ws.put(score.data(), score.size() * sizeof(VScoreItem));
    const size_t o_xf = ws.take((size_t)n_pairs * sizeof(VXform)), o_pts = ws.take((size_t)total_rows * sizeof(float4));
    const size_t o_models = ws.take(n_hyp * 9 * sizeof(float)), o_counts = ws.take(n_hyp * sizeof(int32_t));
    if (!ws.alloc(err)) return -1;
    const VPair* d_pairs = ws.at<const VPair>(o_pairs);
    VXform* d_xf = ws.at<VXform>(o_xf);
    float4* d_pts = ws.at<float4>(o_pts);
    verify_normalize_kernel<<<n_pairs, kNormThreads, 0, st>>>(d_pairs, reinterpret_cast<const float4*>(corr), d_pts, d_xf, (double)prm.threshold);
    int launches = 1;
    const VSolveItem* d_solve = ws.at<const VSolveItem>(o_solve);
    const VScoreItem* d_score = ws.at<const VScoreItem>(o_score);
    float* hyp_models = ws.at<float>(o_models);
    int32_t* hyp_counts = ws.at<int32_t>(o_counts);
    if (prm.model == PS_GEOM_HOMOGRAPHY)
        launches += launch_verify<PS_GEOM_HOMOGRAPHY>(d_pairs, d_xf, d_pts, d_solve, (int)solve.size(), d_score, (int)score.size(), n_pairs, prm,
                                                      hyp_models, hyp_counts, d_models, d_n, d_mask, taps, st);
    else
        launches += launch_verify<PS_GEOM_FUNDAMENTAL>(d_pairs, d_xf, d_pts, d_solve, (int)solve.size(), d_score, (int)score.size(), n_pairs, prm,
                                                       hyp_models, hyp_counts, d_models, d_n, d_mask, taps, st);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

} // namespace psb
