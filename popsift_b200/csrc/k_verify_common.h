// Device pieces shared by ps_verify_batch (k_verify.cu) and ps_relative_pose_batch (k_pose.cu): the pair record, the
// fixed-order block sums, the inlier tests, the tiled scoring loop, the selection rule and the refit's normal matrix with
// its smallest eigenvector.  Both files must run them bit for bit alike, so there is one definition.
#pragma once
#include "k_match_common.h"
#include "popsift_b200.h"

#include <stdint.h>

namespace psb {

namespace {

struct VPair { long long start; int n, pad; };

constexpr int kScoreThreads = 128;
constexpr int kSelectThreads = 128;
constexpr int kTile = 1024;          // points per shared-memory tile (16 KB)

__device__ __forceinline__ double block_sum_d(double v, double* red)
{
    // fixed-order tree: shuffle-down within each warp, then warp 0's partials summed in warp order by thread 0
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
        red[32] = t;
    }
    __syncthreads();
    return red[32];
}

__device__ __forceinline__ int block_sum_i(int v, int* red)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
        red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// ---- the inlier tests (scoring, refit and mask share them bit for bit) ----

__device__ __forceinline__ bool inlier_h(const float (&h)[9], float4 q, float t2)
{
    const float u = fmaf(h[0], q.x, fmaf(h[1], q.y, h[2]));
    const float v = fmaf(h[3], q.x, fmaf(h[4], q.y, h[5]));
    const float w = fmaf(h[6], q.x, fmaf(h[7], q.y, h[8]));
    const float du = fmaf(-q.z, w, u), dv = fmaf(-q.w, w, v);
    return fmaf(du, du, dv * dv) < t2 * (w * w);
}

__device__ __forceinline__ bool inlier_f(const float (&f)[9], float4 q, float t2)
{
    const float a0 = fmaf(f[0], q.x, fmaf(f[1], q.y, f[2]));
    const float a1 = fmaf(f[3], q.x, fmaf(f[4], q.y, f[5]));
    const float a2 = fmaf(f[6], q.x, fmaf(f[7], q.y, f[8]));
    const float b0 = fmaf(f[0], q.z, fmaf(f[3], q.w, f[6]));
    const float b1 = fmaf(f[1], q.z, fmaf(f[4], q.w, f[7]));
    const float e = fmaf(q.z, a0, fmaf(q.w, a1, a2));
    return e * e < t2 * fmaf(a0, a0, fmaf(a1, a1, fmaf(b0, b0, b1 * b1)));
}

template <int MODEL>
__device__ __forceinline__ bool inlier(const float (&m)[9], float4 q, float t2)
{
    if constexpr (MODEL == PS_GEOM_HOMOGRAPHY) return inlier_h(m, q, t2);
    else return inlier_f(m, q, t2);
}

__device__ __forceinline__ void bulk_load(void* dst, const void* src, unsigned bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(s32(dst)), "l"(src), "r"(bytes), "r"(s32(bar)) : "memory");
}

// The scoring loop of one work item: the n points at src stream through shared memory in tiles (cp.async.bulk +
// mbarrier, two buffers) read as broadcast LDS.128; each lane adds its K models' inlier counts to cnt.  Called by every
// thread of the CTA.
template <int MODEL, int K>
__device__ __forceinline__ void score_tiles(const float4* src, int n, const float (&m)[K][9], float t2, float4 (&tile)[2][kTile],
                                            uint64_t (&bar)[2], int (&cnt)[K])
{
    const int ntiles = (n + kTile - 1) / kTile;
    if (threadIdx.x == 0) {
        mb_init(&bar[0], 1);
        mb_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)min(n, kTile) * 16u;
        mb_expect(&bar[0], bytes);
        bulk_load(tile[0], src, bytes, &bar[0]);
    }
    __syncthreads();
    for (int t = 0; t < ntiles; ++t) {
        const int buf = t & 1;
        if (threadIdx.x == 0 && t + 1 < ntiles) {
            // the other buffer was last read in iteration t - 1, which ended with a barrier
            const unsigned bytes = (unsigned)min(n - (t + 1) * kTile, kTile) * 16u;
            mb_expect(&bar[buf ^ 1], bytes);
            bulk_load(tile[buf ^ 1], src + (size_t)(t + 1) * kTile, bytes, &bar[buf ^ 1]);
        }
        mb_wait(&bar[buf], (unsigned)(t >> 1) & 1u);
        const int nt = min(n - t * kTile, kTile);
        const float4* tp = tile[buf];
#pragma unroll 4
        for (int i = 0; i < nt; ++i) {
            const float4 q = tp[i];        // every lane reads the same point: one broadcast LDS.128
#pragma unroll
            for (int j = 0; j < K; ++j) cnt[j] += inlier<MODEL>(m[j], q, t2) ? 1 : 0;
        }
        __syncthreads();
    }
}

// The winner among counts[0 .. nh): most inliers, ties to the smallest h; (-1, -1) when none is valid or !enabled.  Every
// thread of the CTA (kSelectThreads) gets the result.
template <int NW>
__device__ __forceinline__ void select_winner(const int32_t* counts, long long nh, bool enabled, int* win_c, long long* win_h,
                                              int& bc, long long& bh)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    bc = -1;
    bh = -1;
    if (enabled)
        for (long long h = threadIdx.x; h < nh; h += kSelectThreads) {
            const int c = counts[h];
            if (c > bc) { bc = c; bh = h; }          // h ascends within a thread: strict > keeps the smallest
        }
    for (int o = 16; o > 0; o >>= 1) {
        const int oc = __shfl_down_sync(0xffffffffu, bc, o);
        const long long oh = __shfl_down_sync(0xffffffffu, bh, o);
        if (oc > bc || (oc == bc && oc >= 0 && oh < bh)) { bc = oc; bh = oh; }
    }
    if (lane == 0) { win_c[warp] = bc; win_h[warp] = bh; }
    __syncthreads();
    bc = win_c[0]; bh = win_h[0];
    for (int w = 1; w < NW; ++w)
        if (win_c[w] > bc || (win_c[w] == bc && bc >= 0 && win_h[w] < bh)) { bc = win_c[w]; bh = win_h[w]; }
}

// ---- refit ----

// smallest eigenvector of the symmetric 9 x 9 matrix A (shared memory, row-major) by cyclic Jacobi; run by one warp, lane k
// applies each rotation to row / column k.  V (shared) receives the eigenvectors as columns; returns the index of the
// smallest eigenvalue.
__device__ __forceinline__ int jacobi9(double* A, double* V)
{
    const int lane = threadIdx.x & 31;
    for (int k = lane; k < 81; k += 32) V[k] = (k % 10 == 0) ? 1.0 : 0.0;
    __syncwarp();
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0, dia = 0.0;
        for (int p = 0; p < 9; ++p) {
            dia += A[p * 10] * A[p * 10];
            for (int q = p + 1; q < 9; ++q) off += A[p * 9 + q] * A[p * 9 + q];
        }
        if (!(off > 1e-30 * dia)) break;
        for (int p = 0; p < 8; ++p)
            for (int q = p + 1; q < 9; ++q) {
                const double apq = A[p * 9 + q];
                if (fabs(apq) < 1e-300) continue;
                const double th = (A[q * 10] - A[p * 10]) / (2.0 * apq);
                const double t = fabs(th) > 1e150 ? 0.5 / th : (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                __syncwarp();
                if (lane < 9) {
                    const double akp = A[lane * 9 + p], akq = A[lane * 9 + q];
                    A[lane * 9 + p] = c * akp - s * akq;
                    A[lane * 9 + q] = s * akp + c * akq;
                }
                __syncwarp();
                if (lane < 9) {
                    const double apk = A[p * 9 + lane], aqk = A[q * 9 + lane];
                    A[p * 9 + lane] = c * apk - s * aqk;
                    A[q * 9 + lane] = s * apk + c * aqk;
                    const double vkp = V[lane * 9 + p], vkq = V[lane * 9 + q];
                    V[lane * 9 + p] = c * vkp - s * vkq;
                    V[lane * 9 + q] = s * vkp + c * vkq;
                }
                __syncwarp();
            }
    }
    int best = 0;
    for (int p = 1; p < 9; ++p)
        if (A[p * 10] < A[best * 10]) best = p;
    return best;
}

template <int MODEL>
__device__ __forceinline__ void refit_rows(float4 q, double (&N)[45])
{
    const double x = q.x, y = q.y, xr = q.z, yr = q.w;
    if constexpr (MODEL == PS_GEOM_HOMOGRAPHY) {
        const double r1[9] = {x, y, 1.0, 0.0, 0.0, 0.0, -xr * x, -xr * y, -xr};
        const double r2[9] = {0.0, 0.0, 0.0, x, y, 1.0, -yr * x, -yr * y, -yr};
        int e = 0;
#pragma unroll
        for (int a = 0; a < 9; ++a)
#pragma unroll
            for (int b = a; b < 9; ++b, ++e) N[e] += r1[a] * r1[b] + r2[a] * r2[b];
    } else {
        const double r[9] = {xr * x, xr * y, xr, yr * x, yr * y, yr, x, y, 1.0};
        int e = 0;
#pragma unroll
        for (int a = 0; a < 9; ++a)
#pragma unroll
            for (int b = a; b < 9; ++b, ++e) N[e] += r[a] * r[b];
    }
}

// The refit's linear step: the 9 x 9 normal matrix of the rows that pass the inlier test under mw (double, per-thread
// partials, then warp sums and the warps in order), and its smallest eigenvector by jacobi9.  Called by every thread of
// the CTA (kSelectThreads); lane 0 of warp 0 gets the eigenvector in r.
template <int MODEL, int NW>
__device__ __forceinline__ void refit_smallest(const float (&mw)[9], const float4* q, int n, float t2, double (*Nsh)[45], double* A,
                                               double* V, double (&r)[9])
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double N[45];
#pragma unroll
    for (int e = 0; e < 45; ++e) N[e] = 0.0;
    for (int i = threadIdx.x; i < n; i += kSelectThreads) {
        const float4 v = q[i];
        if (inlier<MODEL>(mw, v, t2)) refit_rows<MODEL>(v, N);
    }
#pragma unroll
    for (int e = 0; e < 45; ++e) {
        double v = N[e];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) Nsh[warp][e] = v;
    }
    __syncthreads();
    if (threadIdx.x < 45) {
        double v = 0.0;
        for (int w = 0; w < NW; ++w) v += Nsh[w][threadIdx.x];
        int a = 0, e = threadIdx.x;
        while (e >= 9 - a) { e -= 9 - a; ++a; }
        const int b = a + e;
        A[a * 9 + b] = v;
        A[b * 9 + a] = v;
    }
    __syncthreads();
    if (warp == 0) {
        const int m = jacobi9(A, V);
        if (lane == 0)
#pragma unroll
            for (int e = 0; e < 9; ++e) r[e] = V[e * 9 + m];
    }
}

} // namespace

} // namespace psb
