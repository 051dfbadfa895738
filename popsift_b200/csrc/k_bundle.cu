// Bundle adjustment, hand-written for sm_90a: ps_bundle_adjust (contract in include/popsift_b200_bundle.h).  The
// per-observation math is in k_bundle.h (built on k_triangulate.h), the scan and the radix sort in k_scan.h.
//
// One workspace (workspace.h), all launches on one stream.  Setup (once per call):
//   ba_check_kernel     one thread per member: the checks of ps_triangulate_tracks' ray pass (a flag read back before any
//                       output is written), each member's set and pixel
//   ba_flag_kernel      one thread per track: the used flag of each member; an exclusive scan numbers the used observations
//                       in member order, so each track's used observations are contiguous
//   ba_compact_kernel   one thread per track: each used observation's member, track and set; per-set counts (integer
//                       atomics), scanned into each set's first entry of the camera-major list
//   radix sort          the used observations stably by set (k_scan.h): the camera-major list
// Per LM iteration (H, g at the current parameters; lambda a kernel argument):
//   ba_linearize_kernel    one thread per used observation: sqrt(w) e, sqrt(w) Jc (2 x 6), sqrt(w) Jp (2 x 3), stored
//   ba_cam_grad_kernel     one CTA per set: U_i = sum Jc^T Jc, g_i = sum Jc^T e (after each accepted step only)
//   ba_point_kernel        one thread per track: V_j, g_j, (V_j + lambda D_j)^-1, t_j = (..)^-1 g_j
//   ba_cam_precond_kernel  one CTA per set: the 6 x 6 diagonal block of S by Cholesky, the reduced right-hand side, CG's
//                          first residual
//   ba_cg_init_kernel, then per CG iteration ba_point_matvec_kernel (track-major half of S p), ba_cam_matvec_kernel
//                          (camera-major half), ba_cg_update_kernel (one CTA: the dot products, the vector updates and
//                          the stopping test).  Convergence is a device flag; every CG kernel returns at once when it is
//                          set, so the host queues cg_max_iters iterations without waiting.
//   ba_cam_update_kernel, ba_point_back_kernel, ba_cost_kernel, ba_reduce_kernel: the candidate poses and points, the
//                          predicted decrease and the new cost, read back in one small copy.
// CTA sums are xor butterflies within warps and the warps in index order; a thread's share is summed in index order;
// no floating-point atomics, so two identical calls give identical bytes.
#include "k_bundle.h"
#include "k_scan.h"
#include "ps_internal.h"
#include "popsift_b200_bundle.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kT = 256;                 // threads of the per-member / per-track / per-observation kernels
constexpr int kCamT = 128;              // threads of a per-set CTA
constexpr int kCgT = 256;               // threads of the single-CTA CG kernels
constexpr unsigned kFull = 0xffffffffu;

// one set's pose and intrinsics, and its role: active = free with a used observation; held = the index (3 + axis) of a
// held translation component, or -1
struct BaCam {
    TriCam K;
    int32_t active, held;
};

// one used observation's weighted residual and Jacobians
struct BaObs {
    double Jc[12];
    double Jp[6];
    double e[2];
};

// one set's linear system and CG vectors
struct BaCamSys {
    double U[36];       // sum Jc^T Jc (undamped)
    double g[6];
    double L[36];       // Cholesky factor of the preconditioner block
    double x[6], r[6], z[6], p[6], q[6];
    double pq, rz, rr, gd;
};

// one track's point block
struct BaPoint {
    double V[6];        // sum Jp^T Jp (00 01 02 11 12 22)
    double g[3];
    double Vi[6];       // (V + lambda D)^-1, zero when singular
    double tv[3];       // Vi g
    double y[3];        // Vi sum Jp^T Jc p (CG)
};

struct BaStat {
    int32_t bad, n_obs, n_points, pad_;
};

// the CG state of one LM iteration
struct BaCg {
    double rz, rr0, tol2;
    int32_t done, iters;
};

// what the host reads back per LM iteration
struct BaStep {
    double cost, pred;
    int32_t cg_iters, pad_;
};

struct BaArgs {
    const int32_t* start;
    const int32_t* upos;        // M + 1: exclusive scan of the used flags
    const int32_t* umem;        // U: member of used observation u
    const int32_t* utrack;
    const int32_t* uset;
    const int32_t* clist;       // U: used observations by set
    const int32_t* cstart;      // n_sets + 1
    const float2* mxy;          // M: pixels
    BaObs* obs;
    BaPoint* pts;
    BaCamSys* sys;
    BaCg* cg;
    int n_tracks, n_sets, loss;
    double s2;
};

__device__ __forceinline__ int ba_set_of(const int32_t* __restrict__ off, int n_sets, int g)
{
    int lo = 0, hi = n_sets - 1;    // the last set with off[s] <= g (an empty set shares its offset with the next)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(off + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- setup

__global__ void __launch_bounds__(kT) ba_check_kernel(const int32_t* __restrict__ start, int n_tracks, const int32_t* __restrict__ members,
                                                      int n_members, const int32_t* __restrict__ off, int n_sets,
                                                      const ps_feature* const* __restrict__ feat, int32_t* __restrict__ mset,
                                                      float2* __restrict__ mxy, int* __restrict__ bad)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_tracks) {
        const int s = start[i];
        if ((i == 0 && s != 0) || (i == n_tracks && s != n_members) || (i < n_tracks && start[i + 1] < s)) *bad = 1;
    }
    if (i >= n_members) return;
    const int g = members[i];
    if (g < 0 || g >= off[n_sets]) { *bad = 1; return; }
    const int set = ba_set_of(off, n_sets, g);
    const ps_feature& F = feat[set][g - off[set]];
    mset[i] = set;
    mxy[i] = make_float2(F.xpos, F.ypos);
}

__global__ void __launch_bounds__(kT) ba_flag_kernel(const int32_t* __restrict__ start, int n_tracks, int n_members,
                                                     const ps_track_point* __restrict__ points, const uint8_t* __restrict__ mask,
                                                     int32_t* __restrict__ flag)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) flag[n_members] = 0;
    if (t >= n_tracks) return;
    const bool ok = points[t].status == PS_TRI_OK;
    for (int k = start[t]; k < start[t + 1]; ++k) flag[k] = ok && mask[k] != 0 ? 1 : 0;
}

__global__ void __launch_bounds__(kT) ba_compact_kernel(const BaArgs A, const int32_t* __restrict__ mset, const ps_track_point* __restrict__ points,
                                                        int32_t* __restrict__ umem, int32_t* __restrict__ utrack, int32_t* __restrict__ uset,
                                                        int32_t* __restrict__ ccount, double* __restrict__ X, BaStat* __restrict__ stat)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool has = false;
    if (t < A.n_tracks) {
        for (int k = A.start[t]; k < A.start[t + 1]; ++k) {
            const int u = A.upos[k];
            if (A.upos[k + 1] == u) continue;
            umem[u] = k;
            utrack[u] = (int)t;
            uset[u] = mset[k];
            atomicAdd(ccount + mset[k], 1);
            has = true;
        }
        for (int c = 0; c < 3; ++c) X[3 * t + c] = points[t].X[c];
    }
    const unsigned n = __reduce_add_sync(kFull, has ? 1u : 0u);
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&stat->n_points, (int)n);
}

__global__ void __launch_bounds__(kT) ba_iota_kernel(int32_t* __restrict__ v, int n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = (int)i;
}

struct SetKey {
    const int32_t* uset;
    __device__ __forceinline__ int operator()(int u) const { return uset[u]; }
};

// ---- per LM iteration

__global__ void __launch_bounds__(kT) ba_linearize_kernel(const BaArgs A, const BaCam* __restrict__ cams, const double* __restrict__ X, int n_obs)
{
    const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_obs) return;
    const BaCam& C = cams[A.uset[u]];
    const float2 xy = A.mxy[A.umem[u]];
    const double* Xp = X + 3 * A.utrack[u];
    BaObs o;
    if (!ba_jacobian(C.K, Xp, xy.x, xy.y, o.e, o.Jc, o.Jp)) {
        for (int k = 0; k < 12; ++k) o.Jc[k] = 0.0;
        for (int k = 0; k < 6; ++k) o.Jp[k] = 0.0;
        o.e[0] = o.e[1] = 0.0;
    } else {
        double rho, w;
        ba_loss(A.loss, (o.e[0] * o.e[0] + o.e[1] * o.e[1]) / A.s2, rho, w);
        const double sw = sqrt(w);
        for (int k = 0; k < 12; ++k) o.Jc[k] *= sw;
        for (int k = 0; k < 6; ++k) o.Jp[k] *= sw;
        o.e[0] *= sw;
        o.e[1] *= sw;
        if (!C.active)
            for (int k = 0; k < 12; ++k) o.Jc[k] = 0.0;
        if (C.held >= 0) o.Jc[C.held] = o.Jc[6 + C.held] = 0.0;
    }
    A.obs[u] = o;
}

__global__ void __launch_bounds__(kCamT) ba_cam_grad_kernel(const BaArgs A)
{
    const int i = blockIdx.x;
    const int c0 = A.cstart[i], c1 = A.cstart[i + 1];
    double v[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) v[k] = 0.0;
    for (int j = c0 + threadIdx.x; j < c1; j += kCamT) {
        const BaObs& o = A.obs[A.clist[j]];
        int n = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int b = a; b < 6; ++b) v[n++] += o.Jc[a] * o.Jc[b] + o.Jc[6 + a] * o.Jc[6 + b];
#pragma unroll
        for (int a = 0; a < 6; ++a) v[21 + a] += o.Jc[a] * o.e[0] + o.Jc[6 + a] * o.e[1];
    }
    cta_sum<27, kCamT>(v);
    if (threadIdx.x == 0) {
        BaCamSys& S = A.sys[i];
        int n = 0;
        for (int a = 0; a < 6; ++a)
            for (int b = a; b < 6; ++b) { S.U[6 * a + b] = v[n]; S.U[6 * b + a] = v[n]; ++n; }
        for (int a = 0; a < 6; ++a) S.g[a] = v[21 + a];
    }
}

__global__ void __launch_bounds__(kT) ba_point_kernel(const BaArgs A, double lambda)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.n_tracks) return;
    const int u0 = A.upos[A.start[t]], u1 = A.upos[A.start[t + 1]];
    if (u0 == u1) return;
    double V[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    for (int u = u0; u < u1; ++u) {
        const BaObs& o = A.obs[u];
        const double* J = o.Jp;
        V[0] += J[0] * J[0] + J[3] * J[3];
        V[1] += J[0] * J[1] + J[3] * J[4];
        V[2] += J[0] * J[2] + J[3] * J[5];
        V[3] += J[1] * J[1] + J[4] * J[4];
        V[4] += J[1] * J[2] + J[4] * J[5];
        V[5] += J[2] * J[2] + J[5] * J[5];
        for (int c = 0; c < 3; ++c) g[c] += J[c] * o.e[0] + J[3 + c] * o.e[1];
    }
    BaPoint& P = A.pts[t];
    double Vd[6] = {ba_damp(V[0], lambda), V[1], V[2], ba_damp(V[3], lambda), V[4], ba_damp(V[5], lambda)}, Vi[6], tv[3];
    if (!ba_inv3(Vd, Vi))
        for (int k = 0; k < 6; ++k) Vi[k] = 0.0;
    ba_sym3_mul(Vi, g, tv);
    for (int k = 0; k < 6; ++k) { P.V[k] = V[k]; P.Vi[k] = Vi[k]; }
    for (int k = 0; k < 3; ++k) { P.g[k] = g[k]; P.tv[k] = tv[k]; }
}

// Q = Jp Vi Jp^T (2 x 2: 00 01 11) of one observation
__device__ __forceinline__ void ba_q(const double* Jp, const double* Vi, double* Q)
{
    double a[3], b[3];
    ba_sym3_mul(Vi, Jp, a);
    ba_sym3_mul(Vi, Jp + 3, b);
    Q[0] = Jp[0] * a[0] + Jp[1] * a[1] + Jp[2] * a[2];
    Q[1] = Jp[3] * a[0] + Jp[4] * a[1] + Jp[5] * a[2];
    Q[2] = Jp[3] * b[0] + Jp[4] * b[1] + Jp[5] * b[2];
}

__global__ void __launch_bounds__(kCamT) ba_cam_precond_kernel(const BaArgs A, const BaCam* __restrict__ cams, double lambda)
{
    const int i = blockIdx.x;
    BaCamSys& S = A.sys[i];
    const int c0 = A.cstart[i], c1 = A.cstart[i + 1];
    const bool active = cams[i].active != 0;
    double v[27];
#pragma unroll
    for (int k = 0; k < 27; ++k) v[k] = 0.0;
    if (active) {
        for (int j = c0 + threadIdx.x; j < c1; j += kCamT) {
            const int u = A.clist[j];
            const BaObs& o = A.obs[u];
            const BaPoint& P = A.pts[A.utrack[u]];
            double Q[3];
            ba_q(o.Jp, P.Vi, Q);
            double G0[6], G1[6];
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                G0[a] = Q[0] * o.Jc[a] + Q[1] * o.Jc[6 + a];
                G1[a] = Q[1] * o.Jc[a] + Q[2] * o.Jc[6 + a];
            }
            int n = 0;
#pragma unroll
            for (int a = 0; a < 6; ++a)
#pragma unroll
                for (int b = a; b < 6; ++b) v[n++] += o.Jc[a] * G0[b] + o.Jc[6 + a] * G1[b];
            const double s0 = o.Jp[0] * P.tv[0] + o.Jp[1] * P.tv[1] + o.Jp[2] * P.tv[2];
            const double s1 = o.Jp[3] * P.tv[0] + o.Jp[4] * P.tv[1] + o.Jp[5] * P.tv[2];
#pragma unroll
            for (int a = 0; a < 6; ++a) v[21 + a] += o.Jc[a] * s0 + o.Jc[6 + a] * s1;
        }
    }
    cta_sum<27, kCamT>(v);
    if (threadIdx.x != 0) return;
    double B[36], b[6];
    if (active) {
        int n = 0;
        for (int a = 0; a < 6; ++a)
            for (int c = a; c < 6; ++c) {
                const double u = a == c ? ba_damp(S.U[6 * a + a], lambda) : S.U[6 * a + c];
                B[6 * a + c] = B[6 * c + a] = u - v[n++];
            }
        for (int a = 0; a < 6; ++a) b[a] = -S.g[a] + v[21 + a];
        const int h = cams[i].held;
        if (h >= 0) {
            for (int a = 0; a < 6; ++a) B[6 * a + h] = B[6 * h + a] = 0.0;
            B[6 * h + h] = 1.0;
            b[h] = 0.0;
        }
        if (!ba_chol6(B, S.L))
            for (int k = 0; k < 36; ++k) S.L[k] = k % 7 == 0 ? 1.0 : 0.0;
    } else {
        for (int k = 0; k < 36; ++k) S.L[k] = k % 7 == 0 ? 1.0 : 0.0;
        for (int a = 0; a < 6; ++a) b[a] = 0.0;
    }
    double z[6];
    ba_chol6_solve(S.L, b, z);
    double rz = 0.0, rr = 0.0;
    for (int a = 0; a < 6; ++a) {
        S.x[a] = 0.0;
        S.r[a] = b[a];
        S.z[a] = z[a];
        S.p[a] = z[a];
        rz += b[a] * z[a];
        rr += b[a] * b[a];
    }
    S.rz = rz;
    S.rr = rr;
}

__global__ void __launch_bounds__(kCgT) ba_cg_init_kernel(const BaArgs A, double tol2)
{
    double v[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < A.n_sets; i += kCgT) {
        v[0] += A.sys[i].rz;
        v[1] += A.sys[i].rr;
    }
    cta_sum<2, kCgT>(v);
    if (threadIdx.x == 0) {
        BaCg& G = *A.cg;
        G.rz = v[0];
        G.rr0 = v[1];
        G.tol2 = tol2;
        G.iters = 0;
        G.done = !(v[1] > 0.0) || !isfinite(v[0]) || !isfinite(v[1]);
    }
}

// the track-major half of S p: y_j = Vi_j sum Jp^T (Jc p_set)
__global__ void __launch_bounds__(kT) ba_point_matvec_kernel(const BaArgs A)
{
    if (A.cg->done) return;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.n_tracks) return;
    const int u0 = A.upos[A.start[t]], u1 = A.upos[A.start[t + 1]];
    if (u0 == u1) return;
    double s[3] = {0.0, 0.0, 0.0};
    for (int u = u0; u < u1; ++u) {
        const BaObs& o = A.obs[u];
        const double* p = A.sys[A.uset[u]].p;
        double c0 = 0.0, c1 = 0.0;
#pragma unroll
        for (int a = 0; a < 6; ++a) { c0 += o.Jc[a] * p[a]; c1 += o.Jc[6 + a] * p[a]; }
        for (int c = 0; c < 3; ++c) s[c] += o.Jp[c] * c0 + o.Jp[3 + c] * c1;
    }
    BaPoint& P = A.pts[t];
    ba_sym3_mul(P.Vi, s, P.y);
}

// the camera-major half: q_i = (U_i + lambda D_i) p_i - sum Jc^T (Jp y_j); pq_i = p_i.q_i
__global__ void __launch_bounds__(kCamT) ba_cam_matvec_kernel(const BaArgs A, const BaCam* __restrict__ cams, double lambda)
{
    if (A.cg->done) return;
    const int i = blockIdx.x;
    BaCamSys& S = A.sys[i];
    const bool active = cams[i].active != 0;
    double v[6] = {0, 0, 0, 0, 0, 0};
    if (active) {
        const int c0 = A.cstart[i], c1 = A.cstart[i + 1];
        for (int j = c0 + threadIdx.x; j < c1; j += kCamT) {
            const int u = A.clist[j];
            const BaObs& o = A.obs[u];
            const double* y = A.pts[A.utrack[u]].y;
            const double s0 = o.Jp[0] * y[0] + o.Jp[1] * y[1] + o.Jp[2] * y[2];
            const double s1 = o.Jp[3] * y[0] + o.Jp[4] * y[1] + o.Jp[5] * y[2];
#pragma unroll
            for (int a = 0; a < 6; ++a) v[a] += o.Jc[a] * s0 + o.Jc[6 + a] * s1;
        }
    }
    cta_sum<6, kCamT>(v);
    if (threadIdx.x != 0) return;
    double pq = 0.0;
    for (int a = 0; a < 6; ++a) {
        double q = 0.0;
        if (active && a != cams[i].held) {
            for (int b = 0; b < 6; ++b) q += (a == b ? ba_damp(S.U[6 * a + a], lambda) : S.U[6 * a + b]) * S.p[b];
            q -= v[a];
        }
        S.q[a] = q;
        pq += S.p[a] * q;
    }
    S.pq = pq;
}

__global__ void __launch_bounds__(kCgT) ba_cg_update_kernel(const BaArgs A, int max_iters)
{
    BaCg& G = *A.cg;
    if (G.done) return;
    double v[1] = {0.0};
    for (int i = threadIdx.x; i < A.n_sets; i += kCgT) v[0] += A.sys[i].pq;
    cta_sum<1, kCgT>(v);
    __shared__ double alpha_s;
    if (threadIdx.x == 0) alpha_s = v[0] > 0.0 && isfinite(v[0]) ? G.rz / v[0] : 0.0;
    __syncthreads();
    const double alpha = alpha_s;
    if (alpha == 0.0) {
        if (threadIdx.x == 0) G.done = 1;
        return;
    }
    double w[1] = {0.0};
    for (int i = threadIdx.x; i < A.n_sets; i += kCgT) {
        BaCamSys& S = A.sys[i];
        for (int a = 0; a < 6; ++a) {
            S.x[a] += alpha * S.p[a];
            S.r[a] -= alpha * S.q[a];
            w[0] += S.r[a] * S.r[a];
        }
    }
    cta_sum<1, kCgT>(w);
    __shared__ int stop_s;
    if (threadIdx.x == 0) {
        G.iters += 1;
        stop_s = !(w[0] > G.tol2 * G.rr0) || G.iters >= max_iters;
        if (stop_s) G.done = 1;
    }
    __syncthreads();
    if (stop_s) return;
    double u[1] = {0.0};
    for (int i = threadIdx.x; i < A.n_sets; i += kCgT) {
        BaCamSys& S = A.sys[i];
        ba_chol6_solve(S.L, S.r, S.z);
        for (int a = 0; a < 6; ++a) u[0] += S.r[a] * S.z[a];
    }
    cta_sum<1, kCgT>(u);
    __shared__ double beta_s;
    if (threadIdx.x == 0) {
        beta_s = u[0] / G.rz;
        G.rz = u[0];
    }
    __syncthreads();
    const double beta = beta_s;
    for (int i = threadIdx.x; i < A.n_sets; i += kCgT) {
        BaCamSys& S = A.sys[i];
        for (int a = 0; a < 6; ++a) S.p[a] = S.z[a] + beta * S.p[a];
    }
}

// the candidate poses (active sets: Exp(x_w) R, t + x_t) and g_i.x_i
__global__ void __launch_bounds__(kT) ba_cam_update_kernel(const BaArgs A, const BaCam* __restrict__ cur, BaCam* __restrict__ nxt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n_sets) return;
    BaCam c = cur[i];
    BaCamSys& S = A.sys[i];
    double gd = 0.0;
    if (c.active) {
        double R[9], t[3];
        ba_pose_update(c.K.R, c.K.t, S.x, R, t);
        for (int k = 0; k < 9; ++k) c.K.R[k] = R[k];
        for (int k = 0; k < 3; ++k) c.K.t[k] = t[k];
        tri_centre(c.K.R, c.K.t, c.K.C);
        for (int a = 0; a < 6; ++a) gd += S.g[a] * S.x[a];
    }
    S.gd = gd;
    nxt[i] = c;
}

// back-substitution: dX_j = -t_j - Vi_j sum Jp^T Jc x; the candidate point; per CTA the sum over its tracks of
// g_j.dX_j + 1/2 sum |Jc x + Jp dX_j|^2
__global__ void __launch_bounds__(kT) ba_point_back_kernel(const BaArgs A, const double* __restrict__ X, double* __restrict__ Xn,
                                                           double* __restrict__ part)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double v[1] = {0.0};
    if (t < A.n_tracks) {
        const int u0 = A.upos[A.start[t]], u1 = A.upos[A.start[t + 1]];
        double d[3] = {0.0, 0.0, 0.0};
        if (u0 < u1) {
            const BaPoint& P = A.pts[t];
            double s[3] = {0.0, 0.0, 0.0};
            for (int u = u0; u < u1; ++u) {
                const BaObs& o = A.obs[u];
                const double* x = A.sys[A.uset[u]].x;
                double c0 = 0.0, c1 = 0.0;
#pragma unroll
                for (int a = 0; a < 6; ++a) { c0 += o.Jc[a] * x[a]; c1 += o.Jc[6 + a] * x[a]; }
                for (int c = 0; c < 3; ++c) s[c] += o.Jp[c] * c0 + o.Jp[3 + c] * c1;
            }
            double w[3];
            ba_sym3_mul(P.Vi, s, w);
            for (int c = 0; c < 3; ++c) d[c] = -P.tv[c] - w[c];
            double q = 0.0;
            for (int u = u0; u < u1; ++u) {
                const BaObs& o = A.obs[u];
                const double* x = A.sys[A.uset[u]].x;
                double c0 = 0.0, c1 = 0.0;
#pragma unroll
                for (int a = 0; a < 6; ++a) { c0 += o.Jc[a] * x[a]; c1 += o.Jc[6 + a] * x[a]; }
                for (int c = 0; c < 3; ++c) { c0 += o.Jp[c] * d[c]; c1 += o.Jp[3 + c] * d[c]; }
                q += c0 * c0 + c1 * c1;
            }
            v[0] = (P.g[0] * d[0] + P.g[1] * d[1] + P.g[2] * d[2]) + 0.5 * q;
        }
        for (int c = 0; c < 3; ++c) Xn[3 * t + c] = X[3 * t + c] + d[c];
    }
    cta_sum<1, kT>(v);
    if (threadIdx.x == 0) part[blockIdx.x] = v[0];
}

// per CTA: the cost of its tracks' used observations under (cams, X); +inf when one sees its point with z <= 0
__global__ void __launch_bounds__(kT) ba_cost_kernel(const BaArgs A, const BaCam* __restrict__ cams, const double* __restrict__ X,
                                                     double* __restrict__ part)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double v[1] = {0.0};
    if (t < A.n_tracks) {
        const int u0 = A.upos[A.start[t]], u1 = A.upos[A.start[t + 1]];
        for (int u = u0; u < u1; ++u) {
            const float2 xy = A.mxy[A.umem[u]];
            double ex, ey;
            if (!tri_residual(cams[A.uset[u]].K, X + 3 * t, xy.x, xy.y, ex, ey)) { v[0] = INFINITY; break; }
            double rho, w;
            ba_loss(A.loss, (ex * ex + ey * ey) / A.s2, rho, w);
            v[0] += 0.5 * (A.s2 * rho);
        }
    }
    cta_sum<1, kT>(v);
    if (threadIdx.x == 0) part[blockIdx.x] = v[0];
}

// the step's result: cost = the sum of the cost partials; pred = -(sum g_i.x_i + the sum of the point partials)
__global__ void __launch_bounds__(kCgT) ba_reduce_kernel(const BaArgs A, const double* __restrict__ cost_part,
                                                         const double* __restrict__ pred_part, int n_part, BaStep* __restrict__ out)
{
    double v[3] = {0.0, 0.0, 0.0};
    for (int k = threadIdx.x; k < n_part; k += kCgT) {
        v[0] += cost_part[k];
        if (pred_part) v[1] += pred_part[k];
    }
    if (pred_part)
        for (int i = threadIdx.x; i < A.n_sets; i += kCgT) v[2] += A.sys[i].gd;
    cta_sum<3, kCgT>(v);
    if (threadIdx.x == 0) {
        out->cost = v[0];
        out->pred = -(v[2] + v[1]);
        out->cg_iters = pred_part ? A.cg->iters : 0;
    }
}

// Outputs: OK tracks with a used observation get X, error and angle over the used observations (ps_triangulate_tracks'
// rules); every member's pixel error under the final parameters (+inf outside OK tracks)
__global__ void __launch_bounds__(kT) ba_final_kernel(const BaArgs A, const BaCam* __restrict__ cams, const double* __restrict__ X,
                                                      const int32_t* __restrict__ mset, ps_track_point* __restrict__ points, float* __restrict__ err,
                                                      int write_points)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.n_tracks) return;
    const int s0 = A.start[t], s1 = A.start[t + 1];
    const bool ok = points[t].status == PS_TRI_OK;
    const double* Xt = X + 3 * t;
    if (err)
        for (int k = s0; k < s1; ++k) {
            double e2 = 0.0;
            const float2 xy = A.mxy[k];
            err[k] = ok && tri_error2(cams[mset[k]].K, Xt, xy.x, xy.y, e2) ? (float)sqrt(e2) : INFINITY;
        }
    const int u0 = A.upos[s0], u1 = A.upos[s1];
    if (!write_points || !ok || u0 == u1) return;
    double esum = 0.0, cmin = 2.0;
    for (int u = u0; u < u1; ++u) {
        const TriCam& K = cams[A.uset[u]].K;
        const float2 xy = A.mxy[A.umem[u]];
        double e2 = 0.0;
        tri_error2(K, Xt, xy.x, xy.y, e2);
        esum += sqrt(e2);
        double a[3] = {K.C[0] - Xt[0], K.C[1] - Xt[1], K.C[2] - Xt[2]};
        pose_unit(a);
        for (int v = u + 1; v < u1; ++v) {
            const TriCam& K2 = cams[A.uset[v]].K;
            double b[3] = {K2.C[0] - Xt[0], K2.C[1] - Xt[1], K2.C[2] - Xt[2]};
            pose_unit(b);
            cmin = fmin(cmin, a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
        }
    }
    const int n = u1 - u0;
    ps_track_point& P = points[t];
    P.X[0] = Xt[0]; P.X[1] = Xt[1]; P.X[2] = Xt[2];
    P.error = (float)(esum / n);
    P.angle = n > 1 ? (float)(acos(fmin(1.0, fmax(-1.0, cmin))) * (180.0 / 3.141592653589793)) : 0.0f;
}

} // namespace

int run_bundle_adjust(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const ps_rigid* poses_in,
                      int n_tracks, const int32_t* track_start, const int32_t* members, int n_members, ps_track_point* points,
                      const uint8_t* obs_mask, const uint8_t* fixed, const ps_bundle_params& prm, ps_rigid* poses_out, float* obs_error,
                      ps_bundle_report* report, bool* bad, cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad = false;
    const int S = n_sets, T = n_tracks, M = n_members;
    std::vector<int32_t> off(S + 1, 0);
    for (int i = 0; i < S; ++i) off[i + 1] = off[i] + n_feat[i];
    std::vector<BaCam> bc(S);
    for (int i = 0; i < S; ++i) {
        TriCam& K = bc[i].K;
        std::memcpy(K.R, poses_in[i].R, sizeof(K.R));
        std::memcpy(K.t, poses_in[i].t, sizeof(K.t));
        tri_centre(K.R, K.t, K.C);
        K.fx = cams[i].fx; K.fy = cams[i].fy; K.cx = cams[i].cx; K.cy = cams[i].cy;
        bc[i].active = 0;
        bc[i].held = -1;
    }
    // workspace: the plan (feature pointers, set offsets), the statistics and small records, then per member, per used
    // observation (sized by M, the bound), per track and per set
    const long long n_part = std::max<long long>(blocks_for(std::max(T, 1), kT), 1);
    const int nbr = (int)blocks_for(std::max(M, 1), kRadixTile);
    Workspace ws(st, "cudaMallocFromPoolAsync failed (bundle)", "bundle: plan upload failed");
    const size_t o_feat = ws.put(feat, (size_t)S * sizeof(void*)), o_off = ws.put(off.data(), off.size() * sizeof(int32_t));
    const size_t o_stat = ws.take(sizeof(BaStat)), o_cg = ws.take(sizeof(BaCg)), o_step = ws.take(sizeof(BaStep));
    const size_t o_mset = ws.take((size_t)M * 4), o_mxy = ws.take((size_t)M * 8), o_upos = ws.take(((size_t)M + 1) * 4);
    const size_t o_part = ws.take(8ull * scan_partials(std::max<long long>({(long long)M + 1, 256ll * nbr, (long long)S + 1})));
    const size_t o_umem = ws.take((size_t)M * 4), o_utrack = ws.take((size_t)M * 4), o_uset = ws.take((size_t)M * 4);
    const size_t o_la = ws.take((size_t)M * 4), o_lb = ws.take((size_t)M * 4), o_hist = ws.take(4ull * 256 * nbr);
    const size_t o_obs = ws.take((size_t)M * sizeof(BaObs));
    const size_t o_pts = ws.take((size_t)T * sizeof(BaPoint)), o_X = ws.take((size_t)T * 24), o_Xn = ws.take((size_t)T * 24);
    const size_t o_cpart = ws.take((size_t)n_part * 8), o_ppart = ws.take((size_t)n_part * 8);
    const size_t o_cstart = ws.take(((size_t)S + 1) * 4), o_sys = ws.take((size_t)S * sizeof(BaCamSys));
    const size_t o_cams = ws.take((size_t)S * sizeof(BaCam)), o_camn = ws.take((size_t)S * sizeof(BaCam));
    if (!ws.alloc(err)) return -1;
    BaStat* stat = ws.at<BaStat>(o_stat);
    BaCg* d_cg = ws.at<BaCg>(o_cg);
    BaStep* d_step = ws.at<BaStep>(o_step);
    int32_t* mset = ws.at<int32_t>(o_mset);
    float2* mxy = ws.at<float2>(o_mxy);
    int32_t* upos = ws.at<int32_t>(o_upos);
    int32_t* part = ws.at<int32_t>(o_part);
    int32_t* cstart = ws.at<int32_t>(o_cstart);
    double* X = ws.at<double>(o_X);
    double* Xn = ws.at<double>(o_Xn);
    BaCam* d_cur = ws.at<BaCam>(o_cams);
    BaCam* d_nxt = ws.at<BaCam>(o_camn);
    double* cpart = ws.at<double>(o_cpart);
    double* ppart = ws.at<double>(o_ppart);
    if (cudaMemsetAsync(stat, 0, sizeof(BaStat), st) != cudaSuccess) return ws.fail("bundle: memset failed", err);
    const long long n_items = std::max<long long>(M, (long long)T + 1);
    ba_check_kernel<<<blocks_for(n_items, kT), kT, 0, st>>>(track_start, T, members, M, ws.at<const int32_t>(o_off), S,
                                                            ws.at<const ps_feature* const>(o_feat), mset, mxy, &stat->bad);
    BaStat h{};
    if (!read_back(&h, stat, sizeof(h), st)) return ws.fail("bundle: read-back failed", err);
    if (h.bad) {
        *bad = true;
        return 1;
    }
    // the used observations, track-major (member order) and camera-major
    BaArgs A{};
    A.start = track_start;
    A.upos = upos;
    A.umem = ws.at<const int32_t>(o_umem);
    A.utrack = ws.at<const int32_t>(o_utrack);
    A.uset = ws.at<const int32_t>(o_uset);
    A.cstart = cstart;
    A.mxy = mxy;
    A.obs = ws.at<BaObs>(o_obs);
    A.pts = ws.at<BaPoint>(o_pts);
    A.sys = ws.at<BaCamSys>(o_sys);
    A.cg = d_cg;
    A.n_tracks = T;
    A.n_sets = S;
    A.loss = prm.loss;
    A.s2 = prm.loss_scale * prm.loss_scale;
    int launches = 1;
    ba_flag_kernel<<<blocks_for(std::max(T, 1), kT), kT, 0, st>>>(track_start, T, M, points, obs_mask, upos);
    launches += 1 + scan_exclusive(upos, (long long)M + 1, part, &stat->n_obs, st);
    if (cudaMemsetAsync(cstart, 0, ((size_t)S + 1) * 4, st) != cudaSuccess) return ws.fail("bundle: memset failed", err);
    ba_compact_kernel<<<blocks_for(std::max(T, 1), kT), kT, 0, st>>>(A, mset, points, ws.at<int32_t>(o_umem), ws.at<int32_t>(o_utrack),
                                                                     ws.at<int32_t>(o_uset), cstart, X, stat);
    launches += 1 + scan_exclusive(cstart, (long long)S + 1, part, &stat->pad_, st);
    if (!read_back(&h, stat, sizeof(h), st)) return ws.fail("bundle: read-back failed", err);
    const int U = h.n_obs;
    std::vector<int32_t> cs(S + 1);
    if (!read_back(cs.data(), cstart, cs.size() * 4, st)) return ws.fail("bundle: read-back failed", err);
    int32_t* la = ws.at<int32_t>(o_la);
    int32_t* lb = ws.at<int32_t>(o_lb);
    if (U > 0) {
        ba_iota_kernel<<<blocks_for(U, kT), kT, 0, st>>>(la, U);
        int bits = 0;
        while (bits < 31 && ((S - 1) >> bits) != 0) ++bits;
        const int nb = (int)blocks_for(U, kRadixTile);
        int32_t* hist = ws.at<int32_t>(o_hist);
        for (int p = 0; p < (bits + 7) / 8; ++p) {
            radix_hist_kernel<<<nb, kRadixT, 0, st>>>(la, U, SetKey{A.uset}, 8 * p, hist, nb);
            launches += 1 + scan_exclusive(hist, 256ll * nb, part, &stat->pad_, st);
            radix_scatter_kernel<<<nb, kRadixT, 0, st>>>(la, lb, U, SetKey{A.uset}, 8 * p, hist, nb);
            ++launches;
            std::swap(la, lb);
        }
    }
    A.clist = la;
    int n_free = 0;
    for (int i = 0; i < S; ++i) {
        bc[i].active = !fixed[i] && cs[i + 1] > cs[i];
        n_free += bc[i].active;
        if (i == prm.scale_set && !fixed[i]) bc[i].held = 3 + prm.scale_axis;
    }
    ws.stage(o_cams, bc.data(), (size_t)S * sizeof(BaCam));
    if (!ws.upload()) return ws.fail("bundle: camera upload failed", err);

    ps_bundle_report rep{};
    rep.n_obs = U;
    rep.n_points = h.n_points;
    rep.n_free_cams = n_free;
    const unsigned nt = blocks_for(std::max(T, 1), kT);
    auto finish_outputs = [&](bool write_points) {
        if (T > 0 && (obs_error || write_points)) {
            ba_final_kernel<<<nt, kT, 0, st>>>(A, d_cur, X, mset, points, obs_error, write_points ? 1 : 0);
            ++launches;
        }
    };
    BaStep step{};
    bool write_points = false;
    if (U == 0) {
        rep.termination = PS_BA_NO_OBSERVATIONS;
    } else {
        ba_cost_kernel<<<nt, kT, 0, st>>>(A, d_cur, X, cpart);
        ba_reduce_kernel<<<1, kCgT, 0, st>>>(A, cpart, nullptr, (int)n_part, d_step);
        launches += 2;
        if (!read_back(&step, d_step, sizeof(step), st)) return ws.fail("bundle: read-back failed", err);
        rep.initial_cost = rep.final_cost = step.cost;
        if (!std::isfinite(step.cost)) {
            rep.termination = PS_BA_NONFINITE_START;
        } else {
            write_points = true;
            double cost = step.cost, lambda = prm.initial_lambda, nu = 2.0;
            const double tol2 = prm.cg_tol * prm.cg_tol;
            bool relin = true;
            rep.termination = PS_BA_MAX_ITERS;
            for (int it = 0; it < prm.max_iters; ++it) {
                if (relin) {
                    ba_linearize_kernel<<<blocks_for(U, kT), kT, 0, st>>>(A, d_cur, X, U);
                    if (S > 0) ba_cam_grad_kernel<<<S, kCamT, 0, st>>>(A);
                    launches += 2;
                    relin = false;
                }
                ba_point_kernel<<<nt, kT, 0, st>>>(A, lambda);
                ba_cam_precond_kernel<<<S, kCamT, 0, st>>>(A, d_cur, lambda);
                ba_cg_init_kernel<<<1, kCgT, 0, st>>>(A, tol2);
                launches += 3;
                for (int c = 0; c < prm.cg_max_iters; ++c) {
                    ba_point_matvec_kernel<<<nt, kT, 0, st>>>(A);
                    ba_cam_matvec_kernel<<<S, kCamT, 0, st>>>(A, d_cur, lambda);
                    ba_cg_update_kernel<<<1, kCgT, 0, st>>>(A, prm.cg_max_iters);
                    launches += 3;
                }
                ba_cam_update_kernel<<<blocks_for(S, kT), kT, 0, st>>>(A, d_cur, d_nxt);
                ba_point_back_kernel<<<nt, kT, 0, st>>>(A, X, Xn, ppart);
                ba_cost_kernel<<<nt, kT, 0, st>>>(A, d_nxt, Xn, cpart);
                ba_reduce_kernel<<<1, kCgT, 0, st>>>(A, cpart, ppart, (int)n_part, d_step);
                launches += 4;
                if (!read_back(&step, d_step, sizeof(step), st)) return ws.fail("bundle: read-back failed", err);
                rep.iterations += 1;
                rep.cg_iterations += step.cg_iters;
                const double nc = step.cost;
                if (std::isfinite(nc) && nc < cost) {
                    const double rho = (cost - nc) / step.pred, c = 2.0 * rho - 1.0;
                    const double f = step.pred > 0.0 && std::isfinite(rho) ? std::max(1.0 / 3.0, 1.0 - c * c * c) : 1.0 / 3.0;
                    const bool small = cost - nc < prm.function_tol * cost;
                    lambda *= f;
                    nu = 2.0;
                    cost = nc;
                    std::swap(d_cur, d_nxt);
                    std::swap(X, Xn);
                    rep.accepted += 1;
                    relin = true;
                    if (small) { rep.termination = PS_BA_FUNCTION_TOL; break; }
                } else {
                    lambda *= nu;
                    nu *= 2.0;
                }
                if (lambda > 1e32) { rep.termination = PS_BA_LAMBDA; break; }
            }
            rep.final_cost = cost;
        }
    }
    finish_outputs(write_points);
    std::vector<BaCam> fin(S);
    if (S > 0 && !read_back(fin.data(), d_cur, S * sizeof(BaCam), st)) return ws.fail("bundle: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    for (int i = 0; i < S; ++i) {
        ps_rigid r;
        std::memcpy(r.R, fin[i].K.R, sizeof(r.R));
        std::memcpy(r.t, fin[i].K.t, sizeof(r.t));
        poses_out[i] = r;
    }
    *report = rep;
    return launches;
}

} // namespace psb
