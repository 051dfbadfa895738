// Global camera poses, hand-written for sm_90a: ps_rotation_averaging and ps_global_positioning (contract in
// include/popsift_b200_global.h).  The per-edge math is in k_global.h, the scan, the radix sort and the CTA sums in
// k_scan.h.
//
// Both entry points are IRLS loops around one solver: a weighted graph Laplacian with 3 unknowns per node, L x = b,
// solved by Jacobi-preconditioned CG (GlSys).  An edge e joins nodes (a, b) with weight W_e and a 3-vector g_e that enters
// b_a with + and b_b with -; (L p)_n = sum over n's edges W_e (p_n - p_other).  A node's edges come from a CSR: "camera"
// nodes [0, nC) have an edge list (one CTA per node), "point" nodes [nC, nC + nP) own a contiguous range of edges (one
// thread per node).  One node, the root, is held; a node whose weighted degree is not > 0 is held too.
//   gl_rhs_*        b, the degree D (the preconditioner), r = b, z = p = r / D, x = 0, and the partials of r.z and r.r
//   gl_cg_start     one CTA: r.z, r_0.r_0 and the device convergence flag
// per CG iteration (every kernel returns at once when the flag is set, so the host queues cg_max_iters iterations
// without waiting):
//   gl_matvec_*     q = L p and the partials of p.q
//   gl_cg_alpha     one CTA: alpha = r.z / p.q
//   gl_cg_axpy      x += alpha p, r -= alpha q, z = r / D, the partials of r.z and r.r
//   gl_cg_beta      one CTA: the stopping test and beta
//   gl_cg_dir       p = z + beta p
// Rotation averaging: nodes are the sets (all "camera" nodes, the incidence lists built on the host), edges the pairs;
// gl_rot_lin_kernel gives each used pair W = w, g = -w r; gl_rot_update_kernel applies R <- R Exp(x).
// Global positioning: camera nodes are the sets, point nodes the tracks, edges the members (weight 0 when not used);
// the camera lists are the used members sorted by set (k_scan.h's radix sort), the point ranges the track starts as they
// are.  gp_lin_kernel gives each used observation W = w d^2, g = w d e at the current positions (and its cost);
// gp_move_kernel adds a x to the positions: the solve's step is tried at a = 1, 2, 4, ... while the cost decreases.
// Sums are xor butterflies within warps and the warps in index order, partials summed by one CTA in index order; no
// floating-point atomics, so two identical calls give identical bytes.
#include "k_global.h"
#include "k_scan.h"
#include "ps_internal.h"
#include "popsift_b200_global.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

namespace psb {

namespace {

constexpr int kT = 256;                 // threads of the per-node / per-edge / per-member kernels
constexpr int kNodeT = 128;             // threads of a per-camera-node CTA
constexpr int kRedT = 256;              // threads of the single-CTA kernels
constexpr double kDeg = 3.141592653589793 / 180.0;
constexpr int kMaxDoublings = 20;       // positioning: the longest step tried is 2^20 times the solve's

struct GlCg {
    double rz, rr0, tol2, alpha, beta;
    int32_t done, iters;
};

// what the host reads back per iteration
struct GlStep {
    double cost, max_step;
    int32_t cg_iters, pad_;
};

struct GlSys {
    int nC, nP, N, root;
    const int32_t* off_c;       // nC + 1: camera node n's edges are list_c[off_c[n] .. off_c[n + 1])
    const int32_t* list_c;
    const int32_t* off_p;       // nP + 1: point node nC + j's edges are off_p[j] .. off_p[j + 1]
    const int2* ends;           // per edge (a, b)
    const double* W;            // per edge
    const double* g;            // 3 per edge
    double *x, *r, *z, *p, *q;  // 3 per node
    double* D;                  // per node: the weighted degree, 0 for a held node
    double* part;               // 2 per partial
    GlCg* cg;
};

// one edge's share of node n: MODE 0 the right-hand side (+-g) and the degree; MODE 1 W (p_n - p_other)
template <int MODE>
__device__ __forceinline__ void gl_edge(const GlSys& S, int n, int e, const double* pn, double* acc)
{
    const double w = S.W[e];
    if (w == 0.0) return;
    const int2 ab = S.ends[e];
    if (MODE == 0) {
        const double sg = ab.x == n ? 1.0 : -1.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += sg * S.g[3 * e + c];
        acc[3] += w;
    } else {
        const int o = ab.x == n ? ab.y : ab.x;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += w * (pn[c] - S.p[3 * o + c]);
    }
}

// node n's CG start from its sums (b, D): out = (r.z, r.r)
__device__ __forceinline__ void gl_node_rhs(const GlSys& S, int n, const double* acc, double* out)
{
    const bool fr = n != S.root && acc[3] > 0.0;
    const double D = fr ? acc[3] : 0.0;
    S.D[n] = D;
    out[0] = out[1] = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double r = fr ? acc[c] : 0.0;
        const double z = fr ? r / D : 0.0;
        S.x[3 * n + c] = 0.0;
        S.r[3 * n + c] = r;
        S.z[3 * n + c] = z;
        S.p[3 * n + c] = z;
        out[0] += r * z;
        out[1] += r * r;
    }
}

// node n's q from its sums: out = p.q
__device__ __forceinline__ double gl_node_q(const GlSys& S, int n, const double* acc, const double* pn)
{
    const bool fr = S.D[n] > 0.0;
    double pq = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double q = fr ? acc[c] : 0.0;
        S.q[3 * n + c] = q;
        pq += pn[c] * q;
    }
    return pq;
}

// point nodes, one thread each; partial k = blockIdx.x
template <int MODE>
__global__ void __launch_bounds__(kT) gl_point_kernel(const GlSys S)
{
    if (MODE == 1 && S.cg->done) return;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    double v[2] = {0.0, 0.0};
    if (j < S.nP) {
        const int n = S.nC + j;
        double acc[4] = {0.0, 0.0, 0.0, 0.0}, pn[3] = {0.0, 0.0, 0.0};
        if (MODE == 1)
            for (int c = 0; c < 3; ++c) pn[c] = S.p[3 * n + c];
        for (int e = S.off_p[j]; e < S.off_p[j + 1]; ++e) gl_edge<MODE>(S, n, e, pn, acc);
        if (MODE == 0) gl_node_rhs(S, n, acc, v);
        else v[0] = gl_node_q(S, n, acc, pn);
    }
    cta_sum<2, kT>(v);
    if (threadIdx.x == 0) {
        S.part[2 * blockIdx.x] = v[0];
        S.part[2 * blockIdx.x + 1] = v[1];
    }
}

// camera nodes, one CTA each; partial k = nbP + node
template <int MODE>
__global__ void __launch_bounds__(kNodeT) gl_cam_kernel(const GlSys S, int nbP)
{
    if (MODE == 1 && S.cg->done) return;
    const int n = blockIdx.x;
    double acc[4] = {0.0, 0.0, 0.0, 0.0}, pn[3] = {0.0, 0.0, 0.0};
    if (MODE == 1)
        for (int c = 0; c < 3; ++c) pn[c] = S.p[3 * n + c];
    for (int j = S.off_c[n] + threadIdx.x; j < S.off_c[n + 1]; j += kNodeT) gl_edge<MODE>(S, n, S.list_c[j], pn, acc);
    cta_sum<4, kNodeT>(acc);
    if (threadIdx.x != 0) return;
    double v[2] = {0.0, 0.0};
    if (MODE == 0) gl_node_rhs(S, n, acc, v);
    else v[0] = gl_node_q(S, n, acc, pn);
    S.part[2 * (nbP + n)] = v[0];
    S.part[2 * (nbP + n) + 1] = v[1];
}

// the two partial sums of part[0 .. n_part) in index order (valid in thread 0)
__device__ __forceinline__ void gl_sum_parts(const double* part, int n_part, double (&v)[2])
{
    v[0] = v[1] = 0.0;
    for (int k = threadIdx.x; k < n_part; k += kRedT) {
        v[0] += part[2 * k];
        v[1] += part[2 * k + 1];
    }
    cta_sum<2, kRedT>(v);
}

__global__ void __launch_bounds__(kRedT) gl_cg_start_kernel(const GlSys S, int n_part, double tol2)
{
    double v[2];
    gl_sum_parts(S.part, n_part, v);
    if (threadIdx.x == 0) {
        GlCg& G = *S.cg;
        G.rz = v[0];
        G.rr0 = v[1];
        G.tol2 = tol2;
        G.alpha = G.beta = 0.0;
        G.iters = 0;
        G.done = !(v[1] > 0.0) || !isfinite(v[0]) || !isfinite(v[1]);
    }
}

__global__ void __launch_bounds__(kRedT) gl_cg_alpha_kernel(const GlSys S, int n_part)
{
    GlCg& G = *S.cg;
    if (G.done) return;
    double v[2];
    gl_sum_parts(S.part, n_part, v);
    if (threadIdx.x == 0) {
        G.alpha = v[0] > 0.0 && isfinite(v[0]) ? G.rz / v[0] : 0.0;
        if (G.alpha == 0.0) G.done = 1;
    }
}

__global__ void __launch_bounds__(kT) gl_cg_axpy_kernel(const GlSys S)
{
    if (S.cg->done) return;
    const double alpha = S.cg->alpha;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    double v[2] = {0.0, 0.0};
    if (n < S.N) {
        const double D = S.D[n];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int i = 3 * n + c;
            S.x[i] += alpha * S.p[i];
            const double r = S.r[i] - alpha * S.q[i];
            const double z = D > 0.0 ? r / D : 0.0;
            S.r[i] = r;
            S.z[i] = z;
            v[0] += r * z;
            v[1] += r * r;
        }
    }
    cta_sum<2, kT>(v);
    if (threadIdx.x == 0) {
        S.part[2 * blockIdx.x] = v[0];
        S.part[2 * blockIdx.x + 1] = v[1];
    }
}

__global__ void __launch_bounds__(kRedT) gl_cg_beta_kernel(const GlSys S, int n_part, int max_iters)
{
    GlCg& G = *S.cg;
    if (G.done) return;
    double v[2];
    gl_sum_parts(S.part, n_part, v);
    if (threadIdx.x == 0) {
        G.iters += 1;
        if (!(v[1] > G.tol2 * G.rr0) || G.iters >= max_iters || !(G.rz != 0.0)) {
            G.done = 1;
        } else {
            G.beta = v[0] / G.rz;
            G.rz = v[0];
        }
    }
}

__global__ void __launch_bounds__(kT) gl_cg_dir_kernel(const GlSys S)
{
    if (S.cg->done) return;
    const double beta = S.cg->beta;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= S.N) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) S.p[3 * n + c] = S.z[3 * n + c] + beta * S.p[3 * n + c];
}

// L x = b by PCG from x = 0; the partials need max(nbP + nC, blocks of N) entries.  Returns the launches.
int gl_solve(const GlSys& S, int cg_max_iters, double cg_tol, cudaStream_t st)
{
    const int nbP = S.nP > 0 ? (int)blocks_for(S.nP, kT) : 0;
    const int nbN = (int)blocks_for(std::max(S.N, 1), kT);
    int launches = 2;
    if (nbP) { gl_point_kernel<0><<<nbP, kT, 0, st>>>(S); ++launches; }
    if (S.nC) gl_cam_kernel<0><<<S.nC, kNodeT, 0, st>>>(S, nbP);
    gl_cg_start_kernel<<<1, kRedT, 0, st>>>(S, nbP + S.nC, cg_tol * cg_tol);
    for (int it = 0; it < cg_max_iters; ++it) {
        if (nbP) { gl_point_kernel<1><<<nbP, kT, 0, st>>>(S); ++launches; }
        if (S.nC) { gl_cam_kernel<1><<<S.nC, kNodeT, 0, st>>>(S, nbP); ++launches; }
        gl_cg_alpha_kernel<<<1, kRedT, 0, st>>>(S, nbP + S.nC);
        gl_cg_axpy_kernel<<<nbN, kT, 0, st>>>(S);
        gl_cg_beta_kernel<<<1, kRedT, 0, st>>>(S, nbN, cg_max_iters);
        gl_cg_dir_kernel<<<nbN, kT, 0, st>>>(S);
        launches += 4;
    }
    return launches;
}

size_t gl_part_count(int nC, int nP, int N)
{
    const size_t nbP = nP > 0 ? blocks_for(nP, kT) : 0;
    return 2 * std::max<size_t>(nbP + nC, blocks_for(std::max(N, 1), kT));
}

// the cost partials summed in index order into step->cost; cg iterations copied
__global__ void __launch_bounds__(kRedT) gl_cost_kernel(const double* __restrict__ cpart, int n, const GlCg* __restrict__ cg,
                                                        GlStep* __restrict__ step)
{
    double v[1] = {0.0};
    for (int k = threadIdx.x; k < n; k += kRedT) v[0] += cpart[k];
    cta_sum<1, kRedT>(v);
    if (threadIdx.x == 0) {
        step->cost = v[0];
        step->cg_iters = cg ? cg->iters : 0;
    }
}

// ---- rotation averaging

struct RaArgs {
    const double* Rp;           // 9 per pair
    const int2* ends;           // (l, r)
    const uint8_t* used;
    double* R;                  // 9 per set
    double* W;
    double* g;
    float* err;
    double* cpart;              // per CTA of pairs
    int n_pairs, loss;
    double s2;
};

__global__ void __launch_bounds__(kT) gl_rot_lin_kernel(const RaArgs A)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    double v[1] = {0.0};
    if (p < A.n_pairs) {
        double w = 0.0, r[3] = {0.0, 0.0, 0.0};
        float err = INFINITY;
        if (A.used[p]) {
            const int2 lr = A.ends[p];
            gl_pair_residual(A.R + 9 * lr.x, A.R + 9 * lr.y, A.Rp + 9 * p, r);
            const double r2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
            double rho;
            ba_loss(A.loss, r2 / A.s2, rho, w);
            v[0] = 0.5 * (A.s2 * rho);
            err = (float)(sqrt(r2) / kDeg);
        }
        A.W[p] = w;
        for (int c = 0; c < 3; ++c) A.g[3 * p + c] = -(w * r[c]);
        A.err[p] = err;
    }
    cta_sum<1, kT>(v);
    if (threadIdx.x == 0) A.cpart[blockIdx.x] = v[0];
}

// one CTA: R_i <- R_i Exp(x_i) for the registered sets but the root; the largest |x_i| into step
__global__ void __launch_bounds__(kRedT) gl_rot_update_kernel(const RaArgs A, const GlSys S, const uint8_t* __restrict__ reg, int n_sets,
                                                              GlStep* __restrict__ step)
{
    double m = 0.0;
    for (int i = threadIdx.x; i < n_sets; i += kRedT) {
        if (!reg[i] || i == S.root) continue;
        const double* x = S.x + 3 * i;
        m = fmax(m, sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]));
        double Rn[9];
        gl_rot_update(A.R + 9 * i, x, Rn);
        for (int k = 0; k < 9; ++k) A.R[9 * i + k] = Rn[k];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ double wm[kRedT / 32];
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < kRedT / 32; ++k) m = fmax(m, wm[k]);
        step->max_step = fmax(m, wm[0]);
        step->cg_iters = S.cg->iters;
    }
}

// ---- global positioning

struct GpStat {
    int32_t bad, n_obs, n_points, pad_;
};

__device__ __forceinline__ int gp_set_of(const int32_t* __restrict__ off, int n_sets, int g)
{
    int lo = 0, hi = n_sets - 1;    // the last set with off[s] <= g (an empty set shares its offset with the next)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(off + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// one thread per member (and per track start): the checks of ps_triangulate_tracks, each member's set and its world ray
// (tri_direction); obs = registered set and a valid ray
__global__ void __launch_bounds__(kT) gp_check_kernel(const int32_t* __restrict__ start, int n_tracks, const int32_t* __restrict__ members,
                                                      int n_members, const int32_t* __restrict__ off, int n_sets,
                                                      const ps_feature* const* __restrict__ feat, const TriCam* __restrict__ cams,
                                                      const uint8_t* __restrict__ reg, int32_t* __restrict__ mset, double* __restrict__ ray,
                                                      uint8_t* __restrict__ obs, int* __restrict__ bad)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_tracks) {
        const int s = start[i];
        if ((i == 0 && s != 0) || (i == n_tracks && s != n_members) || (i < n_tracks && start[i + 1] < s)) *bad = 1;
    }
    if (i >= n_members) return;
    const int g = members[i];
    if (g < 0 || g >= off[n_sets]) { *bad = 1; return; }
    const int set = gp_set_of(off, n_sets, g);
    const ps_feature& F = feat[set][g - off[set]];
    double d[3];
    const bool ok = tri_direction(cams[set], F.xpos, F.ypos, d) && reg[set];
    mset[i] = set;
    for (int c = 0; c < 3; ++c) ray[3 * i + c] = ok ? d[c] : 0.0;
    obs[i] = ok ? 1 : 0;
}

// one thread per track: a track with >= 2 observations takes part; each member's ends (point node, camera node) and sort
// key (its set when used, else n_sets); per-set counts of used observations (integer atomics)
__global__ void __launch_bounds__(kT) gp_track_kernel(const int32_t* __restrict__ start, int n_tracks, int n_sets,
                                                      const int32_t* __restrict__ mset, const uint8_t* __restrict__ obs,
                                                      int2* __restrict__ ends, int32_t* __restrict__ key, int32_t* __restrict__ ccount,
                                                      uint8_t* __restrict__ tpart, GpStat* __restrict__ stat)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    int n = 0;
    if (t < n_tracks) {
        const int s0 = start[t], s1 = start[t + 1];
        for (int k = s0; k < s1; ++k) n += obs[k];
        const bool part = n >= 2;
        for (int k = s0; k < s1; ++k) {
            const bool used = part && obs[k];
            ends[k] = make_int2(n_sets + t, mset[k]);
            key[k] = used ? mset[k] : n_sets;
            if (used) atomicAdd(ccount + mset[k], 1);
        }
        tpart[t] = part ? 1 : 0;
        if (!part) n = 0;
    }
    const unsigned np = __reduce_add_sync(0xffffffffu, n > 0 ? 1u : 0u);
    const unsigned no = __reduce_add_sync(0xffffffffu, (unsigned)n);
    if ((threadIdx.x & 31) == 0) {
        if (np) atomicAdd(&stat->n_points, (int)np);
        if (no) atomicAdd(&stat->n_obs, (int)no);
    }
}

__global__ void __launch_bounds__(kT) gp_iota_kernel(int32_t* __restrict__ v, int n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = (int)i;
}

struct KeyOf {
    const int32_t* key;
    __device__ __forceinline__ int operator()(int k) const { return key[k]; }
};

// one thread per member: each used observation's W = w d^2 and g = w d e at the positions pos (cameras, then points);
// INIT: d = 1, w = 1 and no cost.  Per CTA the cost 1/2 s^2 rho.
template <bool INIT>
__global__ void __launch_bounds__(kT) gp_lin_kernel(int n_members, int n_sets, const int32_t* __restrict__ key, const int2* __restrict__ ends,
                                                    const double* __restrict__ ray, const double* __restrict__ pos, int loss, double s2,
                                                    double* __restrict__ W, double* __restrict__ g, double* __restrict__ cpart)
{
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double v[1] = {0.0};
    if (k < n_members) {
        double w = 0.0, e[3] = {0.0, 0.0, 0.0};
        if (key[k] < n_sets) {
            const int2 ab = ends[k];
            const double* Xp = pos + 3 * ab.x;
            const double* cp = pos + 3 * ab.y;
            double d;
            const double e2 = gl_obs(ray + 3 * k, Xp, cp, d, e);
            if (INIT) {
                d = 1.0;
                w = 1.0;
                for (int c = 0; c < 3; ++c) e[c] = ray[3 * k + c] - (Xp[c] - cp[c]);
            } else {
                double rho;
                ba_loss(loss, e2 / s2, rho, w);
                v[0] = 0.5 * (s2 * rho);
            }
            for (int c = 0; c < 3; ++c) e[c] *= w * d;
            w *= d * d;
        }
        W[k] = w;
        for (int c = 0; c < 3; ++c) g[3 * k + c] = e[c];
    }
    cta_sum<1, kT>(v);
    if (threadIdx.x == 0) cpart[blockIdx.x] = v[0];
}

__global__ void __launch_bounds__(kT) gp_move_kernel(double* __restrict__ pos, const double* __restrict__ x, double a, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pos[i] += a * x[i];
}

// d_X: the scaled points of the tracks that take part, 0 for the others
__global__ void __launch_bounds__(kT) gp_out_kernel(const double* __restrict__ pos, const uint8_t* __restrict__ tpart, int n_tracks,
                                                    double scale, double* __restrict__ X)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tracks) return;
    for (int c = 0; c < 3; ++c) X[3 * t + c] = tpart[t] ? scale * pos[3 * t + c] : 0.0;
}


} // namespace

// ---- rotation averaging: the host start

namespace {

int uf_find(std::vector<int>& par, int a)
{
    while (par[a] != a) { par[a] = par[par[a]]; a = par[a]; }
    return a;
}

} // namespace

int run_rotation_averaging(int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view, const ps_rotation_params& prm,
                           double* R_out, uint8_t* registered, float* pair_error, ps_rotation_report* report, cudaStream_t st,
                           const char** err)
{
    *err = nullptr;
    const int S = n_sets, P = n_pairs;
    std::vector<ps_two_view> tv(P);
    if (P > 0 && !read_back(tv.data(), d_two_view, (size_t)P * sizeof(ps_two_view), st)) {
        cudaGetLastError();
        *err = "rotation averaging: read-back failed";
        return -1;
    }
    // 1-2: used pairs, components, the registered one
    std::vector<uint8_t> used(P, 0);
    std::vector<int> par(S);
    std::iota(par.begin(), par.end(), 0);
    for (int p = 0; p < P; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        bool fin = true;
        for (float v : tv[p].R) fin = fin && std::isfinite(v);
        used[p] = tv[p].n_front >= prm.min_inliers && fin && l != r;
        if (used[p]) {
            const int a = uf_find(par, l), b = uf_find(par, r);
            if (a != b) par[std::max(a, b)] = std::min(a, b);
        }
    }
    std::vector<int> size(S, 0);
    for (int i = 0; i < S; ++i) ++size[uf_find(par, i)];
    int best = -1;
    for (int i = 0; i < S; ++i)       // roots are each component's smallest set, visited in ascending order
        if (par[i] == i && (best < 0 || size[i] > size[best])) best = i;
    std::vector<uint8_t> reg(S, 0);
    for (int i = 0; i < S; ++i) reg[i] = uf_find(par, i) == best;
    int n_used = 0, n_reg = 0;
    for (int p = 0; p < P; ++p) {
        used[p] = used[p] && reg[pairs[2 * p]];
        n_used += used[p];
    }
    for (int i = 0; i < S; ++i) n_reg += reg[i];
    const int root = best;              // the smallest registered set
    // 3: maximum spanning tree by n_front (Kruskal, ties to the smaller pair index), rotations chained from the root
    std::vector<double> Rp((size_t)P * 9), R((size_t)S * 9, 0.0);
    for (int p = 0; p < P; ++p)
        if (used[p]) gl_orthonormal(tv[p].R, &Rp[9 * (size_t)p]);
    for (int i = 0; i < S; ++i) R[9 * i] = R[9 * i + 4] = R[9 * i + 8] = 1.0;
    std::vector<int> order;
    for (int p = 0; p < P; ++p)
        if (used[p]) order.push_back(p);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return tv[a].n_front > tv[b].n_front; });
    std::iota(par.begin(), par.end(), 0);
    std::vector<std::vector<int>> adj(S);
    for (int p : order) {
        const int a = uf_find(par, pairs[2 * p]), b = uf_find(par, pairs[2 * p + 1]);
        if (a == b) continue;
        par[a] = b;
        adj[pairs[2 * p]].push_back(p);
        adj[pairs[2 * p + 1]].push_back(p);
    }
    if (S > 0) {
        std::vector<uint8_t> known(S, 0);
        std::vector<int> stack{root};
        known[root] = 1;
        while (!stack.empty()) {
            const int i = stack.back();
            stack.pop_back();
            for (int p : adj[i]) {
                const int l = pairs[2 * p], r = pairs[2 * p + 1];
                const int o = l == i ? r : l;
                if (known[o]) continue;
                if (o == r) gl_mul(&Rp[9 * (size_t)p], &R[9 * (size_t)l], &R[9 * (size_t)r]);
                else gl_mul_tn(&Rp[9 * (size_t)p], &R[9 * (size_t)r], &R[9 * (size_t)l]);
                known[o] = 1;
                stack.push_back(o);
            }
        }
    }
    ps_rotation_report rep{};
    rep.n_pairs = n_used;
    rep.n_registered = n_reg;
    std::vector<float> perr(P, INFINITY);
    int launches = 0;
    if (n_used == 0) {
        rep.termination = PS_RA_NO_PAIRS;
    } else {
        // the incidence lists of the used pairs, set-major, pairs ascending
        std::vector<int32_t> off(S + 1, 0), list;
        for (int p = 0; p < P; ++p)
            if (used[p]) { ++off[pairs[2 * p] + 1]; ++off[pairs[2 * p + 1] + 1]; }
        for (int i = 0; i < S; ++i) off[i + 1] += off[i];
        list.resize(off[S]);
        std::vector<int32_t> fill(off.begin(), off.end() - 1);
        for (int p = 0; p < P; ++p)
            if (used[p]) { list[fill[pairs[2 * p]]++] = p; list[fill[pairs[2 * p + 1]]++] = p; }
        const int nbp = (int)blocks_for(P, kT);
        const size_t npart = gl_part_count(S, 0, S);
        std::vector<int2> ends(P);
        for (int p = 0; p < P; ++p) ends[p] = make_int2(pairs[2 * p], pairs[2 * p + 1]);
        // everything before the partials is uploaded, the solver's state and the per-pair outputs as zeros
        Workspace ws(st, "cudaMallocFromPoolAsync failed (rotation averaging)", "rotation averaging: upload failed");
        const size_t o_cg = ws.put(nullptr, sizeof(GlCg)), o_step = ws.put(nullptr, sizeof(GlStep));
        const size_t o_Rp = ws.put(Rp.data(), (size_t)P * 72), o_ends = ws.put(ends.data(), (size_t)P * 8), o_used = ws.put(used.data(), P);
        const size_t o_W = ws.put(nullptr, (size_t)P * 8), o_g = ws.put(nullptr, (size_t)P * 24), o_err = ws.put(nullptr, (size_t)P * 4);
        const size_t o_cpart = ws.put(nullptr, (size_t)nbp * 8), o_off = ws.put(off.data(), off.size() * 4);
        const size_t o_list = ws.put(list.data(), list.size() * 4), o_R = ws.put(R.data(), (size_t)S * 72), o_reg = ws.put(reg.data(), S);
        const size_t o_vec = ws.put(nullptr, (size_t)S * 5 * 24), o_D = ws.put(nullptr, (size_t)S * 8);
        const size_t o_part = ws.take(npart * 8);
        if (!ws.alloc(err)) return -1;
        GlStep* d_step = ws.at<GlStep>(o_step);
        RaArgs A{};
        A.Rp = ws.at<const double>(o_Rp);
        A.ends = ws.at<const int2>(o_ends);
        A.used = ws.at<uint8_t>(o_used);
        A.R = ws.at<double>(o_R);
        A.W = ws.at<double>(o_W);
        A.g = ws.at<double>(o_g);
        A.err = ws.at<float>(o_err);
        A.cpart = ws.at<double>(o_cpart);
        A.n_pairs = P;
        A.loss = prm.loss;
        const double s = prm.loss_scale * kDeg;
        A.s2 = s * s;
        GlSys G{};
        G.nC = S;
        G.nP = 0;
        G.N = S;
        G.root = root;
        G.off_c = ws.at<const int32_t>(o_off);
        G.list_c = ws.at<const int32_t>(o_list);
        G.ends = A.ends;
        G.W = A.W;
        G.g = A.g;
        double* vec = ws.at<double>(o_vec);
        G.x = vec;
        G.r = vec + 3 * (size_t)S;
        G.z = vec + 6 * (size_t)S;
        G.p = vec + 9 * (size_t)S;
        G.q = vec + 12 * (size_t)S;
        G.D = ws.at<double>(o_D);
        G.part = ws.at<double>(o_part);
        G.cg = ws.at<GlCg>(o_cg);
        const uint8_t* d_reg = ws.at<const uint8_t>(o_reg);
        GlStep step{};
        auto lin = [&]() {
            gl_rot_lin_kernel<<<nbp, kT, 0, st>>>(A);
            gl_cost_kernel<<<1, kRedT, 0, st>>>(A.cpart, nbp, nullptr, d_step);
            launches += 2;
        };
        const double step_tol = prm.step_tol * kDeg;
        rep.termination = PS_RA_MAX_ITERS;
        lin();
        for (int it = 0; it < prm.max_iters; ++it) {
            launches += gl_solve(G, prm.cg_max_iters, prm.cg_tol, st);
            gl_rot_update_kernel<<<1, kRedT, 0, st>>>(A, G, d_reg, S, d_step);
            ++launches;
            if (!read_back(&step, d_step, sizeof(step), st)) return ws.fail("rotation averaging: read-back failed", err);
            if (it == 0) rep.initial_cost = step.cost;
            rep.iterations += 1;
            rep.cg_iterations += step.cg_iters;
            lin();
            if (step.max_step < step_tol) { rep.termination = PS_RA_STEP_TOL; break; }
        }
        if (!read_back(&step, d_step, sizeof(step), st)) return ws.fail("rotation averaging: read-back failed", err);
        if (prm.max_iters == 0) rep.initial_cost = step.cost;
        rep.final_cost = step.cost;
        if (!read_back(R.data(), A.R, R.size() * 8, st) || (P > 0 && !read_back(perr.data(), A.err, (size_t)P * 4, st)))
            return ws.fail("rotation averaging: read-back failed", err);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    }
    for (int i = 0; i < S; ++i) {
        for (int k = 0; k < 9; ++k) R_out[9 * i + k] = reg[i] ? R[9 * i + k] : (k % 4 == 0 ? 1.0 : 0.0);
        registered[i] = reg[i];
    }
    if (pair_error) std::memcpy(pair_error, perr.data(), (size_t)P * 4);
    *report = rep;
    return launches;
}

int run_global_positioning(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const double* R,
                           const uint8_t* registered, int n_tracks, const int32_t* track_start, const int32_t* members, int n_members,
                           const ps_position_params& prm, ps_rigid* poses_out, uint8_t* positioned, double* X_out,
                           ps_position_report* report, bool* bad, cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad = false;
    const int S = n_sets, T = n_tracks, M = n_members, N = S + T;
    std::vector<int32_t> off(S + 1, 0);
    for (int i = 0; i < S; ++i) off[i + 1] = off[i] + n_feat[i];
    std::vector<TriCam> tc(S);
    for (int i = 0; i < S; ++i) {
        TriCam& K = tc[i];
        std::memset(&K, 0, sizeof(K));
        std::memcpy(K.R, R + 9 * (size_t)i, sizeof(K.R));
        K.fx = cams[i].fx; K.fy = cams[i].fy; K.cx = cams[i].cx; K.cy = cams[i].cy;
    }
    const int nbm = (int)blocks_for(std::max(M, 1), kT);
    const int nbr = (int)blocks_for(std::max(M, 1), kRadixTile);
    const size_t npart = gl_part_count(S, T, N);
    Workspace ws(st, "cudaMallocFromPoolAsync failed (positioning)", "positioning: plan upload failed");
    const size_t o_feat = ws.put(feat, (size_t)S * sizeof(void*)), o_off = ws.put(off.data(), off.size() * 4);
    const size_t o_cams = ws.put(tc.data(), (size_t)S * sizeof(TriCam)), o_reg = ws.put(S > 0 ? registered : nullptr, std::max(S, 1));
    const size_t o_stat = ws.take(sizeof(GpStat)), o_cg = ws.take(sizeof(GlCg)), o_step = ws.take(sizeof(GlStep));
    const size_t o_mset = ws.take((size_t)M * 4), o_ray = ws.take((size_t)M * 24), o_obs = ws.take(M), o_ends = ws.take((size_t)M * 8);
    const size_t o_key = ws.take((size_t)M * 4), o_la = ws.take((size_t)M * 4), o_lb = ws.take((size_t)M * 4);
    const size_t o_W = ws.take((size_t)M * 8), o_g = ws.take((size_t)M * 24), o_cpart = ws.take((size_t)nbm * 8);
    const size_t o_hist = ws.take(4ull * 256 * nbr);
    const size_t o_spart = ws.take(4ull * scan_partials(std::max<long long>(256ll * nbr, (long long)S + 1)));
    const size_t o_cstart = ws.take(((size_t)S + 1) * 4), o_tpart = ws.take(std::max(T, 1));
    const size_t o_pos = ws.take((size_t)N * 24), o_vec = ws.take((size_t)N * 5 * 24), o_D = ws.take((size_t)N * 8);
    const size_t o_part = ws.take(npart * 8);
    if (!ws.alloc(err)) return -1;
    GpStat* stat = ws.at<GpStat>(o_stat);
    GlStep* d_step = ws.at<GlStep>(o_step);
    int32_t* mset = ws.at<int32_t>(o_mset);
    double* ray = ws.at<double>(o_ray);
    uint8_t* obs = ws.at<uint8_t>(o_obs);
    int2* ends = ws.at<int2>(o_ends);
    int32_t* key = ws.at<int32_t>(o_key);
    int32_t* spart = ws.at<int32_t>(o_spart);
    int32_t* cstart = ws.at<int32_t>(o_cstart);
    uint8_t* tpart = ws.at<uint8_t>(o_tpart);
    double* pos = ws.at<double>(o_pos);
    double* W = ws.at<double>(o_W);
    double* g = ws.at<double>(o_g);
    double* cpart = ws.at<double>(o_cpart);
    if (cudaMemsetAsync(stat, 0, sizeof(GpStat), st) != cudaSuccess) return ws.fail("positioning: memset failed", err);
    const long long n_items = std::max<long long>(M, (long long)T + 1);
    gp_check_kernel<<<blocks_for(n_items, kT), kT, 0, st>>>(track_start, T, members, M, ws.at<const int32_t>(o_off), S,
                                                            ws.at<const ps_feature* const>(o_feat), ws.at<const TriCam>(o_cams),
                                                            ws.at<const uint8_t>(o_reg), mset, ray, obs, &stat->bad);
    GpStat h{};
    if (!read_back(&h, stat, sizeof(h), st)) return ws.fail("positioning: read-back failed", err);
    if (h.bad) {
        *bad = true;
        return 1;
    }
    int launches = 1;
    if (cudaMemsetAsync(cstart, 0, ((size_t)S + 1) * 4, st) != cudaSuccess || cudaMemsetAsync(pos, 0, (size_t)N * 24, st) != cudaSuccess)
        return ws.fail("positioning: memset failed", err);
    if (T > 0) {
        gp_track_kernel<<<blocks_for(T, kT), kT, 0, st>>>(track_start, T, S, mset, obs, ends, key, cstart, tpart, stat);
        ++launches;
    }
    launches += scan_exclusive(cstart, (long long)S + 1, spart, &stat->pad_, st);
    int32_t* la = ws.at<int32_t>(o_la);
    int32_t* lb = ws.at<int32_t>(o_lb);
    if (M > 0) {
        gp_iota_kernel<<<nbm, kT, 0, st>>>(la, M);
        ++launches;
        int bits = 0;
        while (bits < 31 && (S >> bits) != 0) ++bits;      // keys 0 .. S
        int32_t* hist = ws.at<int32_t>(o_hist);
        for (int p = 0; p < (bits + 7) / 8; ++p) {
            radix_hist_kernel<<<nbr, kRadixT, 0, st>>>(la, M, KeyOf{key}, 8 * p, hist, nbr);
            launches += 1 + scan_exclusive(hist, 256ll * nbr, spart, &stat->pad_, st);
            radix_scatter_kernel<<<nbr, kRadixT, 0, st>>>(la, lb, M, KeyOf{key}, 8 * p, hist, nbr);
            ++launches;
            std::swap(la, lb);
        }
    }
    std::vector<int32_t> cs(S + 1);
    if (!read_back(&h, stat, sizeof(h), st) || !read_back(cs.data(), cstart, cs.size() * 4, st))
        return ws.fail("positioning: read-back failed", err);
    int root = -1, n_cams = 0;
    for (int i = 0; i < S; ++i) {
        positioned[i] = cs[i + 1] > cs[i];
        n_cams += positioned[i];
        if (positioned[i] && root < 0) root = i;
    }
    ps_position_report rep{};
    rep.n_obs = h.n_obs;
    rep.n_points = h.n_points;
    rep.n_cams = n_cams;
    std::vector<double> cpos((size_t)S * 3, 0.0);
    double scale = 1.0;
    if (h.n_obs == 0) {
        rep.termination = PS_GP_NO_OBSERVATIONS;
    } else {
        GlSys G{};
        G.nC = S;
        G.nP = T;
        G.N = N;
        G.root = root;
        G.off_c = cstart;
        G.list_c = la;
        G.off_p = track_start;
        G.ends = ends;
        G.W = W;
        G.g = g;
        double* vec = ws.at<double>(o_vec);
        G.x = vec;
        G.r = vec + 3 * (size_t)N;
        G.z = vec + 6 * (size_t)N;
        G.p = vec + 9 * (size_t)N;
        G.q = vec + 12 * (size_t)N;
        G.D = ws.at<double>(o_D);
        G.part = ws.at<double>(o_part);
        G.cg = ws.at<GlCg>(o_cg);
        const double s2 = prm.loss_scale * prm.loss_scale;
        const unsigned nbn3 = blocks_for(3ll * N, kT);
        GlStep step{};
        // positions += a x, then the weights, right-hand side and cost there (read back into step)
        auto move_lin = [&](double a) {
            gp_move_kernel<<<nbn3, kT, 0, st>>>(pos, G.x, a, 3ll * N);
            gp_lin_kernel<false><<<nbm, kT, 0, st>>>(M, S, key, ends, ray, pos, prm.loss, s2, W, g, cpart);
            gl_cost_kernel<<<1, kRedT, 0, st>>>(cpart, nbm, G.cg, d_step);
            launches += 3;
            return read_back(&step, d_step, sizeof(step), st);
        };
        gp_lin_kernel<true><<<nbm, kT, 0, st>>>(M, S, key, ends, ray, pos, prm.loss, s2, W, g, cpart);
        ++launches;
        launches += gl_solve(G, prm.cg_max_iters, prm.cg_tol, st);
        if (!move_lin(1.0)) return ws.fail("positioning: read-back failed", err);
        rep.initial_cost = rep.final_cost = step.cost;
        rep.cg_iterations = step.cg_iters;
        rep.termination = PS_GP_MAX_ITERS;
        double cost = step.cost;
        for (int it = 0; it < prm.max_iters; ++it) {
            launches += gl_solve(G, prm.cg_max_iters, prm.cg_tol, st);
            if (!move_lin(1.0)) return ws.fail("positioning: read-back failed", err);
            rep.iterations += 1;
            rep.cg_iterations += step.cg_iters;
            // the step lengthened: 2^k x for k = 1 .. kMaxDoublings while the cost keeps decreasing
            double best = step.cost, a = 1.0;
            for (int k = 0; k < kMaxDoublings; ++k) {
                if (!move_lin(a)) return ws.fail("positioning: read-back failed", err);
                if (!(step.cost < best)) {
                    if (!move_lin(-a)) return ws.fail("positioning: read-back failed", err);
                    break;
                }
                best = step.cost;
                a *= 2.0;
            }
            const double nc = best;
            const bool small = !(cost - nc >= prm.function_tol * cost);
            cost = nc;
            if (small) { rep.termination = PS_GP_FUNCTION_TOL; break; }
        }
        rep.final_cost = cost;
        if (S > 0 && !read_back(cpos.data(), pos, cpos.size() * 8, st)) return ws.fail("positioning: read-back failed", err);
        double ss = 0.0;
        for (int i = 0; i < S; ++i)
            if (positioned[i])
                for (int c = 0; c < 3; ++c) ss += cpos[3 * i + c] * cpos[3 * i + c];
        if (n_cams > 1 && ss > 0.0) scale = 1.0 / std::sqrt(ss / n_cams);
    }
    if (X_out && T > 0) {
        gp_out_kernel<<<blocks_for(T, kT), kT, 0, st>>>(pos + 3 * (size_t)S, tpart, T, scale, X_out);
        ++launches;
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) return ws.fail("positioning: synchronise failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    for (int i = 0; i < S; ++i) {
        ps_rigid r;
        std::memcpy(r.R, R + 9 * (size_t)i, sizeof(r.R));
        for (int a = 0; a < 3; ++a) {
            const double* Ri = R + 9 * (size_t)i + 3 * a;
            const double* c = &cpos[3 * i];
            r.t[a] = positioned[i] ? -(Ri[0] * (scale * c[0]) + Ri[1] * (scale * c[1]) + Ri[2] * (scale * c[2])) : 0.0;
        }
        poses_out[i] = r;
    }
    *report = rep;
    return launches;
}

} // namespace psb
