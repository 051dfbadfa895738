// Multi-view triangulation, hand-written for sm_90a: ps_triangulate_tracks (contract in include/popsift_b200_triangulate.h).
// The per-observation math is in k_triangulate.h, the two-ray rule in k_pose_solve.h and the sample hash in
// k_verify_sample.h.
//
// One workspace (workspace.h), all launches on one stream:
//   1. tri_ray_kernel    one thread per member: the member id's bounds and the monotonicity of d_track_start (a flag), the
//                        member's set, pixel and unit ray direction.  The flag is read back before anything is written.
//   2. tri_track_kernel  one warp per track.  Hypotheses go across the lanes; each lane scores its hypotheses on all of
//                        the track's rays, which the whole warp reads at the same address (one broadcast per load).  The
//                        winner by an xor butterfly on (count, h); the Gauss-Newton sums and the error sum by xor
//                        butterflies (every lane ends with the same bits: a + b == b + a), so every lane takes the same
//                        decisions; members' outputs lane-strided; the angle over inlier pairs from blocks of 32 members
//                        exchanged by shuffles.  Each lane reads from memory only what it wrote itself.
//   3. tri_count_kernel  tracks per status and inlier observations: a shared histogram per block, one atomic per block
//                        and counter.
#include "k_triangulate.h"
#include "k_verify_sample.h"
#include "ps_internal.h"
#include "popsift_b200_triangulate.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kRayThreads = 256;
constexpr int kTrackWarps = 4;
constexpr int kCountThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

// one member's observation: its ray direction, pixel and set
struct TriRay {
    double d[3];
    float x, y;
    int32_t set, pad_;
};

struct TriStat {
    int32_t bad;
    int32_t n_status[PS_TRI_NUM_STATUS];
    int32_t n_inlier_obs, pad_;
};

struct TriArgs {
    const int32_t* start;
    const TriRay* rays;
    const TriCam* cams;
    int n_tracks, min_views, n_samples, refine_iters;
    uint64_t seed;
    double thr2, cos_min;
    ps_track_point* points;
    uint8_t* mask;
    float* err;
};

__device__ __forceinline__ int tri_set_of(const int32_t* __restrict__ off, int n_sets, int g)
{
    int lo = 0, hi = n_sets - 1;    // the last set with off[s] <= g (an empty set shares its offset with the next)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(off + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kRayThreads) tri_ray_kernel(const int32_t* __restrict__ start, int n_tracks, const int32_t* __restrict__ members,
                                                              int n_members, const int32_t* __restrict__ off, int n_sets,
                                                              const ps_feature* const* __restrict__ feat, const TriCam* __restrict__ cams,
                                                              TriRay* __restrict__ rays, int* __restrict__ bad)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= n_tracks) {
        const int s = start[i];
        if ((i == 0 && s != 0) || (i == n_tracks && s != n_members) || (i < n_tracks && start[i + 1] < s)) *bad = 1;
    }
    if (i >= n_members) return;
    const int g = members[i];
    if (g < 0 || g >= off[n_sets]) { *bad = 1; return; }
    const int set = tri_set_of(off, n_sets, g);
    const ps_feature& F = feat[set][g - off[set]];
    TriRay r;
    r.x = F.xpos;
    r.y = F.ypos;
    r.set = set;
    r.pad_ = 0;
    tri_direction(cams[set], r.x, r.y, r.d);
    rays[i] = r;
}

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// inliers of X among the track's L rays (the whole warp reads ray j at once)
__device__ int tri_count(const TriArgs& A, const TriRay* __restrict__ ray, int L, const double* X)
{
    int c = 0;
    for (int j = 0; j < L; ++j) {
        const TriRay r = ray[j];
        double e2;
        if (tri_error2(A.cams[r.set], X, r.x, r.y, e2) && e2 <= A.thr2) ++c;
    }
    return c;
}

// The Gauss-Newton sums at X over the members with m[j] != 0: S[0..5] J^T J, S[6..8] -J^T e, S[9] the sum of e2 (+inf
// when one of them sees X with z <= 0); identical on every lane.
__device__ void tri_normal(const TriArgs& A, const TriRay* __restrict__ ray, const uint8_t* m, int L, const double* X, int lane, double (&S)[10])
{
    double s[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    bool behind = false;
    for (int j = lane; j < L; j += 32) {
        if (!m[j]) continue;
        const TriRay r = ray[j];
        double ex, ey, Jx[3], Jy[3];
        if (!tri_residual(A.cams[r.set], X, r.x, r.y, ex, ey, Jx, Jy)) { behind = true; continue; }
        s[0] += Jx[0] * Jx[0] + Jy[0] * Jy[0];
        s[1] += Jx[0] * Jx[1] + Jy[0] * Jy[1];
        s[2] += Jx[0] * Jx[2] + Jy[0] * Jy[2];
        s[3] += Jx[1] * Jx[1] + Jy[1] * Jy[1];
        s[4] += Jx[1] * Jx[2] + Jy[1] * Jy[2];
        s[5] += Jx[2] * Jx[2] + Jy[2] * Jy[2];
        s[6] -= Jx[0] * ex + Jy[0] * ey;
        s[7] -= Jx[1] * ex + Jy[1] * ey;
        s[8] -= Jx[2] * ex + Jy[2] * ey;
        s[9] += ex * ex + ey * ey;
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) S[k] = warp_sum(s[k]);
    if (__any_sync(kFull, behind)) S[9] = INFINITY;
}

// member j < L an inlier under X: *u = the unit vector from X to its camera centre
__device__ bool tri_unit(const TriArgs& A, const TriRay* __restrict__ ray, int j, int L, const double* X, double* u)
{
    if (j >= L) return false;
    const TriRay r = ray[j];
    const TriCam& K = A.cams[r.set];
    double e2;
    if (!(tri_error2(K, X, r.x, r.y, e2) && e2 <= A.thr2)) return false;
    u[0] = K.C[0] - X[0]; u[1] = K.C[1] - X[1]; u[2] = K.C[2] - X[2];
    pose_unit(u);
    return true;
}

__global__ void __launch_bounds__(kTrackWarps * 32) tri_track_kernel(const TriArgs A)
{
    const int lane = threadIdx.x & 31;
    const long long t = (long long)blockIdx.x * kTrackWarps + (threadIdx.x >> 5);
    if (t >= A.n_tracks) return;
    const int s0 = A.start[t], L = A.start[t + 1] - s0;
    const TriRay* ray = A.rays + s0;
    uint8_t* mask = A.mask + s0;
    float* err = A.err ? A.err + s0 : nullptr;
    ps_track_point rec{};
    int bc = -1, bh = 0x7fffffff;
    double X[3] = {0.0, 0.0, 0.0};
    if (L >= A.min_views) {
        const bool all = (long long)L * (L - 1) / 2 <= A.n_samples;
        const int H = all ? L * (L - 1) / 2 : A.n_samples;
        for (int h = lane; h < H; h += 32) {
            int a, b;
            if (all) {
                int r = h;
                a = 0;
                while (r >= L - 1 - a) { r -= L - 1 - a; ++a; }
                b = a + 1 + r;
            } else {
                uint32_t idx[2];
                if (!verify_sample<2>(A.seed, (int)t, h, (uint32_t)L, idx)) continue;
                a = (int)min(idx[0], idx[1]);
                b = (int)max(idx[0], idx[1]);
            }
            const TriRay ra = ray[a], rb = ray[b];
            double Xh[3];
            if (!tri_hypothesis(A.cams[ra.set].C, ra.d, A.cams[rb.set].C, rb.d, A.cos_min, Xh)) continue;
            const int c = tri_count(A, ray, L, Xh);
            if (c > bc) { bc = c; bh = h; X[0] = Xh[0]; X[1] = Xh[1]; X[2] = Xh[2]; }
        }
        // the winner: most inliers, ties to the smallest h (a total order, so every lane ends with it)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int oc = __shfl_xor_sync(kFull, bc, o), oh = __shfl_xor_sync(kFull, bh, o);
            const double x0 = __shfl_xor_sync(kFull, X[0], o), x1 = __shfl_xor_sync(kFull, X[1], o), x2 = __shfl_xor_sync(kFull, X[2], o);
            if (oc > bc || (oc == bc && oh < bh)) { bc = oc; bh = oh; X[0] = x0; X[1] = x1; X[2] = x2; }
        }
        rec.status = bc < 0 ? PS_TRI_NO_HYPOTHESIS : PS_TRI_OK;
    } else {
        rec.status = PS_TRI_TOO_FEW_OBS;
    }
    if (bc < 0) {
        for (int j = lane; j < L; j += 32) {
            mask[j] = 0;
            if (err) err[j] = INFINITY;
        }
        if (lane == 0) A.points[t] = rec;
        return;
    }
    if (A.refine_iters > 0) {
        // the winner's inliers, kept in the mask for the refinement (each lane reads back only its own members)
        for (int j = lane; j < L; j += 32) {
            const TriRay r = ray[j];
            double e2;
            mask[j] = tri_error2(A.cams[r.set], X, r.x, r.y, e2) && e2 <= A.thr2 ? 1 : 0;
        }
        double S[10], Xr[3] = {X[0], X[1], X[2]};
        tri_normal(A, ray, mask, L, Xr, lane, S);
        for (int it = 0; it < A.refine_iters; ++it) {
            double dX[3], Sn[10];
            if (!tri_step(S, dX)) break;
            const double Xn[3] = {Xr[0] + dX[0], Xr[1] + dX[1], Xr[2] + dX[2]};
            tri_normal(A, ray, mask, L, Xn, lane, Sn);
            if (!(Sn[9] < S[9])) break;
            for (int k = 0; k < 3; ++k) Xr[k] = Xn[k];
            for (int k = 0; k < 10; ++k) S[k] = Sn[k];
        }
        int c = 0;
        for (int j = lane; j < L; j += 32) {
            const TriRay r = ray[j];
            double e2;
            c += tri_error2(A.cams[r.set], Xr, r.x, r.y, e2) && e2 <= A.thr2 ? 1 : 0;
        }
        if (__reduce_add_sync(kFull, (unsigned)c) >= (unsigned)bc)
            for (int k = 0; k < 3; ++k) X[k] = Xr[k];
    }
    // the outputs under the final X
    int n_in = 0;
    double esum = 0.0;
    for (int j = lane; j < L; j += 32) {
        const TriRay r = ray[j];
        double e2 = 0.0;
        const bool front = tri_error2(A.cams[r.set], X, r.x, r.y, e2);
        const bool in = front && e2 <= A.thr2;
        mask[j] = in ? 1 : 0;
        if (err) err[j] = front ? (float)sqrt(e2) : INFINITY;
        if (in) {
            ++n_in;
            esum += sqrt(e2);
        }
    }
    n_in = (int)__reduce_add_sync(kFull, (unsigned)n_in);
    esum = warp_sum(esum);
    // The smallest cosine over pairs of inliers.  Blocks of 32 members: lane k holds member ca + k of block ca and
    // compares it with the 32 members of each block cb >= ca, which come by shuffles; no lane reads another's results
    // from memory.
    double cmin = 2.0;
    if (n_in > 1) {
        for (int ca = 0; ca < L; ca += 32) {
            double ua[3] = {0.0, 0.0, 0.0};
            const bool ia = tri_unit(A, ray, ca + lane, L, X, ua);
            for (int cb = ca; cb < L; cb += 32) {
                double ub[3] = {ua[0], ua[1], ua[2]};
                const bool ib = cb == ca ? ia : tri_unit(A, ray, cb + lane, L, X, ub);
                const int kn = min(32, L - cb);      // the block's members (the same on every lane)
                for (int k = 0; k < kn; ++k) {
                    const double v0 = __shfl_sync(kFull, ub[0], k), v1 = __shfl_sync(kFull, ub[1], k), v2 = __shfl_sync(kFull, ub[2], k);
                    const bool iv = __shfl_sync(kFull, ib ? 1 : 0, k) != 0;
                    if (ia && iv && cb + k > ca + lane) cmin = fmin(cmin, ua[0] * v0 + ua[1] * v1 + ua[2] * v2);
                }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmin = fmin(cmin, __shfl_xor_sync(kFull, cmin, o));
    if (lane == 0) {
        rec.X[0] = X[0]; rec.X[1] = X[1]; rec.X[2] = X[2];
        rec.n_inliers = n_in;
        rec.error = n_in > 0 ? (float)(esum / n_in) : 0.0f;
        rec.angle = n_in > 1 ? (float)(acos(fmin(1.0, fmax(-1.0, cmin))) * (180.0 / 3.141592653589793)) : 0.0f;
        rec.status = n_in < A.min_views ? PS_TRI_TOO_FEW_INLIERS : (cmin > A.cos_min ? PS_TRI_SMALL_ANGLE : PS_TRI_OK);
        A.points[t] = rec;
    }
}

__global__ void __launch_bounds__(kCountThreads) tri_count_kernel(const ps_track_point* __restrict__ points, int n_tracks, TriStat* __restrict__ stat)
{
    __shared__ int h[PS_TRI_NUM_STATUS + 1];
    if (threadIdx.x <= PS_TRI_NUM_STATUS) h[threadIdx.x] = 0;
    __syncthreads();
    int c[PS_TRI_NUM_STATUS + 1] = {0, 0, 0, 0, 0, 0};
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_tracks; t += (long long)gridDim.x * blockDim.x) {
        const ps_track_point& p = points[t];
        const int s = p.status;
#pragma unroll
        for (int k = 0; k < PS_TRI_NUM_STATUS; ++k) c[k] += s == k ? 1 : 0;
        c[PS_TRI_NUM_STATUS] += p.n_inliers;
    }
#pragma unroll
    for (int k = 0; k <= PS_TRI_NUM_STATUS; ++k) {
        const int v = (int)__reduce_add_sync(kFull, (unsigned)c[k]);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(&h[k], v);
    }
    __syncthreads();
    if (threadIdx.x < PS_TRI_NUM_STATUS && h[threadIdx.x]) atomicAdd(&stat->n_status[threadIdx.x], h[threadIdx.x]);
    if (threadIdx.x == PS_TRI_NUM_STATUS && h[threadIdx.x]) atomicAdd(&stat->n_inlier_obs, h[threadIdx.x]);
}

} // namespace

int run_triangulate_tracks(int n_sets, const int32_t* n_feat, const ps_feature* const* feat, const ps_camera* cams, const ps_rigid* poses,
                           int n_tracks, const int32_t* track_start, const int32_t* members, int n_members,
                           const ps_triangulate_params& prm, ps_track_point* points, uint8_t* obs_mask, float* obs_error,
                           ps_triangulate_counts* counts, bool* bad, cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad = false;
    std::vector<int32_t> off(n_sets + 1, 0);
    for (int i = 0; i < n_sets; ++i) off[i + 1] = off[i] + n_feat[i];
    std::vector<TriCam> tc(n_sets);
    for (int i = 0; i < n_sets; ++i) {
        TriCam& K = tc[i];
        std::memcpy(K.R, poses[i].R, sizeof(K.R));
        std::memcpy(K.t, poses[i].t, sizeof(K.t));
        tri_centre(K.R, K.t, K.C);
        K.fx = cams[i].fx; K.fy = cams[i].fy; K.cx = cams[i].cx; K.cy = cams[i].cy;
    }
    // workspace: the plan (cameras, feature pointers, set offsets), the statistics, then 40 bytes per member
    Workspace ws(st, "cudaMallocFromPoolAsync failed (triangulate)", "triangulate: plan upload failed");
    const size_t o_cams = ws.put(tc.data(), tc.size() * sizeof(TriCam)), o_feat = ws.put(feat, (size_t)n_sets * sizeof(void*));
    const size_t o_off = ws.put(off.data(), off.size() * sizeof(int32_t));
    const size_t o_stat = ws.take(sizeof(TriStat));
    const size_t o_rays = ws.take((size_t)n_members * sizeof(TriRay));
    if (!ws.alloc(err)) return -1;
    TriStat* stat = ws.at<TriStat>(o_stat);
    if (cudaMemsetAsync(stat, 0, sizeof(TriStat), st) != cudaSuccess) return ws.fail("triangulate: memset failed", err);
    const TriCam* d_cams = ws.at<const TriCam>(o_cams);
    TriRay* rays = ws.at<TriRay>(o_rays);
    const long long n_items = std::max<long long>(n_members, (long long)n_tracks + 1);
    tri_ray_kernel<<<blocks_for(n_items, kRayThreads), kRayThreads, 0, st>>>(
        track_start, n_tracks, members, n_members, ws.at<const int32_t>(o_off), n_sets, ws.at<const ps_feature* const>(o_feat), d_cams,
        rays, &stat->bad);
    TriStat h{};
    if (!read_back(&h, stat, sizeof(TriStat), st)) return ws.fail("triangulate: read-back failed", err);
    if (h.bad) {
        *bad = true;
        return 1;
    }
    TriArgs A;
    A.start = track_start;
    A.rays = rays;
    A.cams = d_cams;
    A.n_tracks = n_tracks;
    A.min_views = prm.min_views;
    A.n_samples = prm.n_samples;
    A.refine_iters = prm.refine_iters;
    A.seed = prm.seed;
    A.thr2 = (double)prm.max_error * (double)prm.max_error;
    A.cos_min = std::cos((double)prm.min_angle * (3.141592653589793 / 180.0));
    A.points = points;
    A.mask = obs_mask;
    A.err = obs_error;
    tri_track_kernel<<<blocks_for(n_tracks, kTrackWarps), kTrackWarps * 32, 0, st>>>(A);
    const unsigned nc = std::min<unsigned>(blocks_for(n_tracks, kCountThreads), 4u * (unsigned)sm_count());
    tri_count_kernel<<<nc, kCountThreads, 0, st>>>(points, n_tracks, stat);
    if (!read_back(&h, stat, sizeof(TriStat), st)) return ws.fail("triangulate: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    std::memcpy(counts->n_status, h.n_status, sizeof(counts->n_status));
    counts->n_inlier_obs = h.n_inlier_obs;
    return 4;
}

} // namespace psb
