// Calibrated two-view geometry, hand-written for sm_90a: the batched five-point RANSAC, relative pose and triangulated
// inliers of ps_relative_pose_batch (contract in include/popsift_b200_pose.h).  The sample hash, the Sampson test, the
// scoring loop, the selection rule and the refit's normal matrix are ps_verify_batch's (k_verify_common.h); the
// calibrated math is in k_pose_solve.h.
//
// One workspace (workspace.h), all launches on one stream:
//   1. pose_calibrate_kernel  one CTA per pair: the calibrated float4 rows.
//   2. pose_solve_kernel      one lane per minimal sample, in double: the five-point solver; ten slots per sample, count
//                             0 (valid) or -1 (invalid).  The 5 x 9 and 10 x 20 eliminations are in local memory.
//   3. pose_compact_kernel    one CTA per pair: the valid slots' h in ascending order (warp ballots + a prefix over the
//                             warps) and their number, which is read back to plan the scoring.
//   4. pose_score_kernel      the hot path: work items (pair, 128 valid hypotheses, chunk of correspondences) through
//                             verify's tiled loop with the Sampson test, so no FP32 work goes to invalid slots.
//   5. pose_select_kernel     one CTA per pair: the winner, the refit and its projection onto the essential matrices, the
//                             SVD and the four (R, t), cheirality counts of all four in one pass, the outputs.
//   6. pose_taps_kernel       (taps only) every hypothesis's count and calibrated E.
#include "k_pose_solve.h"
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

struct PSolveItem { int pair, s0; };
struct PScoreItem { int pair, k0, c0, c1; };

constexpr int kCalThreads = 256;
constexpr int kPoseSolveThreads = 64;
constexpr int kCompactThreads = 256;
constexpr int kMinSample = 5;
constexpr int kMinRefit = 8;

__global__ void __launch_bounds__(kCalThreads) pose_calibrate_kernel(const VPair* __restrict__ pairs, const PCam* __restrict__ cams,
                                                                     const float4* __restrict__ corr, float4* __restrict__ pts)
{
    const VPair P = pairs[blockIdx.x];
    const PCam K = cams[blockIdx.x];
    for (int i = threadIdx.x; i < P.n; i += blockDim.x) {
        const float4 v = corr[P.start + i];
        float c[4];
        pose_calibrate(K, v.x, v.y, v.z, v.w, c);
        pts[P.start + i] = make_float4(c[0], c[1], c[2], c[3]);
    }
}

__global__ void __launch_bounds__(kPoseSolveThreads) pose_solve_kernel(const PSolveItem* __restrict__ items, const VPair* __restrict__ pairs,
                                                                       const float4* __restrict__ pts, int n_samples, uint64_t seed,
                                                                       float* __restrict__ models, int32_t* __restrict__ counts)
{
    const PSolveItem it = items[blockIdx.x];
    const int s = it.s0 + (int)threadIdx.x;
    if (s >= n_samples) return;
    const VPair P = pairs[it.pair];
    const size_t h0 = ((size_t)it.pair * n_samples + s) * kPoseSlots;
    uint32_t idx[kMinSample];
    const bool ok = P.n >= kMinSample && verify_sample<kMinSample>(seed, it.pair, s, (uint32_t)P.n, idx);
    int n = 0;
    double Es[kPoseSlots][9];
    if (ok) {
        double p[kMinSample][4];
#pragma unroll
        for (int j = 0; j < kMinSample; ++j) {
            const float4 v = pts[P.start + idx[j]];
            p[j][0] = v.x; p[j][1] = v.y; p[j][2] = v.z; p[j][3] = v.w;
        }
        n = pose_five_point(p, Es);
    }
    for (int j = 0; j < kPoseSlots; ++j) {
        if (j < n) {
            double e[9];
            pose_scale(Es[j], e);          // cannot fail: pose_five_point keeps only finite, non-zero E
            for (int k = 0; k < 9; ++k) models[9 * (h0 + j) + k] = (float)e[k];
        }
        counts[h0 + j] = j < n ? 0 : -1;
    }
}

// the valid slots of each pair in ascending h: dense[p * nh + k] = h, n_valid[p]
__global__ void __launch_bounds__(kCompactThreads) pose_compact_kernel(int nh, const int32_t* __restrict__ counts, int32_t* __restrict__ dense,
                                                                       int32_t* __restrict__ n_valid)
{
    __shared__ int warp_tot[kCompactThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t h0 = (size_t)blockIdx.x * nh;
    int base = 0;
    for (int i0 = 0; i0 < nh; i0 += kCompactThreads) {
        const int h = i0 + (int)threadIdx.x;
        const bool keep = h < nh && counts[h0 + h] >= 0;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_tot[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kCompactThreads / 32; ++w) {
            before += w < warp ? warp_tot[w] : 0;
            total += warp_tot[w];
        }
        if (keep) dense[h0 + base + before + __popc(bal & ((1u << lane) - 1u))] = h;
        base += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) n_valid[blockIdx.x] = base;
}

__global__ void __launch_bounds__(kScoreThreads) pose_score_kernel(const PScoreItem* __restrict__ items, const VPair* __restrict__ pairs,
                                                                   const PCam* __restrict__ cams, const float4* __restrict__ pts, int nh,
                                                                   const int32_t* __restrict__ dense, const int32_t* __restrict__ n_valid,
                                                                   const float* __restrict__ models, int32_t* __restrict__ counts)
{
    __shared__ __align__(128) float4 tile[2][kTile];
    __shared__ __align__(8) uint64_t bar[2];
    const PScoreItem it = items[blockIdx.x];
    const VPair P = pairs[it.pair];
    const float t2 = cams[it.pair].t2;
    const size_t h0 = (size_t)it.pair * nh;
    const int k = it.k0 + (int)threadIdx.x;
    const bool act = k < n_valid[it.pair];
    const int h = act ? dense[h0 + k] : 0;
    float m[1][9];
    int cnt[1] = {0};
#pragma unroll
    for (int e = 0; e < 9; ++e) m[0][e] = act ? models[9 * (h0 + h) + e] : 0.0f;
    score_tiles<PS_GEOM_FUNDAMENTAL, 1>(pts + P.start + it.c0, it.c1 - it.c0, m, t2, tile, bar, cnt);
    if (act && cnt[0]) atomicAdd(&counts[h0 + h], cnt[0]);
}

__global__ void pose_taps_kernel(const float* __restrict__ models, const int32_t* __restrict__ counts, long long n_hyp,
                                 int32_t* __restrict__ tap_counts, float* __restrict__ tap_models)
{
    const long long h = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_hyp) return;
    const int c = counts[h];
    tap_counts[h] = c;
    for (int e = 0; e < 9; ++e) tap_models[9 * h + e] = c >= 0 ? models[9 * h + e] : 0.0f;
}

__global__ void __launch_bounds__(kSelectThreads, 1) pose_select_kernel(const VPair* __restrict__ pairs, const PCam* __restrict__ cams,
                                                                     const float4* __restrict__ pts, int nh, int refine,
                                                                     const float* __restrict__ models, const int32_t* __restrict__ counts,
                                                                     ps_two_view* __restrict__ out, uint8_t* __restrict__ out_mask,
                                                                     float4* __restrict__ out_pts)
{
    constexpr int NW = kSelectThreads / 32;
    __shared__ int red_i[33];
    __shared__ int win_c[NW];
    __shared__ long long win_h[NW];
    __shared__ double Nsh[NW][45];
    __shared__ double A[81], V[81];
    __shared__ float model[9], refit[9];
    __shared__ double cR[4][9], ct[4][3];
    __shared__ int svd_ok;
    __shared__ ps_two_view res;
    const int p = blockIdx.x;
    const VPair P = pairs[p];
    const PCam K = cams[p];
    const float4* q = pts + P.start;
    const long long h0 = (long long)p * nh;
    int bc;
    long long bh;
    select_winner<NW>(counts + h0, nh, P.n >= kMinSample, win_c, win_h, bc, bh);
    if (bc >= 0) {
        if (threadIdx.x < 9) model[threadIdx.x] = models[9 * (h0 + bh) + threadIdx.x];
        __syncthreads();
    }
    float mw[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) mw[e] = bc >= 0 ? model[e] : 0.0f;
    if (bc >= 0 && refine && bc >= kMinRefit) {
        double r[9];
        refit_smallest<PS_GEOM_FUNDAMENTAL, NW>(mw, q, P.n, K.t2, Nsh, A, V, r);
        if (threadIdx.x == 0) {
            // the projection onto the essential matrices: U diag(1, 1, 0) V^T
            double U3[3][3], V3[3][3], e[9], s[9];
            const bool ok = pose_svd(r, U3, V3);
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) e[3 * a + b] = U3[0][a] * V3[0][b] + U3[1][a] * V3[1][b];
            if (!ok || !pose_scale(e, s))
                for (int j = 0; j < 9; ++j) s[j] = 0.0;
            for (int j = 0; j < 9; ++j) refit[j] = (float)s[j];
        }
        __syncthreads();
        float mr[9];
#pragma unroll
        for (int e = 0; e < 9; ++e) mr[e] = refit[e];
        int c = 0;
        for (int i = threadIdx.x; i < P.n; i += kSelectThreads) c += inlier_f(mr, q[i], K.t2) ? 1 : 0;
        const int rc = block_sum_i(c, red_i);
        if (rc >= bc) {
#pragma unroll
            for (int e = 0; e < 9; ++e) mw[e] = mr[e];
        }
    }
    // the four (R, t) of the selected E
    if (threadIdx.x == 0) {
        double e[9], U3[3][3], V3[3][3];
        for (int j = 0; j < 9; ++j) e[j] = mw[j];
        svd_ok = bc >= 0 && pose_svd(e, U3, V3);
        if (svd_ok) pose_candidates(U3, V3, cR, ct);
    }
    __syncthreads();
    if (!svd_ok) {
        // no valid hypothesis (or too few correspondences): everything zero
        for (int j = threadIdx.x; j < (int)(sizeof(ps_two_view) / 4); j += kSelectThreads) reinterpret_cast<int32_t*>(out + p)[j] = 0;
        for (int i = threadIdx.x; i < P.n; i += kSelectThreads) {
            out_mask[P.start + i] = 0;
            if (out_pts) out_pts[P.start + i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        return;
    }
    // cheirality of the four candidates in one pass over the inlier rows
    int f[4] = {0, 0, 0, 0};
    for (int i = threadIdx.x; i < P.n; i += kSelectThreads) {
        const float4 v = q[i];
        if (!inlier_f(mw, v, K.t2)) continue;
#pragma unroll
        for (int c = 0; c < 4; ++c) f[c] += pose_front(cR[c], ct[c], v.x, v.y, v.z, v.w) ? 1 : 0;
    }
    int best = 0, bf = -1;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int s = block_sum_i(f[c], red_i);
        if (s > bf) { bf = s; best = c; }
    }
    if (threadIdx.x == 0) {
        double R[9], t[3], E[9], F[9];
        for (int j = 0; j < 9; ++j) { res.R[j] = (float)cR[best][j]; R[j] = res.R[j]; }
        for (int j = 0; j < 3; ++j) { res.t[j] = (float)ct[best][j]; t[j] = res.t[j]; }
        pose_essential(R, t, E);
        for (int j = 0; j < 9; ++j) res.E[j] = (float)E[j];
        pose_pixels(E, K, F);
        for (int j = 0; j < 9; ++j) res.F[j] = (float)F[j];
    }
    __syncthreads();
    float eo[9];
    double Ro[9], to[3];
#pragma unroll
    for (int j = 0; j < 9; ++j) { eo[j] = res.E[j]; Ro[j] = res.R[j]; }
#pragma unroll
    for (int j = 0; j < 3; ++j) to[j] = res.t[j];
    int ni = 0, nf = 0;
    for (int i = threadIdx.x; i < P.n; i += kSelectThreads) {
        const float4 v = q[i];
        const bool in = inlier_f(eo, v, K.t2);
        double X[3];
        const bool fr = in && pose_front(Ro, to, v.x, v.y, v.z, v.w, X);
        out_mask[P.start + i] = (uint8_t)((in ? 1 : 0) | (fr ? 2 : 0));
        if (out_pts) out_pts[P.start + i] = fr ? make_float4((float)X[0], (float)X[1], (float)X[2], 1.0f) : make_float4(0.f, 0.f, 0.f, 0.f);
        ni += in ? 1 : 0;
        nf += fr ? 1 : 0;
    }
    ni = block_sum_i(ni, red_i);
    nf = block_sum_i(nf, red_i);
    if (threadIdx.x == 0) {
        res.n_inliers = ni;
        res.n_front = nf;
        out[p] = res;
    }
}

} // namespace

int run_relative_pose_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_camera* cams,
                            const ps_pose_params& prm, ps_two_view* d_out, uint8_t* d_mask, float* d_points, const ps_verify_taps* taps,
                            cudaStream_t st, const char** err)
{
    *err = nullptr;
    const int ns = prm.n_samples, nh = kPoseSlots * ns;
    long long total_rows = 0;
    std::vector<VPair> vp(n_pairs);
    std::vector<PCam> pc(n_pairs);
    std::vector<PSolveItem> solve;
    for (int p = 0; p < n_pairs; ++p) {
        total_rows = std::max(total_rows, (long long)corr_start[p] + n_corr[p]);
        vp[p] = {corr_start[p], n_corr[p], 0};
        pc[p] = pose_cam(cams[2 * p], cams[2 * p + 1], prm.threshold);
        for (int s0 = 0; s0 < ns; s0 += kPoseSolveThreads) solve.push_back({p, s0});
    }
    if (solve.size() > 0x7fffffffu) { *err = "ps_relative_pose_batch: too many work items"; return -1; }
    const size_t n_hyp = (size_t)n_pairs * nh;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (pose workspace)", "pose: plan upload failed");
    const size_t o_pairs = ws.put(vp.data(), vp.size() * sizeof(VPair)), o_cams = ws.put(pc.data(), pc.size() * sizeof(PCam));
    const size_t o_solve = ws.put(solve.data(), solve.size() * sizeof(PSolveItem));
    const size_t o_pts = ws.take((size_t)total_rows * sizeof(float4)), o_models = ws.take(n_hyp * 9 * sizeof(float));
    const size_t o_counts = ws.take(n_hyp * sizeof(int32_t)), o_dense = ws.take(n_hyp * sizeof(int32_t));
    const size_t o_nvalid = ws.take((size_t)n_pairs * sizeof(int32_t));
    if (!ws.alloc(err)) return -1;
    const VPair* d_pairs = ws.at<const VPair>(o_pairs);
    const PCam* d_cams = ws.at<const PCam>(o_cams);
    float4* d_pts = ws.at<float4>(o_pts);
    float* hyp_models = ws.at<float>(o_models);
    int32_t* hyp_counts = ws.at<int32_t>(o_counts);
    int32_t* d_dense = ws.at<int32_t>(o_dense);
    int32_t* d_nvalid = ws.at<int32_t>(o_nvalid);
    pose_calibrate_kernel<<<n_pairs, kCalThreads, 0, st>>>(d_pairs, d_cams, reinterpret_cast<const float4*>(corr), d_pts);
    pose_solve_kernel<<<(unsigned)solve.size(), kPoseSolveThreads, 0, st>>>(ws.at<const PSolveItem>(o_solve), d_pairs, d_pts,
                                                                            ns, prm.seed, hyp_models, hyp_counts);
    pose_compact_kernel<<<n_pairs, kCompactThreads, 0, st>>>(nh, hyp_counts, d_dense, d_nvalid);
    int launches = 3;
    // the scoring plan needs each pair's number of valid hypotheses
    std::vector<int32_t> nv(n_pairs);
    if (!read_back(nv.data(), d_nvalid, (size_t)n_pairs * sizeof(int32_t), st)) {
        *err = cudaGetErrorString(cudaGetLastError());
        return -1;
    }
    double work = 0.0;
    for (int p = 0; p < n_pairs; ++p)
        if (n_corr[p] >= kMinSample) work += (double)((nv[p] + kScoreThreads - 1) / kScoreThreads) * n_corr[p];
    // correspondences per score item: about 16 items per SM over the whole call, at least two tiles (as ps_verify_batch)
    const double per = std::ceil(work / (16.0 * sm_count()));
    const int chunk = (int)std::min<double>(1 << 30, std::max<double>(2 * kTile, std::ceil(per / kTile) * kTile));
    std::vector<PScoreItem> score;
    for (int p = 0; p < n_pairs; ++p) {
        if (n_corr[p] < kMinSample) continue;
        for (int c0 = 0; c0 < n_corr[p]; c0 += chunk)
            for (int k0 = 0; k0 < nv[p]; k0 += kScoreThreads)
                score.push_back({p, k0, c0, (int)std::min<long long>((long long)c0 + chunk, n_corr[p])});
    }
    if (score.size() > 0x7fffffffu) { *err = "ps_relative_pose_batch: too many work items"; return -1; }
    Workspace sws(st, "cudaMallocFromPoolAsync failed (pose score plan)", "pose: plan upload failed");
    if (!score.empty()) {
        const size_t o_score = sws.put(score.data(), score.size() * sizeof(PScoreItem));
        if (!sws.alloc(err)) return -1;
        pose_score_kernel<<<(unsigned)score.size(), kScoreThreads, 0, st>>>(sws.at<const PScoreItem>(o_score), d_pairs, d_cams, d_pts, nh,
                                                                            d_dense, d_nvalid, hyp_models, hyp_counts);
        ++launches;
    }
    pose_select_kernel<<<n_pairs, kSelectThreads, 0, st>>>(d_pairs, d_cams, d_pts, nh, prm.refine, hyp_models, hyp_counts, d_out, d_mask,
                                                           reinterpret_cast<float4*>(d_points));
    ++launches;
    if (taps) {
        pose_taps_kernel<<<(unsigned)((n_hyp + 255) / 256), 256, 0, st>>>(hyp_models, hyp_counts, (long long)n_hyp, taps->d_counts, taps->d_models);
        ++launches;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

} // namespace psb
