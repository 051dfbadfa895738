// Two-view configuration, hand-written for sm_90a: ps_two_view_config_batch (contract in include/popsift_b200_twoview.h).
// The calibration, the SVD, the cheirality rule, E and F are ps_relative_pose_batch's (k_pose_solve.h), the block sums
// ps_verify_batch's (k_verify_common.h); the math of this stage is in k_twoview.h.
//
// One workspace (workspace.h), all launches on one stream:
//   1. tv_config_kernel  one CTA per pair, up to four sweeps over the pair's rows (they stay in L2 between sweeps):
//                          a. n_h, the Kabsch sum B and the sign count of the calibrated homography;
//                          b. (planar or panoramic) the rotation test under R0;
//                          c. (planar) the cheirality counts of the two kept (R, t, n);
//                          d. the outputs: record, mask, points, each bit-1 row's angle bits, and the pair's info.
//                        Thread 0 runs the 3 x 3 solves between the sweeps.
//   2. tv_median_kernel  one CTA per pair: the lower median of the angles by radix select, four 8-bit histogram passes
//                        in shared memory with integer atomics (exact, so deterministic).
// Then one read-back of the info records.
#include "k_twoview.h"
#include "k_verify_common.h"
#include "popsift_b200_twoview.h"
#include "ps_internal.h"
#include "workspace.h"

#include <algorithm>
#include <vector>

namespace psb {

static_assert(kTvDegenerate == PS_TV_DEGENERATE && kTvGeneral == PS_TV_GENERAL && kTvPlanar == PS_TV_PLANAR &&
              kTvPanoramic == PS_TV_PANORAMIC && kTvUncalibrated == PS_TV_UNCALIBRATED, "k_twoview.h's configurations");
static_assert(sizeof(ps_two_view_config_params) == 32 && sizeof(ps_two_view_info) == 40, "header layouts");

namespace {

constexpr int kTvThreads = 256;
constexpr uint32_t kNoAngle = 0xffffffffu;     // angle bits of a row without one (above every non-negative float)

struct TvParams { int min_inliers, pad; double thr2, min_ef_ratio, max_h_ratio, min_rotation_ratio; };

__global__ void __launch_bounds__(kTvThreads) tv_config_kernel(const VPair* __restrict__ pairs, const PCam* __restrict__ cams,
                                                               const float4* __restrict__ corr, const ps_two_view* __restrict__ ess,
                                                               const uint8_t* __restrict__ emask, const int32_t* __restrict__ f_inl,
                                                               const float* __restrict__ hom, const uint8_t* __restrict__ hmask,
                                                               TvParams prm, ps_two_view* __restrict__ out, uint8_t* __restrict__ out_mask,
                                                               float4* __restrict__ out_pts, uint32_t* __restrict__ angle_bits,
                                                               ps_two_view_info* __restrict__ info)
{
    __shared__ int red_i[33];
    __shared__ double red_d[33];
    __shared__ double sHc[9], sR0[9], cR[2][9], ct[2][3], cn[2][3];
    __shared__ int s_cfg, s_nc, s_r0ok;
    __shared__ ps_two_view res;
    const int p = blockIdx.x;
    const VPair P = pairs[p];
    const PCam K = cams[p];
    const float4* q = corr + P.start;
    const uint8_t* hm = hmask + P.start;
    const int n_e = ess[p].n_inliers, n_f = f_inl[p];
    if (threadIdx.x == 0) {
        double H[9];
        for (int j = 0; j < 9; ++j) H[j] = hom[9 * p + j];
        tv_h_calibrated(H, K, sHc);
        s_r0ok = 0;
        s_nc = 0;
    }
    __syncthreads();
    // a. n_h, B and the sign count
    double B[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) B[j] = 0.0;
    int nh = 0, npos = 0;
    for (int i = threadIdx.x; i < P.n; i += kTvThreads) {
        if (!hm[i]) continue;
        const float4 v = q[i];
        float c[4];
        pose_calibrate(K, v.x, v.y, v.z, v.w, c);
        double a[3], b[3];
        tv_ray(c[0], c[1], a);
        tv_ray(c[2], c[3], b);
        tv_outer_acc(b, a, B);
        npos += tv_h_side(sHc, c[0], c[1], c[2], c[3]) > 0.0 ? 1 : 0;
        ++nh;
    }
    const int n_h = block_sum_i(nh, red_i);
    int cfg = tv_classify(n_e, n_f, n_h, prm.min_inliers, prm.min_ef_ratio, prm.max_h_ratio);
    int n_rot = 0;
    if (cfg == kTvPlanar) {
        npos = block_sum_i(npos, red_i);
        double Bs[9];
#pragma unroll
        for (int j = 0; j < 9; ++j) Bs[j] = block_sum_d(B[j], red_d);
        if (threadIdx.x == 0) {
            s_r0ok = tv_kabsch(Bs, sR0) ? 1 : 0;
            if (!s_r0ok)
                for (int j = 0; j < 9; ++j) sR0[j] = 0.0;
        }
        __syncthreads();
        // b. the rotation test
        int nr = 0;
        if (s_r0ok)
            for (int i = threadIdx.x; i < P.n; i += kTvThreads) {
                if (!hm[i]) continue;
                const float4 v = q[i];
                float c[4];
                pose_calibrate(K, v.x, v.y, v.z, v.w, c);
                nr += tv_rotation_ok(sR0, K, c[0], c[1], v.z, v.w, prm.thr2) ? 1 : 0;
            }
        n_rot = block_sum_i(nr, red_i);
        if ((double)n_rot >= prm.min_rotation_ratio * (double)n_h) {
            cfg = kTvPanoramic;
        } else {
            if (threadIdx.x == 0) {
                // 4. the homography's (R, t, n): normalise, sign, decompose, prune
                double Hn[9], R[4][9], t[4][3], n[4][3];
                int nd = -1, keep[4], nk = 0;
                bool finite = true;
                for (int j = 0; j < 9; ++j) finite = finite && isfinite(sHc[j]);
                if (finite && tv_h_normalise(sHc, Hn)) {
                    if (2 * npos < n_h)
                        for (int j = 0; j < 9; ++j) Hn[j] = -Hn[j];
                    nd = tv_h_decompose(Hn, R, t, n);
                }
                if (nd > 0) nk = tv_prune(n, keep);
                int c = 0;
                for (int k = 0; k < nk && c < 2; ++k) {
                    const int j = keep[k];
                    double u[3] = {t[j][0], t[j][1], t[j][2]};
                    if (!pose_unit(u)) continue;
                    for (int e = 0; e < 9; ++e) cR[c][e] = R[j][e];
                    for (int e = 0; e < 3; ++e) { ct[c][e] = u[e]; cn[c][e] = n[j][e]; }
                    ++c;
                }
                s_nc = c;
                s_cfg = nd == 0 ? kTvPanoramic
                                : c > 0 ? kTvPlanar : tv_classify(n_e, n_f, n_h, prm.min_inliers, prm.min_ef_ratio, prm.max_h_ratio, false);
            }
            __syncthreads();
            cfg = s_cfg;
        }
    }
    // c. cheirality of the kept candidates
    int best = 0;
    if (cfg == kTvPlanar) {
        const int nc = s_nc;
        int f[2] = {0, 0};
        for (int i = threadIdx.x; i < P.n; i += kTvThreads) {
            if (!hm[i]) continue;
            const float4 v = q[i];
            float c[4];
            pose_calibrate(K, v.x, v.y, v.z, v.w, c);
            for (int k = 0; k < nc; ++k) f[k] += pose_front(cR[k], ct[k], c[0], c[1], c[2], c[3]) ? 1 : 0;
        }
        int bf = -1;
        for (int k = 0; k < nc; ++k) {
            const int s = block_sum_i(f[k], red_i);
            if (s > bf) { bf = s; best = k; }
        }
    }
    if (threadIdx.x == 0) {
        if (cfg == kTvGeneral) {
            res = ess[p];
        } else {
            for (int j = 0; j < (int)(sizeof(ps_two_view) / 4); ++j) reinterpret_cast<int32_t*>(&res)[j] = 0;
            if (cfg == kTvPlanar) {
                double R[9], t[3], E[9], F[9];
                for (int j = 0; j < 9; ++j) { res.R[j] = (float)cR[best][j]; R[j] = res.R[j]; }
                for (int j = 0; j < 3; ++j) { res.t[j] = (float)ct[best][j]; t[j] = res.t[j]; }
                pose_essential(R, t, E);
                for (int j = 0; j < 9; ++j) res.E[j] = (float)E[j];
                pose_pixels(E, K, F);
                for (int j = 0; j < 9; ++j) res.F[j] = (float)F[j];
            } else if (cfg == kTvPanoramic) {
                for (int j = 0; j < 9; ++j) res.R[j] = (float)sR0[j];
            }
        }
    }
    __syncthreads();
    // d. the outputs
    double Ro[9], to[3];
#pragma unroll
    for (int j = 0; j < 9; ++j) Ro[j] = res.R[j];
#pragma unroll
    for (int j = 0; j < 3; ++j) to[j] = res.t[j];
    const bool rot_ok = s_r0ok != 0;
    int ni = 0, nf = 0;
    for (int i = threadIdx.x; i < P.n; i += kTvThreads) {
        const float4 v = q[i];
        float c[4];
        pose_calibrate(K, v.x, v.y, v.z, v.w, c);
        bool in = false, fr = false;
        double X[3];
        bool point = false;
        if (cfg == kTvGeneral) {
            // the mask byte as it is; the points of the bit-1 rows by rule 8 (pose_front holds again: same rows, same R, t)
            const uint8_t m = emask[P.start + i];
            in = (m & 1) != 0;
            fr = (m & 2) != 0;
            point = fr && pose_front(Ro, to, c[0], c[1], c[2], c[3], X);
        } else if (cfg == kTvPlanar) {
            in = hm[i] != 0;
            fr = in && pose_front(Ro, to, c[0], c[1], c[2], c[3], X);
            point = fr;
        } else if (cfg == kTvPanoramic) {
            in = hm[i] != 0;
            fr = in && rot_ok && tv_rotation_ok(sR0, K, c[0], c[1], v.z, v.w, prm.thr2);
        }
        out_mask[P.start + i] = (uint8_t)((in ? 1 : 0) | (fr ? 2 : 0));
        if (out_pts) out_pts[P.start + i] = point ? make_float4((float)X[0], (float)X[1], (float)X[2], 1.0f) : make_float4(0.f, 0.f, 0.f, 0.f);
        angle_bits[P.start + i] = point ? __float_as_uint((float)tv_angle(X, Ro, to)) : kNoAngle;
        ni += in ? 1 : 0;
        nf += fr ? 1 : 0;
    }
    ni = block_sum_i(ni, red_i);
    nf = block_sum_i(nf, red_i);
    if (threadIdx.x == 0) {
        if (cfg == kTvPlanar || cfg == kTvPanoramic) {
            res.n_inliers = ni;
            res.n_front = nf;
        }
        out[p] = res;
        ps_two_view_info r;
        r.config = cfg;
        r.n_e = n_e; r.n_f = n_f; r.n_h = n_h;
        r.n_rotation = n_rot;
        r.tri_angle = 0.0f;
        for (int j = 0; j < 3; ++j) r.normal[j] = cfg == kTvPlanar ? (float)cn[best][j] : 0.0f;
        r.pad_ = 0;
        info[p] = r;
    }
}

// the lower median (rank floor((k - 1) / 2)) of the pair's k angle bit patterns that are not kNoAngle, by four 8-bit
// radix passes, most significant byte first
__global__ void __launch_bounds__(kTvThreads) tv_median_kernel(const VPair* __restrict__ pairs, const uint32_t* __restrict__ angle_bits,
                                                               ps_two_view_info* __restrict__ info)
{
    __shared__ int red_i[33];
    __shared__ unsigned hist[256];
    __shared__ uint32_t s_prefix;
    __shared__ int s_rank;
    const VPair P = pairs[blockIdx.x];
    const uint32_t* a = angle_bits + P.start;
    int k = 0;
    for (int i = threadIdx.x; i < P.n; i += kTvThreads) k += a[i] != kNoAngle ? 1 : 0;
    k = block_sum_i(k, red_i);
    if (k == 0) return;                 // tri_angle stays 0
    if (threadIdx.x == 0) { s_prefix = 0; s_rank = (k - 1) / 2; }
    for (int shift = 24; shift >= 0; shift -= 8) {
        hist[threadIdx.x] = 0;          // kTvThreads == 256 bins
        __syncthreads();
        const uint32_t hi = shift == 24 ? 0u : 0xffffffffu << (shift + 8);
        const uint32_t pre = s_prefix & hi;
        for (int i = threadIdx.x; i < P.n; i += kTvThreads) {
            const uint32_t b = a[i];
            if (b != kNoAngle && (b & hi) == pre) atomicAdd(&hist[(b >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int cum = 0;
            for (int d = 0; d < 256; ++d) {
                if (s_rank < cum + (int)hist[d]) {
                    s_prefix |= (uint32_t)d << shift;
                    s_rank -= cum;
                    break;
                }
                cum += (int)hist[d];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) info[blockIdx.x].tri_angle = __uint_as_float(s_prefix);
}
static_assert(kTvThreads == 256, "tv_median_kernel: one histogram bin per thread");

} // namespace

int run_two_view_config_batch(int n_pairs, const float* corr, const int32_t* corr_start, const int32_t* n_corr, const ps_camera* cams,
                              const ps_two_view* d_essential, const uint8_t* d_essential_mask, const int32_t* d_f_inliers,
                              const float* d_homography, const uint8_t* d_h_mask, const ps_two_view_config_params& prm,
                              ps_two_view* d_out, uint8_t* d_out_mask, float* d_points, ps_two_view_info* info, cudaStream_t st,
                              const char** err)
{
    *err = nullptr;
    long long total_rows = 0;
    std::vector<VPair> vp(n_pairs);
    std::vector<PCam> pc(n_pairs);
    for (int p = 0; p < n_pairs; ++p) {
        total_rows = std::max(total_rows, (long long)corr_start[p] + n_corr[p]);
        vp[p] = {corr_start[p], n_corr[p], 0};
        pc[p] = pose_cam(cams[2 * p], cams[2 * p + 1], prm.threshold);
    }
    Workspace ws(st, "cudaMallocFromPoolAsync failed (two-view configuration)", "two-view configuration: plan upload failed");
    const size_t o_pairs = ws.put(vp.data(), vp.size() * sizeof(VPair)), o_cams = ws.put(pc.data(), pc.size() * sizeof(PCam));
    const size_t o_info = ws.take((size_t)n_pairs * sizeof(ps_two_view_info));
    const size_t o_bits = ws.take((size_t)std::max(total_rows, 1ll) * sizeof(uint32_t));
    if (!ws.alloc(err)) return -1;
    const VPair* pairs = ws.at<const VPair>(o_pairs);
    ps_two_view_info* d_info = ws.at<ps_two_view_info>(o_info);
    uint32_t* bits = ws.at<uint32_t>(o_bits);
    const TvParams tp{prm.min_inliers, 0, (double)prm.threshold * (double)prm.threshold, prm.min_ef_ratio, prm.max_h_ratio,
                      prm.min_rotation_ratio};
    tv_config_kernel<<<n_pairs, kTvThreads, 0, st>>>(pairs, ws.at<const PCam>(o_cams), reinterpret_cast<const float4*>(corr), d_essential,
                                                     d_essential_mask, d_f_inliers, d_homography, d_h_mask, tp, d_out, d_out_mask,
                                                     reinterpret_cast<float4*>(d_points), bits, d_info);
    tv_median_kernel<<<n_pairs, kTvThreads, 0, st>>>(pairs, bits, d_info);
    if (!read_back(info, d_info, (size_t)n_pairs * sizeof(ps_two_view_info), st)) return ws.fail("two-view configuration: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return 2;
}

} // namespace psb
