// Describe path -- orientations and descriptors at caller-supplied keypoints (ps_describe_u8 / ps_describe_f32),
// hand-written for sm_90a.
//
// The reference has no such entry point.  Only the front of the tail is new; the orientation kernel, the descriptor
// kernels, the num_ori scan and prep_features are the extraction path's own, unchanged:
//   * kp_ingest_kernel validates each keypoint, derives or takes its octave and level, and maps it to octave-local
//     coordinates by the exact power of two 2^(up_fac - octave) that prep_features_kernel undoes;
//   * GIVEN: record i goes straight to ext[i] (input order) with the caller's angle;
//   * ORIENT: the valid keypoints are placed in per-octave InitialExtremum regions (warp-aggregated atomics, one per
//     octave present in a warp), the orientation kernel runs on them as if they were detected extrema, and
//     kp_restore_kernel writes its records back to input order.  The placement order within an octave does not reach
//     the output: every record is independent of the others and returns to its own index;
//   * kp_finish_kernel writes each keypoint's own x, y and sigma bits into its Feature, so that the caller gets back
//     exactly what it passed in, rejected and extreme keypoints included.
#include "ps_internal.h"

#include <algorithm>

namespace psb {

namespace {

constexpr int kThreads = 256;
constexpr int kSlice = PS_ORI_SLICE;

// 2^e for -126 <= e <= 127, exact
__device__ __forceinline__ float pow2i(int e) { return __int_as_float((127 + e) << 23); }

// octave, level and octave-local x, y, sigma of keypoint p; false if it is rejected (see ps_describe_u8)
__device__ __forceinline__ bool kp_place(const PyramidView& pyr, const Consts& k, const ps_keypoint& p, bool orient,
                                         int& o, int& lvl, float& xl, float& yl, float& sl)
{
    const int L = pyr.levels, no = pyr.num_octaves;
    if (!isfinite(p.xpos) || !isfinite(p.ypos) || !isfinite(p.sigma) || !(p.sigma > 0.0f)) return false;
    if (!orient && !isfinite(p.orientation)) return false;
    if (p.octave != -1 && (p.octave < 0 || p.octave >= no)) return false;
    if (p.level != -1 && (p.level < 0 || p.level > L + 2)) return false;
    // S = L * (log2 sigma + up_fac - log2 sigma0): the scale index the pyramid gives this sigma, counted from octave 0
    const float S = __fmul_rn((float)L, __fsub_rn(__fadd_rn(log2f(p.sigma), (float)k.up_fac), log2f(k.sigma0)));
    o = p.octave;
    if (o == -1) o = min(max((int)floorf(__fdiv_rn(__fsub_rn(S, 0.5f), (float)L)), 0), no - 1);
    lvl = p.level;
    if (lvl == -1) lvl = min(max((int)roundf(__fsub_rn(S, (float)(o * L))), 0), L + 2);
    const float sc = pow2i(k.up_fac - o);
    xl = __fmul_rn(p.xpos, sc);
    yl = __fmul_rn(p.ypos, sc);
    sl = __fmul_rn(p.sigma, sc);
    const OctaveView& ov = pyr.oct[o];
    return xl >= 0.0f && xl <= (float)(ov.w - 1) && yl >= 0.0f && yl <= (float)(ov.h - 1);
}

template <bool ORIENT>
__global__ void __launch_bounds__(kThreads)
kp_ingest_kernel(PyramidView pyr, Consts k, const ps_keypoint* __restrict__ kp, int n, ps_extremum* __restrict__ ext,
                 InitialExtremum* __restrict__ iext, int* __restrict__ src, int stride, int* __restrict__ slice_sum,
                 Counters* ct_ori, Counters* ct)
{
    const int lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0) ct->ext_ct[0] = n;
    // warp-uniform trip count: the warp collectives below need all 32 lanes
    for (long long i0 = (long long)blockIdx.x * kThreads; i0 < n; i0 += (long long)gridDim.x * kThreads) {
        const bool in = i0 + threadIdx.x < n;
        const int i = in ? (int)(i0 + threadIdx.x) : 0;
        int o = -1, lvl = 0;
        float xl = 0.0f, yl = 0.0f, sl = 0.0f;
        bool ok = false;
        ps_keypoint p{};
        if (in) {
            p = kp[i];
            ok = kp_place(pyr, k, p, ORIENT, o, lvl, xl, yl, sl);
        }
        ps_extremum e{};
        e.octave = -1;
        if (ORIENT) {
            const unsigned grp = __match_any_sync(0xffffffffu, ok ? o : -1);
            const int leader = __ffs(grp) - 1;
            int base = 0;
            if (ok && lane == leader) base = atomicAdd(&ct_ori->ext_ct[o], __popc(grp));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (ok) {
                const size_t at = (size_t)o * stride + base + __popc(grp & ((1u << lane) - 1u));
                InitialExtremum ie;
                ie.xpos = xl; ie.ypos = yl; ie.lpos = lvl; ie.sigma = sl;
                iext[at] = ie;
                src[at] = i;
            } else if (in) {
                ext[i] = e;
            }
        } else {
            if (ok) {
                e.xpos = xl; e.ypos = yl; e.lpos = lvl; e.sigma = sl;
                e.octave = o; e.num_ori = 1; e.orientation[0] = p.orientation;
            }
            if (in) ext[i] = e;
            // a warp lies inside one slice of the num_ori scan
            const int sum = __reduce_add_sync(0xffffffffu, ok ? 1 : 0);
            if (lane == 0 && sum) atomicAdd(&slice_sum[i / kSlice], sum);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
kp_restore_kernel(int num_octaves, const ps_extremum* __restrict__ ext_sorted, const int* __restrict__ src, int stride, int n,
                  ps_extremum* __restrict__ ext, int* __restrict__ slice_sum, const Counters* ct_ori)
{
    __shared__ int ps[kMaxOctaves + 1];
    if (threadIdx.x == 0) {
        int t = 0;
        for (int o = 0; o < num_octaves; ++o) { ps[o] = t; t += ct_ori->ext_ct[o]; }
        ps[num_octaves] = t;
    }
    __syncthreads();
    const int total = ps[num_octaves];
    for (long long item = (long long)blockIdx.x * kThreads + threadIdx.x; item < total; item += (long long)gridDim.x * kThreads) {
        int o = 0;
        while (o + 1 < num_octaves && item >= ps[o + 1]) ++o;
        const int i = src[(size_t)o * stride + (item - ps[o])];
        const ps_extremum e = ext_sorted[item];
        ext[i] = e;
        if (e.num_ori > 0) atomicAdd(&slice_sum[i / kSlice], e.num_ori);
    }
}

__global__ void __launch_bounds__(kThreads)
kp_finish_kernel(const ps_keypoint* __restrict__ kp, int n, ps_feature* __restrict__ feat)
{
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        feat[i].xpos = kp[i].xpos;
        feat[i].ypos = kp[i].ypos;
        feat[i].sigma = kp[i].sigma;
    }
}

int grid_for(long long n)
{
    return (int)std::max<long long>(1, std::min<long long>((n + kThreads - 1) / kThreads, (long long)sm_count() * 32));
}

} // namespace

int launch_kp_ingest(const PyramidView& pyr, const Consts& k, const ps_keypoint* kp, int n, bool orient, ps_extremum* ext,
                     InitialExtremum* iext, int* src, int stride, int* slice_sum, Counters* ct_ori, Counters* ct, cudaStream_t st)
{
    if (orient) kp_ingest_kernel<true><<<grid_for(n), kThreads, 0, st>>>(pyr, k, kp, n, ext, iext, src, stride, slice_sum, ct_ori, ct);
    else        kp_ingest_kernel<false><<<grid_for(n), kThreads, 0, st>>>(pyr, k, kp, n, ext, iext, src, stride, slice_sum, ct_ori, ct);
    return 1;
}

int launch_kp_restore(int num_octaves, const ps_extremum* ext_sorted, const int* src, int stride, int n, ps_extremum* ext,
                      int* slice_sum, const Counters* ct_ori, cudaStream_t st)
{
    kp_restore_kernel<<<grid_for(n), kThreads, 0, st>>>(num_octaves, ext_sorted, src, stride, n, ext, slice_sum, ct_ori);
    return 1;
}

int launch_kp_finish(const ps_keypoint* kp, int n, ps_feature* feat, cudaStream_t st)
{
    if (n <= 0) return 0;
    kp_finish_kernel<<<grid_for(n), kThreads, 0, st>>>(kp, n, feat);
    return 1;
}

} // namespace psb
