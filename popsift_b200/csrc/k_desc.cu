// Stage 3b -- 128-D descriptors + normalisation + Feature records, hand-written for sm_90a.
//
// Replaces ext_desc_loop / ext_desc_loop_sub, normalize_histogram<RootSift|L2> and prep_features
// (reference src/popsift/s_desc_loop.cu:11-158, s_desc_norm_rs.h:41-77, s_desc_norm_l2.h:46-135,
// s_desc_normalize.h:14-33, sift_pyramid.cu:250-280).  Structure:
//   * one launch for all octaves; a fixed grid of warps pulls descriptors from a device-side work
//     counter (the reference reads the count back to the host, sift_desc.cu:55-110);
//   * ONE small CTA (4 warps) per descriptor visits every pixel of the rotated 5x5-SBP support once: gradient,
//     Gaussian weight and orientation split are computed once per pixel and scattered to the (at
//     most) 2x2 cells whose bilinear windows cover it.  The reference runs 16 warps per descriptor,
//     each scanning its own cell's bounding box: ~2.6x redundant atan2f/hypotf and mostly-idle
//     lanes; this form issues ~9x fewer instructions;
//   * the 128 bins live in shared memory (one 512-byte histogram per warp); normalisation is fused
//     and the descriptor leaves with one float4 per lane -- one launch and one HBM round trip less,
//     and without the reference's last-descriptor race (SURVEY 8a quirk 1).
// Per-sample math uses the task's descriptor tolerance (normalised descriptors within 1e-3 L2 of the reference's;
// measured <= 2e-4 on make_frame content and <= 8e-4 on the full-contrast and saturated images of tests/stress_images.py): atan2 is one rcp.approx + a degree-6 minimax polynomial (< 1e-6 rad), the gradient magnitude
// sqrt.approx, the Gaussian weight ex2.approx, floor / float -> fixed conversions are magic-number adds instead of the
// conversion pipe, and the 128 bins are accumulated as order-independent 32-bit fixed-point shared-memory adds (the
// reference: per-lane round-up float sums and a shuffle tree) -- run-to-run deterministic descriptors.  Only
// __sincosf of the keypoint angle and the normalisation (fused below) keep the reference's intrinsics.
#include "ps_internal.h"
#include "k_desc_norm.h"

namespace psb {

namespace {

__device__ const float dPi2 = 2.0f * 3.14159265358979323846f;
__device__ const float d4RPi = 4.0f / 3.14159265358979323846f;

__device__ __forceinline__ float plane_at(const float* pl, int w, int h, int pitch, int x, int y)
{
    x = min(max(x, 0), w - 1);
    y = min(max(y, 0), h - 1);
    return __ldg(pl + (size_t)y * pitch + x);
}

constexpr int DWARPS = 4;     // warps that share one descriptor (one CTA per descriptor in flight); == histogram copies
constexpr int DTHREADS = DWARPS * 32;
// a bin can reach ~8e4 (232 fully weighted pixels of gradient magnitude 360): 17 integer bits; one
// contribution stays below 360 * 2^14 < 2^23, so float -> fixed point is a single FFMA onto 2^23.
// Known limit: the scale is fixed by the top of the range, so on low-contrast content a contribution is a few units
// and its rounding, through RootSift's square root, shows in nearly empty bins.  On a 0..3 grey-level image RootSift
// descriptors are up to 5e-3 L2 from the oracle and 4.4e-3 from the reference (median 8e-4); classic normalisation
// stays within 1e-3.  A second, finer pass for descriptors whose largest weighted gradient is below one grey level
// brings that to 1.5e-4 but cost 1.8 % of bench.py's time per frame (H100, 400 W), so it is not done.
__device__ const float kFix = 16384.0f;
__device__ const float kUnfix = 1.0f / 16384.0f;
__device__ const float kMagic = 8388608.0f;      // 2^23

// atan2 to < 1e-6 rad (tests/test_host_cpu.py): one reciprocal, a degree-6 minimax polynomial in a^2 on [0,1] and three
// selects (atan2f is ~40 instructions).  The orientation only feeds a linear interpolation between
// two bins, so the error moves a normalised descriptor by < 1e-6.
__device__ __forceinline__ float fast_rcp(float v) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
__device__ __forceinline__ float fast_ex2(float v) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }

__device__ __forceinline__ float fast_atan2(float y, float x)
{
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    // dark regions hold denormal gradients: rcp.ftz would turn them into inf (and 0 * inf into NaN);
    // their magnitude is ~0, so the angle is irrelevant
    const float a = mx > 1e-30f ? mn * fast_rcp(mx) : 0.0f;
    const float s = a * a;
    float p = 0.006811764091253281f;
    p = fmaf(p, s, -0.03360414132475853f);
    p = fmaf(p, s, 0.07962359488010406f);
    p = fmaf(p, s, -0.1323333978652954f);
    p = fmaf(p, s, 0.19807815551757812f);
    p = fmaf(p, s, -0.3331736922264099f);
    p = fmaf(p, s, 0.9999961256980896f);
    float r = p * a;
    if (ay > ax) r = 1.57079632679489662f - r;
    if (x < 0.0f) r = 3.14159265358979323846f - r;
    return copysignf(r, y);
}

// floor(v) for |v| < 2^22 without the conversion pipe: v + 1.5 * 2^23 rounded down keeps floor(v) (two's
// complement) in the low mantissa bits; floor_val turns the same float back into floor(v)
__device__ const float kMagicS = 12582912.0f;    // 1.5 * 2^23
__device__ __forceinline__ unsigned floor_bits(float v) { return __float_as_uint(__fadd_rd(v, kMagicS)); }
__device__ __forceinline__ float floor_val(unsigned bits) { return __fsub_rn(__uint_as_float(bits), kMagicS); }
// round(w * c) for 0 <= w*c < 2^23 (fixed-point contribution)
__device__ __forceinline__ unsigned fix_bits(float w, float c) { return __float_as_uint(__fmaf_rn(w, c, kMagic)) & 0x7fffffu; }

__device__ __forceinline__ float fast_sqrt(float v) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }

__global__ void __launch_bounds__(DTHREADS)
descriptor_kernel(PyramidView pyr, Consts k, const ps_extremum* __restrict__ ext,
                  const int* __restrict__ feat_to_ext, ps_descriptor* __restrict__ desc, Counters* ct)
{
    // 128 bins in 32-bit fixed point (15 fractional bits): integer shared-memory atomics are
    // native (ATOMS.ADD) whereas float ones are compare-and-swap loops, and integer sums do not depend
    // on the order of the adds -> run-to-run deterministic descriptors
    // kCopies copies of the histogram, selected by lane % kCopies and skewed by 8 banks each: neighbouring
    // lanes that add to the same (cell, bin) -- the common case along a row of samples -- hit different
    // banks instead of serialising on one word; the copies are summed before normalisation
    // kCopies = 8: the 8 lanes of a band (consecutive pixels of one row: usually the same cell and often the same bin)
    // each add to their own copy, and the copies start 4 banks apart; lanes 8 apart share a copy but work in different
    // bands = distant rows = other cells.
    // Every copy is a 6 x 6 grid of cells: the 4 x 4 descriptor cells plus a guard ring, so that the 2 x 2 cells a sample
    // spreads over always exist and its eight adds need no range checks, no predicates and no branches (the four
    // conditional blocks of the 4 x 4 form diverged in almost every warp, so all four bodies ran anyway); the ring is
    // simply not read back.
    constexpr int kCopies = 8, kRing = 6, kHStride = kRing * kRing * 8 + 4;
    __shared__ __align__(16) unsigned H[kCopies * kHStride];
    __shared__ int next_d;
    // per row of the support: x = candidates before the row (exclusive prefix), y = first column - x
    __shared__ int2 row_tab[DTHREADS + 1];
    __shared__ int warp_sum[DWARPS];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int total = ct->ori_total;

    for (;;) {
        // dynamic distribution: descriptor sizes vary by two orders of magnitude with scale
        if (threadIdx.x == 0) next_d = atomicAdd(&ct->work_desc, 1);
        __syncthreads();
        const int d = next_d;
        if (d >= total) break;

        const int ei = feat_to_ext[d];
        const ps_extremum e = ext[ei];
        const float ang = e.orientation[min(max(d - e.idx_ori, 0), PS_MAX_ORI - 1)];
        const OctaveView& ov = pyr.oct[e.octave];
        const int width = ov.w, height = ov.h, pitch = ov.pitch;
        const long long pitch_l = pitch;
        const int lvl = min(max(e.lpos, 0), pyr.levels + 2);
        const float* pl = ov.gauss + (size_t)lvl * ov.plane;

        for (int i = threadIdx.x; i < kCopies * kHStride / 4; i += DTHREADS)
            reinterpret_cast<uint4*>(H)[i] = make_uint4(0u, 0u, 0u, 0u);

        const float x = e.xpos, y = e.ypos;
        const float SBP = fabsf(__fmul_rn(3.0f, e.sigma));
        if (SBP != 0.0f) {
            float sin_t, cos_t;
            __sincosf(ang, &sin_t, &cos_t);
            const float csbp = __fmul_rn(cos_t, SBP), ssbp = __fmul_rn(sin_t, SBP);
            const float crsbp = __fdiv_rn(cos_t, SBP), srsbp = __fdiv_rn(sin_t, SBP);
            // union of the 16 cell windows: |r| < 2.5 in units of SBP, r = R(-ang) (p - keypoint) / SBP
            const float half = __fmul_rn(2.5f, __fadd_rn(fabsf(csbp), fabsf(ssbp)));
            const int xmin = max(1, (int)floorf(x - half) - 1);
            const int ymin = max(1, (int)floorf(y - half) - 1);
            const int xmax = min(width - 2, (int)floorf(x + half) + 1);
            const int ymax = min(height - 2, (int)floorf(y + half) + 1);
            const int hy = ymax - ymin + 1;
            // The support is a rotated square; only ~half of its bounding box lies inside.  Each row's
            // candidate interval [lo, hi] is bounded from the two slabs |rx| < 2.5, |ry| < 2.5 (one pixel
            // of slack; the exact test stays in the sample loop), the candidates of up to DTHREADS rows are
            // numbered with a prefix sum and handed out round-robin, so lanes only visit pixels that are
            // (almost always) inside.
            const float inv_c = 1.0f / crsbp, inv_s = 1.0f / srsbp;     // +-inf when the support is axis-aligned
            for (int rb = 0; rb < hy; rb += DTHREADS) {
                const int r = rb + threadIdx.x;
                int lo = xmin, hi = xmax;
                if (r < hy) {
                    const float ddy = (float)(ymin + r) - y;
                    // |crsbp*ddx + srsbp*ddy| < 2.5
                    if (fabsf(crsbp) > 1e-6f) {
                        const float u0 = (-2.5f - srsbp * ddy) * inv_c, u1 = (2.5f - srsbp * ddy) * inv_c;
                        lo = max(lo, (int)floorf(fmaxf(x + fminf(u0, u1), -1e6f)) - 1);
                        hi = min(hi, (int)floorf(fminf(x + fmaxf(u0, u1), 1e6f)) + 2);
                    }
                    // |crsbp*ddy - srsbp*ddx| < 2.5
                    if (fabsf(srsbp) > 1e-6f) {
                        const float v0 = (crsbp * ddy - 2.5f) * inv_s, v1 = (crsbp * ddy + 2.5f) * inv_s;
                        lo = max(lo, (int)floorf(fmaxf(x + fminf(v0, v1), -1e6f)) - 1);
                        hi = min(hi, (int)floorf(fminf(x + fmaxf(v0, v1), 1e6f)) + 2);
                    }
                }
                const int cnt = (r < hy && hi >= lo) ? hi - lo + 1 : 0;
                int inc = cnt;                                   // inclusive scan over the CTA
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += t;
                }
                if (lane == 31) warp_sum[warp] = inc;
                __syncthreads();                                 // also orders the reset of H / previous pass
                int base = 0;
#pragma unroll
                for (int wq = 0; wq < DWARPS; ++wq) if (wq < warp) base += warp_sum[wq];
                row_tab[threadIdx.x] = make_int2(base + inc - cnt, lo - (base + inc - cnt));
                if (threadIdx.x == DTHREADS - 1) row_tab[DTHREADS] = make_int2(base + inc, 0);
                __syncthreads();
                const int n = row_tab[DTHREADS].x;

                // Hand-out of the n candidates.  32 consecutive candidates are neighbours in a row: they fall
                // into the same cell and, where the image is smooth, the same orientation bin, so a warp that
                // took 32 consecutive ones serialised ~8 lanes per shared-memory atomic (ncu: 7.7 wavefronts
                // per ATOMS, LSU data pipe 81 % busy).  Instead the candidate list is cut into kBands bands
                // (distant rows -> different cells) and every group of 32/kBands lanes of a warp works in its own
                // band: still whole 32-byte sectors per group for the gradient loads.
                constexpr int kBands = 4, kTeam = DTHREADS / kBands;          // threads per band
                const int nq = (n + kBands - 1) / kBands;
                const int band = lane / (32 / kBands);
                const int band_end = min(n, (band + 1) * nq);
                int i = band * nq + warp * (32 / kBands) + (lane & (32 / kBands - 1));
                int row = 0, cur_off = 0, next_pre = 0;
                if (i < band_end) {
                    int lo = 0, hi = DTHREADS;                          // last row with row_tab[row].x <= i
                    while (hi - lo > 1) {
                        const int mid = (lo + hi) >> 1;
                        if (row_tab[mid].x <= i) lo = mid; else hi = mid;
                    }
                    row = lo; cur_off = row_tab[lo].y; next_pre = row_tab[lo + 1].x;
                }
                for (; i < band_end; i += kTeam) {
                    while (i >= next_pre) {
                        ++row;
                        cur_off = row_tab[row].y;
                        next_pre = row_tab[row + 1].x;
                    }
                    const int ii = ymin + rb + row;
                    const int jj = i + cur_off;
                    const float ddx = (float)jj - x, ddy = (float)ii - y;
                    const float rx = __fmaf_rn(crsbp, ddx, __fmul_rn(srsbp, ddy));
                    const float ry = __fmaf_rn(crsbp, ddy, __fmul_rn(-srsbp, ddx));
                    if (!(fabsf(rx) < 2.5f && fabsf(ry) < 2.5f)) continue;
                    const float* p = pl + (ii * pitch + jj);             // interior pixel: neighbours exist; a plane is < 2^31 floats
                    const float gdx = __fsub_rn(__ldg(p + 1), __ldg(p - 1));
                    const float gdy = __fsub_rn(__ldg(p + pitch_l), __ldg(p - pitch_l));
                    const float mod = fast_sqrt(__fmaf_rn(gdx, gdx, __fmul_rn(gdy, gdy)));
                    // exp(-(rx^2 + ry^2) / 8); the exponent stays above -2.3, no range handling needed
                    const float ww = fast_ex2(__fmul_rn(__fmaf_rn(ry, ry, __fmul_rn(rx, rx)), -0.125f * 1.4426950408889634f));
                    // orientation relative to the keypoint in bin units; any multiple of 8 bins is the same
                    // orientation, so the value is not wrapped: floor_bits keeps floor(tth) mod 8 in its low bits
                    const float tth = __fmul_rn(__fsub_rn(fast_atan2(gdy, gdx), ang), d4RPi);
                    const unsigned fb = floor_bits(tth);
                    const float do0 = __fsub_rn(tth, floor_val(fb));
                    const unsigned b0 = fb & 7u, b1 = (fb + 1u) & 7u;
                    const float wm = __fmul_rn(__fmul_rn(ww, mod), kFix);
                    const float w1 = __fmul_rn(do0, wm), w0 = __fsub_rn(wm, w1);
                    // the (at most) 2x2 cells whose bilinear window covers this pixel
                    // cell coordinates biased by one so that the floor trick sees a non-negative number
                    // (rx + 2.5 can round to exactly 5.0: clamped to the last float below, which keeps the guard column index at 5)
                    const float fx = fminf(__fadd_rn(rx, 2.5f), 4.99999952f), fy = fminf(__fadd_rn(ry, 2.5f), 4.99999952f);   // in [0, 5)
                    const unsigned bx = floor_bits(fx), by = floor_bits(fy);
                    const unsigned gx = bx & 7u, gy = by & 7u;                          // ring cell of the lower-left window: 0 .. 4
                    const float ax1 = __fsub_rn(fx, floor_val(bx));                     // in [0,1)
                    const float ay1 = __fsub_rn(fy, floor_val(by));
                    const float ax0 = __fsub_rn(1.0f, ax1), ay0 = __fsub_rn(1.0f, ay1);
                    unsigned* hb = H + (lane & (kCopies - 1)) * kHStride + (gy * kRing + gx) * 8;
                    const float c00 = __fmul_rn(ax0, ay0), c10 = __fmul_rn(ax1, ay0), c01 = __fmul_rn(ax0, ay1), c11 = __fmul_rn(ax1, ay1);
                    atomicAdd(hb + b0, fix_bits(w0, c00));
                    atomicAdd(hb + b1, fix_bits(w1, c00));
                    atomicAdd(hb + 8 + b0, fix_bits(w0, c10));
                    atomicAdd(hb + 8 + b1, fix_bits(w1, c10));
                    atomicAdd(hb + kRing * 8 + b0, fix_bits(w0, c01));
                    atomicAdd(hb + kRing * 8 + b1, fix_bits(w1, c01));
                    atomicAdd(hb + kRing * 8 + 8 + b0, fix_bits(w0, c11));
                    atomicAdd(hb + kRing * 8 + 8 + b1, fix_bits(w1, c11));
                }
                // the next pass (or the next descriptor) rewrites row_tab only after its own barrier
            }
        }
        __syncthreads();
        if (warp == 0) {
            // lane = (cell, half of its 8 bins); descriptor cell (cx, cy) is ring cell (cx + 1, cy + 1)
            const int cell = lane >> 1;
            const int hoff = (((cell >> 2) + 1) * kRing + (cell & 3) + 1) * 8 + (lane & 1) * 4;
            uint4 hv = *reinterpret_cast<const uint4*>(H + hoff);
#pragma unroll
            for (int c = 1; c < kCopies; ++c) {
                const uint4 t = *reinterpret_cast<const uint4*>(H + c * kHStride + hoff);
                hv.x += t.x; hv.y += t.y; hv.z += t.z; hv.w += t.w;
            }
            float4 v = make_float4((float)hv.x * kUnfix, (float)hv.y * kUnfix, (float)hv.z * kUnfix, (float)hv.w * kUnfix);
            v = normalize_descriptor(v, lane, k.norm_mode, k.norm_multi);
            reinterpret_cast<float4*>(desc[d].features)[lane] = v;
        }
        // the next iteration's first __syncthreads orders this read of H before the next reset
    }
}

// Extremum -> user-facing Feature (octave-local -> input-image coordinates); desc[] pointers are
// filled in on the host by ps_download.
__global__ void prep_features_kernel(Consts k, const ps_extremum* __restrict__ ext, ps_feature* __restrict__ feat,
                                     const Counters* ct)
{
    const int total = ct->ext_total;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const ps_extremum e = ext[i];
        const float s = powf(2.0f, (float)(e.octave - k.up_fac));
        ps_feature f;
        f.debug_octave = e.octave;
        f.xpos = __fmul_rn(e.xpos, s);
        f.ypos = __fmul_rn(e.ypos, s);
        f.sigma = __fmul_rn(e.sigma, s);
        f.num_ori = e.num_ori;
        f.pad_ = e.idx_ori;          // first descriptor index; ps_download turns it into pointers
#pragma unroll
        for (int r = 0; r < PS_MAX_ORI; ++r) {
            f.orientation[r] = r < e.num_ori ? e.orientation[r] : 0.0f;
            f.desc[r] = nullptr;
        }
        feat[i] = f;
    }
}

// ps_download_dev: the copied Feature records get device pointers into the copied descriptor array
// (the reference's prep_features does this for its device clone, sift_pyramid.cu:324-330)
__global__ void fix_feature_pointers_kernel(ps_feature* __restrict__ feat, ps_descriptor* __restrict__ desc, int n)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int first = feat[i].pad_;
        const int num = feat[i].num_ori;
        feat[i].pad_ = 0;
#pragma unroll
        for (int r = 0; r < PS_MAX_ORI; ++r) feat[i].desc[r] = r < num ? desc + first + r : nullptr;
    }
}

} // namespace

int launch_fix_feature_pointers(ps_feature* feat, ps_descriptor* desc, int n, cudaStream_t st)
{
    if (n <= 0) return 0;
    fix_feature_pointers_kernel<<<(n + 255) / 256, 256, 0, st>>>(feat, desc, n);
    return 1;
}

int launch_descriptors(const PyramidView& pyr, const Consts& k, const ps_extremum* ext, const int* feat_to_ext,
                       ps_descriptor* desc, Counters* ct, cudaStream_t st)
{
    descriptor_kernel<<<sm_count() * 16, DTHREADS, 0, st>>>(pyr, k, ext, feat_to_ext, desc, ct);
    return 1;
}

int launch_prep_features(const Consts& k, const ps_extremum* ext, ps_feature* feat, const Counters* ct, cudaStream_t st)
{
    prep_features_kernel<<<sm_count(), 256, 0, st>>>(k, ext, feat, ct);
    return 1;
}

} // namespace psb
