// Brute-force 2-nearest-neighbour descriptor matcher, hand-written for sm_90a (wgmma + TMA + mbarrier).
//
// Replaces FeaturesDev::match -> compute_distance (reference src/popsift/features.cu:165-227,282-304): for every
// left descriptor the best and second-best right descriptor by squared L2 distance and the ratio test
// best / second < 0.8.  The reference runs one 32-thread block per left descriptor and walks all right
// descriptors one by one (n_left x n_right x 128 scalar flops on CUDA cores, every right descriptor re-read
// n_left times).  This is the one dense contraction of the library:
//     |a - b|^2 = |a|^2 + |b|^2 - 2 a.b        ->   S = A . B^T  on the tensor cores.
//
// Pipeline (ps_match):
//   1. match_split_kernel     a = hi + lo with hi = tf32(a) (round to nearest), lo = a - hi; |b|^2 per right
//                             descriptor.  Three tf32 products hi.hi + hi.lo + lo.hi give a.b to ~2^-21 relative.
//   2. match_tc_kernel        one CTA (three warpgroups) per 128 left descriptors.  The A tile (hi and lo, 128 x 128
//                             floats each) is loaded once with TMA (SWIZZLE_128B, K-major) and stays in shared memory;
//                             the right descriptors stream through a 3-stage TMA ring of [128 descriptors x 32 floats]
//                             tiles (hi and lo).  Warpgroup 0 is the TMA producer (one thread); warpgroups 1 and 2 each
//                             own 64 left descriptors and issue wgmma.mma_async m64n128k8 tf32 into a register
//                             accumulator, then keep each of their rows' four best candidates |b|^2 - 2 a.b (a row's
//                             128 columns are spread over the four lanes of a quad, merged at the end).  The
//                             n_left x n_right distance matrix never touches HBM.
//   3. match_rerank_kernel    one warp per left descriptor recomputes the exact float32 distance of its four
//                             candidates in the reference's own evaluation order (per lane x*x, fma, fma, fma over its
//                             float4, shuffle-down tree 16, 8, 4, 2, 1) and applies the reference's scan rule
//                             (strict <, ties keep the lower index) and ratio test.
// The result equals the reference's except when three or more right descriptors lie within ~4e-6 (relative) of the second
// best (the candidate pass could then miss the reference's pick among exact near-ties).
// match_exact_kernel is the same computation on CUDA cores (one warp per left descriptor over all right ones): used
// for small problems and as the in-library cross-check (PS_MATCH_EXACT).
#include "ps_internal.h"
#include "tma_util.h"

#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace psb {

namespace {

// ------------------------------------------------------------------------------------------------ exact (CUDA cores)

// squared distance of the warp's left descriptor (lane holds l4) to right descriptor r, reference order
// (features.cu:165-185: per lane x*x + y*y + z*z + w*w -- SASS FMUL, FFMA, FFMA, FFMA -- then shuffle_down 16..1)
__device__ __forceinline__ float warp_sq_dist(const float4 l4, const float4* __restrict__ r, int lane)
{
    const float4 r4 = __ldg(r + lane);
    const float dx = __fsub_rn(l4.x, r4.x), dy = __fsub_rn(l4.y, r4.y), dz = __fsub_rn(l4.z, r4.z), dw = __fsub_rn(l4.w, r4.w);
    float res = __fmul_rn(dx, dx);
    res = __fmaf_rn(dy, dy, res);
    res = __fmaf_rn(dz, dz, res);
    res = __fmaf_rn(dw, dw, res);
    res = __fadd_rn(res, __shfl_down_sync(0xffffffffu, res, 16));
    res = __fadd_rn(res, __shfl_down_sync(0xffffffffu, res, 8));
    res = __fadd_rn(res, __shfl_down_sync(0xffffffffu, res, 4));
    res = __fadd_rn(res, __shfl_down_sync(0xffffffffu, res, 2));
    res = __fadd_rn(res, __shfl_down_sync(0xffffffffu, res, 1));
    return __shfl_sync(0xffffffffu, res, 0);
}

struct Best2 {
    float v1, v2; int i1, i2;
    __device__ __forceinline__ void init() { v1 = v2 = INFINITY; i1 = i2 = 0; }
    // the reference's scan step (features.cu:205-217); candidates must arrive in increasing index order
    __device__ __forceinline__ void step(float res, int i)
    {
        if (res < v1) { v2 = v1; i2 = i1; v1 = res; i1 = i; }
        else if (res < v2) { v2 = res; i2 = i; }
    }
    __device__ __forceinline__ void store(int32_t* out) const
    {
        out[0] = i1; out[1] = i2; out[2] = (__fdiv_rn(v1, v2) < 0.8f) ? 1 : 0;
    }
};

__global__ void __launch_bounds__(128)
match_exact_kernel(const ps_descriptor* __restrict__ l, int nl, const ps_descriptor* __restrict__ r, int nr, int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= nl) return;
    const float4 l4 = __ldg(reinterpret_cast<const float4*>(l + row) + lane);
    Best2 b; b.init();
    for (int i = 0; i < nr; ++i) b.step(warp_sq_dist(l4, reinterpret_cast<const float4*>(r + i), lane), i);
    if (lane == 0) b.store(out + 3 * (size_t)row);
}

// ------------------------------------------------------------------------------------------------ split / norms

__device__ __forceinline__ float to_tf32(float v)
{
    unsigned u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    return __uint_as_float(u);
}

// one warp per descriptor: hi / lo planes (rows padded with zero descriptors up to n_pad) and, for the right set,
// |b|^2 (+inf for the padding rows so that they never become candidates)
__global__ void __launch_bounds__(128)
match_split_kernel(const ps_descriptor* __restrict__ d, int n, int n_pad, float* __restrict__ hi, float* __restrict__ lo, float* __restrict__ norm)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= n_pad) return;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < n) v = __ldg(reinterpret_cast<const float4*>(d + row) + lane);
    const float4 h = make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    const float4 lw = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
    reinterpret_cast<float4*>(hi + (size_t)row * 128)[lane] = h;
    reinterpret_cast<float4*>(lo + (size_t)row * 128)[lane] = lw;
    if (norm) {
        float s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) norm[row] = row < n ? s : INFINITY;
    }
}

// ------------------------------------------------------------------------------------------------ tensor-core pass

constexpr int BM = 128, BN = 128;            // left descriptors per CTA, right descriptors per tile (= N of one wgmma)
constexpr int KB = 32;                       // floats per K-block = one 128-byte swizzle span
constexpr int NKB = 128 / KB;                // K-blocks per descriptor
constexpr int MMA_K = 8;                     // tf32: 32 bytes per instruction
constexpr int TILE_BYTES = 128 * KB * 4;     // 16 KB: one [128 rows x 128 bytes] operand tile
constexpr int STAGES = 3;                    // B ring: one K-block of a right tile (hi and lo) per stage
constexpr int TC_THREADS = 384;              // warpgroup 0 = TMA producer, warpgroups 1 and 2 = MMA + epilogue
constexpr int kCand = 4;                     // candidates kept per left descriptor
// A hi/lo resident (128 KB) + the ring (96 KB) + slack to align the dynamic buffer to 1024 bytes
constexpr size_t TC_SMEM = (size_t)2 * NKB * TILE_BYTES + (size_t)STAGES * 2 * TILE_BYTES + 1024;

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* b, unsigned n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(s32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void mb_expect(uint64_t* b, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mb_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mb_wait(uint64_t* b, unsigned parity)
{
    unsigned ok, spins = 0;
    for (;;) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(s32(b)), "r"(parity) : "memory");
        if (ok) break;
        if (++spins > (1u << 24)) __trap();          // abort instead of hanging the device
    }
}
__device__ __forceinline__ void tma_tile(void* dst, const CUtensorMap* map, int k0, int row0, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(s32(dst)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(k0), "r"(row0), "r"(s32(bar)) : "memory");
}
// wgmma shared-memory descriptor of a K-major operand tile, SWIZZLE_128B, rows 128 bytes wide, 8-row groups 1024 bytes
// apart: start >> 4 in [0,14), LBO = 1 in [16,30) (unused by swizzled K-major layouts), SBO = 1024 >> 4 in [32,46),
// layout SWIZZLE_128B = 1 in [62,64)
__device__ __forceinline__ uint64_t gmma_desc(const void* tile)
{
    return (uint64_t)((s32(tile) >> 4) & 0x3fffu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// D[64 x 128] (+)= A[64 x 8] . B[128 x 8]^T, tf32 in, fp32 accumulate, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc, int accumulate)
{
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}

// Candidate bookkeeping of one left descriptor: the four smallest keys seen so far and where they came from.  A key is
// the approximate distance |b|^2 - 2 a.b with its 5 low mantissa bits replaced by the column's position e (0..31) among
// the 32 columns of the tile this thread holds for the row (relative 2^-18: far below what separates candidates that
// matter, the exact re-rank follows), so that the minimum -- a branch-free FMNMX tree -- carries its own position.
struct Top4 {
    float t0 = INFINITY, t1 = INFINITY, t2 = INFINITY, t3 = INFINITY;
    int i0 = -1, i1 = -1, i2 = -1, i3 = -1;
    __device__ __forceinline__ void insert(float key, int idx)           // key < t3
    {
        t3 = key; i3 = idx;
        if (t3 < t2) { float tf = t2; t2 = t3; t3 = tf; int ti = i2; i2 = i3; i3 = ti;
            if (t2 < t1) { tf = t1; t1 = t2; t2 = tf; ti = i1; i1 = i2; i2 = ti;
                if (t1 < t0) { tf = t0; t0 = t1; t1 = tf; ti = i0; i0 = i1; i1 = ti; } } }
    }
    // the four best of this list and lane (lane ^ x)'s, whose columns are disjoint from ours
    __device__ __forceinline__ void merge_xor(int x)
    {
        const float pt[4] = {__shfl_xor_sync(0xffffffffu, t0, x), __shfl_xor_sync(0xffffffffu, t1, x),
                             __shfl_xor_sync(0xffffffffu, t2, x), __shfl_xor_sync(0xffffffffu, t3, x)};
        const int pi[4] = {__shfl_xor_sync(0xffffffffu, i0, x), __shfl_xor_sync(0xffffffffu, i1, x),
                           __shfl_xor_sync(0xffffffffu, i2, x), __shfl_xor_sync(0xffffffffu, i3, x)};
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (pt[k] < t3) insert(pt[k], pi[k]);
    }
};

// One row of the accumulator fragment: in the m64nNk8 layout a thread holds, for its row, the columns
// 8b + 2q + u (b = 0..15, u = 0..1, q = lane % 4) in d[4b + 2h + u] (h = 0: row lane / 4, h = 1: that row + 8).  The keys
// are formed in place; e = 2b + u is the column's position among the thread's 32.
template <int HALF>
__device__ __forceinline__ void top4_row(Top4& T, float (&d)[64], int nb, int q)
{
    float m[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const float a = d[4 * (i >> 1) + 2 * HALF + (i & 1)], b = d[4 * ((i + 16) >> 1) + 2 * HALF + (i & 1)];
        m[i] = fminf(a, b);                                                        // fminf drops NaNs
    }
#pragma unroll
    for (int w = 8; w >= 1; w >>= 1)
#pragma unroll
        for (int i = 0; i < w; ++i) m[i] = fminf(m[i], m[i + w]);
    float best = m[0];
    // rare after the first tiles: the k-th best of n random items improves about 4 / n of the time
    while (best < T.t3) {
        const int e = (int)(__float_as_uint(best) & 31u);
        T.insert(best, nb + 8 * (e >> 1) + 2 * q + (e & 1));
        float nxt = INFINITY;                                                  // the next key above `best`
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float k = d[4 * (i >> 1) + 2 * HALF + (i & 1)];
            nxt = (k > best) ? fminf(nxt, k) : nxt;
        }
        best = nxt;
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
match_tc_kernel(const __grid_constant__ CUtensorMap tm_lhi, const __grid_constant__ CUtensorMap tm_llo,
                const __grid_constant__ CUtensorMap tm_rhi, const __grid_constant__ CUtensorMap tm_rlo,
                const float* __restrict__ rnorm, int nl, int n_tiles, int32_t* __restrict__ cand)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t a_full, b_full[STAGES], b_empty[STAGES];
    // SWIZZLE_128B tiles: 1024-byte aligned
    uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
    uint8_t* A_hi = smem;                                       // NKB tiles
    uint8_t* A_lo = smem + NKB * TILE_BYTES;
    uint8_t* B_st = smem + 2 * NKB * TILE_BYTES;                // [STAGES][hi, lo]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM;

    if (threadIdx.x == 0) {
        mb_init(&a_full, 1);
        for (int s = 0; s < STAGES; ++s) { mb_init(&b_full[s], 1); mb_init(&b_empty[s], 8); }   // 8 consumer warps
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer (one thread) =====
        if (threadIdx.x == 0) {
            mb_expect(&a_full, 2 * NKB * TILE_BYTES);
            for (int kb = 0; kb < NKB; ++kb) {
                tma_tile(A_hi + kb * TILE_BYTES, &tm_lhi, kb * KB, m0, &a_full);
                tma_tile(A_lo + kb * TILE_BYTES, &tm_llo, kb * KB, m0, &a_full);
            }
            int s = 0; unsigned ph = 0;
            for (int j = 0; j < n_tiles; ++j)
                for (int kb = 0; kb < NKB; ++kb) {
                    mb_wait(&b_empty[s], ph ^ 1u);               // the MMAs that read this slot have completed
                    mb_expect(&b_full[s], 2 * TILE_BYTES);
                    tma_tile(B_st + (s * 2 + 0) * TILE_BYTES, &tm_rhi, kb * KB, j * BN, &b_full[s]);
                    tma_tile(B_st + (s * 2 + 1) * TILE_BYTES, &tm_rlo, kb * KB, j * BN, &b_full[s]);
                    if (++s == STAGES) { s = 0; ph ^= 1u; }
                }
        }
        return;
    }
    // ===== consumers: warpgroup c owns left rows 64c .. 64c+63 of the CTA's 128 =====
    const int c = (warp >> 2) - 1;
    const int q = lane & 3;
    const int row0 = m0 + 64 * c + 16 * (warp & 3) + (lane >> 2);      // fragment rows: row0 (h = 0) and row0 + 8 (h = 1)
    const unsigned a_off = (unsigned)(64 * c * 128);                   // 64 rows x 128 bytes into every A tile
    Top4 T0, T1;
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.0f;
    mb_wait(&a_full, 0);
    int s = 0; unsigned ph = 0;
    for (int j = 0; j < n_tiles; ++j) {
        const int nb0 = j * BN;
        // |b|^2 of the thread's 32 columns is on its way while the MMAs run
        float2 rn[16];
#pragma unroll
        for (int b = 0; b < 16; ++b) rn[b] = __ldg(reinterpret_cast<const float2*>(rnorm + nb0 + 8 * b + 2 * q));
        int prev = -1;
        for (int kb = 0; kb < NKB; ++kb) {
            mb_wait(&b_full[s], ph);
            wg_fence();
            const uint64_t a_hi = gmma_desc(A_hi + kb * TILE_BYTES + a_off), a_lo = gmma_desc(A_lo + kb * TILE_BYTES + a_off);
            const uint64_t b_hi = gmma_desc(B_st + (s * 2 + 0) * TILE_BYTES), b_lo = gmma_desc(B_st + (s * 2 + 1) * TILE_BYTES);
#pragma unroll
            for (int k8 = 0; k8 < KB / MMA_K; ++k8) {
                const uint64_t adv = (uint64_t)(k8 * MMA_K * 4 / 16);          // +32 bytes inside the swizzle span
                wgmma_tf32(d, a_hi + adv, b_hi + adv, (kb | k8) != 0);
                wgmma_tf32(d, a_hi + adv, b_lo + adv, 1);
                wgmma_tf32(d, a_lo + adv, b_hi + adv, 1);
            }
            wg_commit();
            if (prev >= 0) {                                   // the previous K-block's MMAs have read their slot
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) mb_arrive(&b_empty[prev]);
            }
            prev = s;
            if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mb_arrive(&b_empty[prev]);
        // keys |b|^2 - 2 a.b (+inf for padding columns, whose |b|^2 is +inf) with the column position in the low bits
#pragma unroll
        for (int b = 0; b < 16; ++b)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int i = 4 * b + 2 * h + u;
                    const float val = fmaf(-2.0f, d[i], u ? rn[b].y : rn[b].x);
                    d[i] = __uint_as_float((__float_as_uint(val) & 0xffffffe0u) | (unsigned)(2 * b + u));   // padding: inf or NaN
                }
        top4_row<0>(T0, d, nb0, q);
        top4_row<1>(T1, d, nb0, q);
    }
    // the four lanes of a quad hold disjoint columns of the same two rows
    T0.merge_xor(1); T1.merge_xor(1);
    T0.merge_xor(2); T1.merge_xor(2);
    if (q == 0) {
        if (row0 < nl) *reinterpret_cast<int4*>(cand + (size_t)row0 * kCand) = make_int4(T0.i0, T0.i1, T0.i2, T0.i3);
        if (row0 + 8 < nl) *reinterpret_cast<int4*>(cand + (size_t)(row0 + 8) * kCand) = make_int4(T1.i0, T1.i1, T1.i2, T1.i3);
    }
}

// exact distances of the candidates, in increasing index order, through the reference's scan
__global__ void __launch_bounds__(128)
match_rerank_kernel(const ps_descriptor* __restrict__ l, int nl, const ps_descriptor* __restrict__ r, int nr,
                    const int32_t* __restrict__ cand, int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= nl) return;
    const float4 l4 = __ldg(reinterpret_cast<const float4*>(l + row) + lane);
    int c[kCand];
#pragma unroll
    for (int k = 0; k < kCand; ++k) { c[k] = cand[(size_t)row * kCand + k]; if (c[k] < 0 || c[k] >= nr) c[k] = 0x7fffffff; }
    // sort the four indices ascending (the scan rule depends on arrival order)
#pragma unroll
    for (int a = 0; a < kCand; ++a)
#pragma unroll
        for (int b = a + 1; b < kCand; ++b)
            if (c[b] < c[a]) { const int t = c[a]; c[a] = c[b]; c[b] = t; }
    Best2 best; best.init();
#pragma unroll
    for (int k = 0; k < kCand; ++k) {
        if (c[k] == 0x7fffffff) continue;                         // warp-uniform
        if (k > 0 && c[k] == c[k - 1]) continue;
        best.step(warp_sq_dist(l4, reinterpret_cast<const float4*>(r + c[k]), lane), c[k]);
    }
    if (lane == 0) best.store(out + 3 * (size_t)row);
}

} // namespace

// POPSIFT_B200_MATCH=exact|tc overrides the automatic choice (A/B switch, cross-check)
int match_choice(int flags)
{
    static const int env = [] {
        const char* e = getenv("POPSIFT_B200_MATCH");
        if (!e) return 0;
        return e[0] == 'e' ? PS_MATCH_EXACT : e[0] == 't' ? PS_MATCH_TENSOR : 0;
    }();
    return flags ? flags : env;
}

int run_match(const ps_descriptor* l, int nl, const ps_descriptor* r, int nr, int32_t* out, int flags, cudaStream_t st,
              const char** err)
{
    *err = nullptr;
    if (nl <= 0) return 0;
    flags = match_choice(flags);
    // the tensor-core pass pays off from a few thousand pairs per left descriptor; below that (and for nr < 2, where
    // the reference's scan has its own corner cases) the CUDA-core kernel is the whole job
    const bool tensor = flags == PS_MATCH_TENSOR ? nr >= 1 : (flags == PS_MATCH_EXACT ? false : (nr >= 256 && (long long)nl * nr >= (1LL << 20)));
    if (!tensor) {
        match_exact_kernel<<<(nl + 3) / 4, 128, 0, st>>>(l, nl, r, nr, out);
        return 1;
    }
    const int nl_pad = (nl + BM - 1) / BM * BM, n_tiles = (nr + BN - 1) / BN, nr_pad = n_tiles * BN;
    float *lhi = nullptr, *llo = nullptr, *rhi = nullptr, *rlo = nullptr, *rnorm = nullptr;
    int32_t* cand = nullptr;
    const size_t lb = (size_t)nl_pad * 512, rb = (size_t)nr_pad * 512;
    // one workspace allocation per call, stream-ordered so nothing blocks, from the library's own pool per device: a pool
    // gives freed memory back to the OS at the next synchronisation unless told to keep it, and mapping 50 MB again on
    // every call costs more than the matching itself (the application's default pool is left alone)
    cudaMemPool_t pool = nullptr;
    {
        static std::mutex mu;
        static cudaMemPool_t pools[64] = {};
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); *err = "cudaGetDevice failed (matcher)"; return -1; }
        std::lock_guard<std::mutex> g(mu);
        if (!pools[dev]) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            if (cudaMemPoolCreate(&pools[dev], &props) != cudaSuccess) { cudaGetLastError(); pools[dev] = nullptr; *err = "cudaMemPoolCreate failed (matcher)"; return -1; }
            unsigned long long keep = 1ull << 30;                          // up to 1 GB of freed workspace stays mapped
            cudaMemPoolSetAttribute(pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
        }
        pool = pools[dev];
    }
    uint8_t* ws = nullptr;
    const size_t total = 2 * lb + 2 * rb + (size_t)nr_pad * 4 + (size_t)nl_pad * kCand * 4;
    if (cudaMallocFromPoolAsync(&ws, total, pool, st) != cudaSuccess) { *err = "cudaMallocFromPoolAsync failed (matcher workspace)"; cudaGetLastError(); return -1; }
    lhi = reinterpret_cast<float*>(ws); llo = reinterpret_cast<float*>(ws + lb);
    rhi = reinterpret_cast<float*>(ws + 2 * lb); rlo = reinterpret_cast<float*>(ws + 2 * lb + rb);
    rnorm = reinterpret_cast<float*>(ws + 2 * lb + 2 * rb);
    cand = reinterpret_cast<int32_t*>(ws + 2 * lb + 2 * rb + (size_t)nr_pad * 4);
    CUtensorMap m_lhi, m_llo, m_rhi, m_rlo;
    const bool ok = make_tmap_2d(&m_lhi, lhi, 128, nl_pad, 512, KB, BM, true) && make_tmap_2d(&m_llo, llo, 128, nl_pad, 512, KB, BM, true) &&
                    make_tmap_2d(&m_rhi, rhi, 128, nr_pad, 512, KB, BN, true) && make_tmap_2d(&m_rlo, rlo, 128, nr_pad, 512, KB, BN, true);
    if (!ok) { cudaFreeAsync(ws, st); *err = "cuTensorMapEncodeTiled failed (matcher)"; return -1; }
    static_assert(TC_SMEM + 1024 <= 227 * 1024, "matcher shared memory");
    match_split_kernel<<<(nl_pad + 3) / 4, 128, 0, st>>>(l, nl, nl_pad, lhi, llo, nullptr);
    match_split_kernel<<<(nr_pad + 3) / 4, 128, 0, st>>>(r, nr, nr_pad, rhi, rlo, rnorm);
    cudaFuncSetAttribute(match_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    match_tc_kernel<<<nl_pad / BM, TC_THREADS, TC_SMEM, st>>>(m_lhi, m_llo, m_rhi, m_rlo, rnorm, nl, n_tiles, cand);
    match_rerank_kernel<<<(nl + 3) / 4, 128, 0, st>>>(l, nl, r, nr, cand, out);
    cudaFreeAsync(ws, st);
    return 4;
}

} // namespace psb
