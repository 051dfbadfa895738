// Brute-force 2-nearest-neighbour descriptor matcher, hand-written for sm_90a (wgmma + TMA + mbarrier).
//
// Replaces FeaturesDev::match -> compute_distance (reference src/popsift/features.cu:165-227,282-304): for every
// left descriptor the best and second-best right descriptor by squared L2 distance and the ratio test
// best / second < 0.8.  The reference runs one 32-thread block per left descriptor and walks all right
// descriptors one by one (n_left x n_right x 128 scalar flops on CUDA cores, every right descriptor re-read
// n_left times).  This is the one dense contraction of the library:
//     |a - b|^2 = |a|^2 + |b|^2 - 2 a.b        ->   S = A . B^T  on the tensor cores.
//
// Pipeline (ps_match = a batch of one pair, ps_match_batch = many; per group of pairs planned by k_match_plan.h):
//   1. match_split_kernel     a = hi + lo with hi = tf32(a) (round to nearest), lo = a - hi, and |a|^2, for every set of
//                             the group once, into one pooled hi plane, lo plane and norm array (each set's rows padded
//                             to a multiple of 128; padding rows have norm +inf).  Three tf32 products hi.hi + hi.lo +
//                             lo.hi give a.b to ~2^-21 relative.
//   2. match_tc_kernel        persistent, one CTA (three warpgroups) per SM drawing work items (pair, 128-row left
//                             tile, contiguous chunk of right tiles).  The A tile (hi and lo, 128 x 128 floats each) is
//                             loaded with TMA (SWIZZLE_128B, K-major) and stays in shared memory while consecutive items
//                             share it; the right tiles stream through a 3-stage TMA ring of [128 descriptors x 32
//                             floats] tiles (hi and lo).  Both are row offsets into the same two tensor maps.  Warpgroup
//                             0 is the TMA producer (one thread); warpgroups 1 and 2 each own 64 left descriptors and
//                             issue wgmma.mma_async m64n128k8 tf32 into a register accumulator, then keep each of their
//                             rows' four best candidates |b|^2 - 2 a.b per item (a row's 128 columns are spread over the
//                             four lanes of a quad, merged at the end).  The n_left x n_right distance matrix never
//                             touches HBM.
//   3. match_rerank_kernel    one warp per (pair, left row) gathers the four candidates of each of the row's chunks and
//                             recomputes their exact float32 distances in the reference's own evaluation order (per lane
//                             x*x, fma, fma, fma over its float4, shuffle-down tree 16, 8, 4, 2, 1), in increasing index
//                             order, with the reference's scan rule (strict <, ties keep the lower index) and ratio test.
// The result equals the reference's except when three or more right descriptors of one chunk lie within ~4e-6 (relative)
// of the second best (the candidate pass could then miss the reference's pick among exact near-ties); more chunks keep
// more candidates and can only bring the result closer.
// match_exact_kernel is the same computation on CUDA cores (one warp per left descriptor over all right ones): used
// for small problems and as the in-library cross-check (PS_MATCH_EXACT).
#include "ps_internal.h"
#include "k_match_common.h"
#include "k_match_plan.h"
#include "k_guided.h"
#include "tma_util.h"
#include "workspace.h"

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

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

// one set of a group: its descriptors and its first row in the pooled planes (its padded rows run up to the next set's)
struct SplitSet { const ps_descriptor* d; int32_t n; int32_t row; };

// one warp per pooled row: hi / lo planes (each set's rows padded with zero descriptors to a multiple of 128) and |b|^2
// (+inf for the padding rows so that they never become candidates)
__global__ void __launch_bounds__(128)
match_split_kernel(const SplitSet* __restrict__ sets, int n_sets, int rows, float* __restrict__ hi, float* __restrict__ lo, float* __restrict__ norm)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= rows) return;
    int a = 0, b = n_sets - 1;                                    // the last set that starts at or before `row`
    while (a < b) { const int m = (a + b + 1) >> 1; if (sets[m].row <= row) a = m; else b = m - 1; }
    const SplitSet ss = sets[a];
    const int n = ss.n;
    const ps_descriptor* d = ss.d;
    const int local = row - ss.row;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (local < n) v = __ldg(reinterpret_cast<const float4*>(d + local) + lane);
    const float4 h = make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    const float4 lw = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
    reinterpret_cast<float4*>(hi + (size_t)row * 128)[lane] = h;
    reinterpret_cast<float4*>(lo + (size_t)row * 128)[lane] = lw;
    float s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, v.w * v.w)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) norm[row] = local < n ? s : INFINITY;
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

// Persistent: CTA b runs the work items b, b + gridDim.x, ... (k_match_plan.h), each one 128-row left tile (A) against
// a contiguous run of right tiles (B), both addressed as rows of the same pooled hi / lo planes.  The producer and the
// consumers walk the same item sequence; the B ring's stage / phase carries across items, and A is reloaded only when
// the next item's left tile differs (a_empty: both consumer warpgroups' MMAs on the old A have completed).
__global__ void __launch_bounds__(TC_THREADS, 1)
match_tc_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                const float* __restrict__ norm, const MatchItem* __restrict__ items, int n_items, int32_t* __restrict__ cand)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t a_full, a_empty, b_full[STAGES], b_empty[STAGES];
    // SWIZZLE_128B tiles: 1024-byte aligned
    uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
    uint8_t* A_hi = smem;                                       // NKB tiles
    uint8_t* A_lo = smem + NKB * TILE_BYTES;
    uint8_t* B_st = smem + 2 * NKB * TILE_BYTES;                // [STAGES][hi, lo]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        mb_init(&a_full, 1);
        mb_init(&a_empty, 8);                                                                    // 8 consumer warps
        for (int s = 0; s < STAGES; ++s) { mb_init(&b_full[s], 1); mb_init(&b_empty[s], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer (one thread) =====
        if (threadIdx.x == 0) {
            int s = 0; unsigned ph = 0;
            int a_cur = -1; unsigned a_ph = 0;
            for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
                const MatchItem w = items[it];
                if (w.a_row != a_cur) {
                    if (a_cur >= 0) { mb_wait(&a_empty, a_ph); a_ph ^= 1u; }   // the consumers are done with the old A
                    a_cur = w.a_row;
                    mb_expect(&a_full, 2 * NKB * TILE_BYTES);
                    for (int kb = 0; kb < NKB; ++kb) {
                        tma_tile(A_hi + kb * TILE_BYTES, &tm_hi, kb * KB, w.a_row, &a_full);
                        tma_tile(A_lo + kb * TILE_BYTES, &tm_lo, kb * KB, w.a_row, &a_full);
                    }
                }
                for (int j = 0; j < w.b_tiles; ++j)
                    for (int kb = 0; kb < NKB; ++kb) {
                        mb_wait(&b_empty[s], ph ^ 1u);               // the MMAs that read this slot have completed
                        mb_expect(&b_full[s], 2 * TILE_BYTES);
                        tma_tile(B_st + (s * 2 + 0) * TILE_BYTES, &tm_hi, kb * KB, w.b_row + j * BN, &b_full[s]);
                        tma_tile(B_st + (s * 2 + 1) * TILE_BYTES, &tm_lo, kb * KB, w.b_row + j * BN, &b_full[s]);
                        if (++s == STAGES) { s = 0; ph ^= 1u; }
                    }
            }
        }
        return;
    }
    // ===== consumers: warpgroup c owns rows 64c .. 64c+63 of each item's 128 =====
    const int c = (warp >> 2) - 1;
    const int q = lane & 3;
    const int r0 = 64 * c + 16 * (warp & 3) + (lane >> 2);             // fragment rows: r0 (h = 0) and r0 + 8 (h = 1)
    const unsigned a_off = (unsigned)(64 * c * 128);                   // 64 rows x 128 bytes into every A tile
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.0f;
    int s = 0; unsigned ph = 0;
    int a_cur = -1; unsigned a_ph = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const MatchItem w = items[it];
        if (w.a_row != a_cur) { mb_wait(&a_full, a_ph); a_ph ^= 1u; a_cur = w.a_row; }
        const float* __restrict__ rnorm = norm + w.b_row;
        Top4 T0, T1;
        for (int j = 0; j < w.b_tiles; ++j) {
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
            // candidate indices relative to the right set
            top4_row<0>(T0, d, w.b_col0 + nb0, q);
            top4_row<1>(T1, d, w.b_col0 + nb0, q);
        }
        // the four lanes of a quad hold disjoint columns of the same two rows
        T0.merge_xor(1); T1.merge_xor(1);
        T0.merge_xor(2); T1.merge_xor(2);
        if (q == 0) {
            int32_t* cw = cand + (size_t)(w.cand + (int64_t)r0 * w.stride) * kCand;
            if (w.l_row0 + r0 < w.nl) *reinterpret_cast<int4*>(cw) = make_int4(T0.i0, T0.i1, T0.i2, T0.i3);
            if (w.l_row0 + r0 + 8 < w.nl) *reinterpret_cast<int4*>(cw + (size_t)8 * w.stride * kCand) = make_int4(T1.i0, T1.i1, T1.i2, T1.i3);
        }
        // every MMA of this warp on the current A has completed (wg_wait<0> of the last tile): release it if the next item
        // needs another left tile
        const int nx = it + gridDim.x;
        if (nx < n_items && items[nx].a_row != a_cur) {
            __syncwarp();
            if (lane == 0) mb_arrive(&a_empty);
        }
    }
}

// the re-rank's view of one pair of a group
struct RerankPair {
    const ps_descriptor* l;
    const ps_descriptor* r;
    int64_t out_row;      // first output row of the pair
    int64_t row;          // first row of the pair among the group's rows (ascending over the group's pairs)
    int64_t cand;         // first candidate slot; row i, chunk c: cand + i * chunks + c
    int32_t nr, chunks;
};

// One warp per (pair, left row): the 4 x chunks candidates (one lane each), sorted ascending by a warp bitonic sort,
// duplicates and empty slots dropped, then their exact distances in increasing index order through the reference's scan.
// With one chunk this is the four-candidate re-rank of the single-pair matcher, step for step.
__global__ void __launch_bounds__(128)
match_rerank_kernel(const RerankPair* __restrict__ pairs, int n_pairs, int64_t rows, const int32_t* __restrict__ cand,
                    int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int64_t g = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (g >= rows) return;
    int a = 0, b = n_pairs - 1;                                   // the last pair that starts at or before row g
    while (a < b) { const int m = (a + b + 1) >> 1; if (pairs[m].row <= g) a = m; else b = m - 1; }
    const RerankPair P = pairs[a];
    const int64_t row = g - P.row;
    int v = 0x7fffffff;
    if (lane < kCand * P.chunks) {
        v = cand[(size_t)(P.cand + row * P.chunks) * kCand + lane];
        if (v < 0 || v >= P.nr) v = 0x7fffffff;
    }
    // ascending across the first K lanes, K = 4 x chunks rounded up to a power of two (the scan rule depends on arrival
    // order; the lanes beyond 4 x chunks hold 0x7fffffff)
    const int K = P.chunks <= 1 ? 4 : P.chunks <= 2 ? 8 : P.chunks <= 4 ? 16 : 32;
    for (int k = 2; k <= K; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            const int o = __shfl_xor_sync(0xffffffffu, v, j);
            v = (((lane & j) == 0) == ((lane & k) == 0)) ? min(v, o) : max(v, o);
        }
    Best2 best; best.init();
    if (P.chunks > 0) {
        const float4 l4 = __ldg(reinterpret_cast<const float4*>(P.l + row) + lane);
        int prev = -1;
        for (int k = 0; k < K; ++k) {
            const int ck = __shfl_sync(0xffffffffu, v, k);        // warp-uniform
            if (ck == 0x7fffffff) break;
            if (ck == prev) continue;
            prev = ck;
            best.step(warp_sq_dist(l4, reinterpret_cast<const float4*>(P.r + ck), lane), ck);
        }
    }
    if (lane == 0) best.store(out + 3 * (size_t)(P.out_row + row));
}

// ------------------------------------------------------------------------------------------------ guided matching
//
// ps_match_guided_batch (include/popsift_b200_guided.h): the same 2-NN, restricted per left row to the right descriptors
// that pass the pair's geometric test (k_guided.h).  The EXACT kernel skips ineligible columns (the test is warp-uniform);
// the tensor-core kernel is match_tc_kernel with the test fused into its epilogue: an ineligible element's value becomes
// +inf before its key is packed, so that it behaves like a padding column (inf or NaN after the low bits are replaced,
// dropped by fminf, never < t3) and never becomes a candidate.  The re-rank is match_rerank_kernel unchanged: it only
// sees candidates, and every candidate is eligible.

// launched only for pairs with a non-empty right set (the model is read unconditionally)
template <int MODEL>
__global__ void __launch_bounds__(128, 8)
match_exact_guided_kernel(const ps_descriptor* __restrict__ l, const ps_feature* __restrict__ fl, const int32_t* __restrict__ revl, int nl,
                          const ps_descriptor* __restrict__ r, const ps_feature* __restrict__ fr, const int32_t* __restrict__ revr, int nr,
                          const float* __restrict__ model, float t2, int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= nl) return;
    const float4 l4 = __ldg(reinterpret_cast<const float4*>(l + row) + lane);
    float m[9];
    load_model(m, model);
    const float2 p = feat_xy(fl, revl, row);
    const GuidedRow gr = guided_row<MODEL>(m, t2, p.x, p.y);
    Best2 b; b.init();
    for (int i = 0; i < nr; ++i) {
        const float2 P = feat_xy(fr, revr, i);                            // the same for every lane
        if (!guided_ok<MODEL>(gr, guided_col<MODEL>(m, P.x, P.y), t2, P.x, P.y)) continue;
        b.step(warp_sq_dist(l4, reinterpret_cast<const float4*>(r + i), lane), i);
    }
    if (lane == 0) b.store(out + 3 * (size_t)row);
}

// one thread per pooled row: its pixel position (NaN for padding rows)
__global__ void __launch_bounds__(256)
match_coords_kernel(const MatchCoordSet* __restrict__ sets, int n_sets, int rows, float2* __restrict__ out)
{
    const int row = blockIdx.x * 256 + threadIdx.x;
    if (row >= rows) return;
    int a = 0, b = n_sets - 1;                                    // the last set that starts at or before `row`
    while (a < b) { const int m = (a + b + 1) >> 1; if (sets[m].row <= row) a = m; else b = m - 1; }
    const MatchCoordSet cs = sets[a];
    const int local = row - cs.row;
    out[row] = local < cs.n ? feat_xy(cs.f, cs.rev, local) : make_float2(NAN, NAN);
}

// top4_row with constant bounds at every level of the min tree, so that m[] stays in registers
template <int HALF>
__device__ __forceinline__ void top4_row_guided(Top4& T, float (&d)[64], int nb, int q)
{
    float m[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) m[i] = fminf(d[4 * (i >> 1) + 2 * HALF + (i & 1)], d[4 * ((i + 16) >> 1) + 2 * HALF + (i & 1)]);
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = fminf(m[i], m[i + 8]);
#pragma unroll
    for (int i = 0; i < 4; ++i) m[i] = fminf(m[i], m[i + 4]);
    m[0] = fminf(m[0], m[2]); m[1] = fminf(m[1], m[3]);
    float best = fminf(m[0], m[1]);
    while (best < T.t3) {
        const int e = (int)(__float_as_uint(best) & 31u);
        T.insert(best, nb + 8 * (e >> 1) + 2 * q + (e & 1));
        float nxt = INFINITY;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float k = d[4 * (i >> 1) + 2 * HALF + (i & 1)];
            nxt = (k > best) ? fminf(nxt, k) : nxt;
        }
        best = nxt;
    }
}

// match_tc_kernel plus the geometric test.  coords: the group's pooled pixel positions; models: the caller's 9 floats per
// pair; gpair: group pair -> caller pair.  A right tile's 128 positions (1 KB) come with the tile: the producer copies
// them with cp.async.bulk into a one-stage buffer (c_full / c_empty) after the tile's last K-block, and the consumers
// release it when their epilogue has read it.  One stage is what fits next to the 225 KB of operand tiles, and it is
// enough: the copy for tile j + 1 is issued while the consumers run tile j + 1's MMAs.
template <int MODEL>
__global__ void __launch_bounds__(TC_THREADS, 1)
match_tc_guided_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                       const float* __restrict__ norm, const float2* __restrict__ coords, const float* __restrict__ models,
                       const int32_t* __restrict__ gpair, float t2, const MatchItem* __restrict__ items, int n_items,
                       int32_t* __restrict__ cand)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t a_full, a_empty, b_full[STAGES], b_empty[STAGES], c_full, c_empty;
    __shared__ __align__(128) float2 cpos[BN];
    uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
    uint8_t* A_hi = smem;
    uint8_t* A_lo = smem + NKB * TILE_BYTES;
    uint8_t* B_st = smem + 2 * NKB * TILE_BYTES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        mb_init(&a_full, 1);
        mb_init(&a_empty, 8);
        for (int s = 0; s < STAGES; ++s) { mb_init(&b_full[s], 1); mb_init(&b_empty[s], 8); }
        mb_init(&c_full, 1);
        mb_init(&c_empty, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer (one thread) =====
        if (threadIdx.x == 0) {
            int s = 0; unsigned ph = 0, cph = 0;
            int a_cur = -1; unsigned a_ph = 0;
            for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
                const MatchItem w = items[it];
                if (w.a_row != a_cur) {
                    if (a_cur >= 0) { mb_wait(&a_empty, a_ph); a_ph ^= 1u; }
                    a_cur = w.a_row;
                    mb_expect(&a_full, 2 * NKB * TILE_BYTES);
                    for (int kb = 0; kb < NKB; ++kb) {
                        tma_tile(A_hi + kb * TILE_BYTES, &tm_hi, kb * KB, w.a_row, &a_full);
                        tma_tile(A_lo + kb * TILE_BYTES, &tm_lo, kb * KB, w.a_row, &a_full);
                    }
                }
                for (int j = 0; j < w.b_tiles; ++j) {
                    for (int kb = 0; kb < NKB; ++kb) {
                        mb_wait(&b_empty[s], ph ^ 1u);
                        mb_expect(&b_full[s], 2 * TILE_BYTES);
                        tma_tile(B_st + (s * 2 + 0) * TILE_BYTES, &tm_hi, kb * KB, w.b_row + j * BN, &b_full[s]);
                        tma_tile(B_st + (s * 2 + 1) * TILE_BYTES, &tm_lo, kb * KB, w.b_row + j * BN, &b_full[s]);
                        if (++s == STAGES) { s = 0; ph ^= 1u; }
                    }
                    mb_wait(&c_empty, cph ^ 1u);                     // the epilogue of the previous tile has read it
                    mb_expect(&c_full, BN * sizeof(float2));
                    bulk_copy(cpos, coords + w.b_row + j * BN, BN * sizeof(float2), &c_full);
                    cph ^= 1u;
                }
            }
        }
        return;
    }
    // ===== consumers: warpgroup c owns rows 64c .. 64c+63 of each item's 128 =====
    const int c = (warp >> 2) - 1;
    const int q = lane & 3;
    const int r0 = 64 * c + 16 * (warp & 3) + (lane >> 2);
    const unsigned a_off = (unsigned)(64 * c * 128);
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.0f;
    int s = 0; unsigned ph = 0, cph = 0;
    int a_cur = -1; unsigned a_ph = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const MatchItem w = items[it];
        if (w.a_row != a_cur) { mb_wait(&a_full, a_ph); a_ph ^= 1u; a_cur = w.a_row; }
        const float* __restrict__ rnorm = norm + w.b_row;
        // the pair's model, and the per-row part of the test for the thread's two left rows (NaN rows: nothing eligible)
        float m[9];
        load_model(m, models + 9 * (size_t)__ldg(gpair + w.pair));
        const float2 p0 = __ldg(coords + w.a_row + r0), p1 = __ldg(coords + w.a_row + r0 + 8);
        const GuidedRow g0 = guided_row<MODEL>(m, t2, p0.x, p0.y), g1 = guided_row<MODEL>(m, t2, p1.x, p1.y);
        Top4 T0, T1;
        for (int j = 0; j < w.b_tiles; ++j) {
            const int nb0 = j * BN;
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
                    const uint64_t adv = (uint64_t)(k8 * MMA_K * 4 / 16);
                    wgmma_tf32(d, a_hi + adv, b_hi + adv, (kb | k8) != 0);
                    wgmma_tf32(d, a_hi + adv, b_lo + adv, 1);
                    wgmma_tf32(d, a_lo + adv, b_hi + adv, 1);
                }
                wg_commit();
                if (prev >= 0) {
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
            mb_wait(&c_full, cph);
            cph ^= 1u;
            // keys as in match_tc_kernel; an ineligible element is +inf before packing.  Columns 8b + 2q and 8b + 2q + 1
            // are one float4 of the position buffer; the per-column part of the test serves both rows.
#pragma unroll
            for (int b = 0; b < 16; ++b) {
                const float4 xy = reinterpret_cast<const float4*>(cpos)[4 * b + q];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const float X = u ? xy.z : xy.x, Y = u ? xy.w : xy.y;
                    const float cb = guided_col<MODEL>(m, X, Y);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * b + 2 * h + u;
                        const bool ok = guided_ok<MODEL>(h ? g1 : g0, cb, t2, X, Y);
                        const float val = ok ? fmaf(-2.0f, d[i], u ? rn[b].y : rn[b].x) : INFINITY;
                        d[i] = __uint_as_float((__float_as_uint(val) & 0xffffffe0u) | (unsigned)(2 * b + u));
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mb_arrive(&c_empty);
            top4_row_guided<0>(T0, d, w.b_col0 + nb0, q);
            top4_row_guided<1>(T1, d, w.b_col0 + nb0, q);
        }
        T0.merge_xor(1); T1.merge_xor(1);
        T0.merge_xor(2); T1.merge_xor(2);
        if (q == 0) {
            int32_t* cw = cand + (size_t)(w.cand + (int64_t)r0 * w.stride) * kCand;
            if (w.l_row0 + r0 < w.nl) *reinterpret_cast<int4*>(cw) = make_int4(T0.i0, T0.i1, T0.i2, T0.i3);
            if (w.l_row0 + r0 + 8 < w.nl) *reinterpret_cast<int4*>(cw + (size_t)8 * w.stride * kCand) = make_int4(T1.i0, T1.i1, T1.i2, T1.i3);
        }
        const int nx = it + gridDim.x;
        if (nx < n_items && items[nx].a_row != a_cur) {
            __syncwarp();
            if (lane == 0) mb_arrive(&a_empty);
        }
    }
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

size_t match_workspace_cap()
{
    static const size_t cap = [] {
        const char* e = getenv("POPSIFT_B200_MATCH_WS");
        const unsigned long long v = e ? strtoull(e, nullptr, 10) : 0ull;
        return v > 0 ? (size_t)v : kMatchPoolKeep;
    }();
    return cap;
}

namespace {

constexpr int kUnguided = -1;

// The host side of the batched matcher: plan, metadata upload, workspace, launches.  MODE = kUnguided: ps_match_batch;
// MODE = kGuidedH / kGuidedF: ps_match_guided_batch, which also uses feat, rev, models and t2, and whose pooled rows carry
// the row's pixel position (8 more bytes per row).  Arguments already validated, flags already resolved.
template <int MODE>
int run_batch(const ps_descriptor* const* sets, const ps_feature* const* feat, const int32_t* const* rev, const int32_t* n_desc,
              int n_sets, const int32_t* pairs, int n_pairs, const float* models, float t2, int32_t* out, int flags,
              cudaStream_t st, const char** err)
{
    constexpr bool guided = MODE != kUnguided;
    constexpr size_t row_bytes = guided ? kMatchGuidedRowBytes : kMatchRowBytes;
    const MatchPlan plan = plan_match(n_sets, n_desc, n_pairs, pairs, sm_count(), match_workspace_cap(), row_bytes);
    int launches = 0;
    if (flags == PS_MATCH_EXACT) {
        // the CUDA-core kernel, pair by pair: the in-library reference
        for (int p = 0; p < n_pairs; ++p) {
            const int l = pairs[2 * p], r = pairs[2 * p + 1];
            if (n_desc[l] <= 0) continue;
            int32_t* o = out + 3 * (size_t)plan.out_row[p];
            if constexpr (guided) {
                // an empty right set gives rows (0, 0, 0), and the pair's model need not exist: it is not read
                if (n_desc[r] <= 0) {
                    if (cudaMemsetAsync(o, 0, (size_t)n_desc[l] * 3 * sizeof(int32_t), st) != cudaSuccess) {
                        cudaGetLastError(); *err = "guided matcher: cudaMemsetAsync failed"; return -1;
                    }
                    continue;
                }
                match_exact_guided_kernel<MODE><<<(n_desc[l] + 3) / 4, 128, 0, st>>>(sets[l], feat[l], rev[l], n_desc[l], sets[r], feat[r], rev[r],
                                                                                  n_desc[r], models + 9 * (size_t)p, t2, o);
            } else {
                match_exact_kernel<<<(n_desc[l] + 3) / 4, 128, 0, st>>>(sets[l], n_desc[l], sets[r], n_desc[r], o);
            }
            ++launches;
        }
        return launches;
    }
    if (plan.groups.empty()) return 0;
    // every group's sets, pairs and items (guided: also its position sets and its group pair -> caller pair map), uploaded
    // once; one workspace for the largest group's planes, reused in turn
    struct Meta { size_t sets, csets, pairs, gpair, items; };
    std::vector<Meta> meta;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (matcher workspace)", "matcher: plan upload failed");
    size_t planes = 0;
    for (const MatchGroup& g : plan.groups) {
        if (g.rows > 0x7fffff80) { *err = "matcher: a group of pairs has more than 2^31 rows"; return -1; }
        std::vector<SplitSet> hs(g.sets.size());
        std::vector<MatchCoordSet> hc(guided ? g.sets.size() : 0);
        for (size_t k = 0; k < g.sets.size(); ++k) {
            const int si = g.sets[k].set;
            hs[k] = {sets[si], n_desc[si], (int32_t)g.sets[k].row};
            if (guided) hc[k] = {feat[si], rev[si], n_desc[si], (int32_t)g.sets[k].row};
        }
        std::vector<RerankPair> hp(g.pairs.size());
        std::vector<int32_t> hg(guided ? g.pairs.size() : 0);
        for (size_t k = 0; k < g.pairs.size(); ++k) {
            const MatchGroupPair& gp = g.pairs[k];
            const int l = pairs[2 * gp.pair], r = pairs[2 * gp.pair + 1];
            hp[k] = {sets[l], sets[r], plan.out_row[gp.pair], gp.row, gp.cand, n_desc[r], gp.chunks};
            if (guided) hg[k] = gp.pair;
        }
        Meta m;
        m.sets = ws.put(hs.data(), hs.size() * sizeof(SplitSet), 16);
        m.csets = ws.put(hc.data(), hc.size() * sizeof(MatchCoordSet), 16);
        m.pairs = ws.put(hp.data(), hp.size() * sizeof(RerankPair), 16);
        m.gpair = ws.put(hg.data(), hg.size() * sizeof(int32_t), 16);
        m.items = ws.put(g.items.data(), g.items.size() * sizeof(MatchItem), 16);
        meta.push_back(m);
        planes = std::max(planes, g.bytes());
    }
    const size_t o_planes = ws.take(planes, 1024);
    if (!ws.alloc(err)) return -1;
    static_assert(TC_SMEM + 1024 <= 227 * 1024, "matcher shared memory");
    static_assert(TC_SMEM + 1024 + BN * sizeof(float2) <= 227 * 1024, "guided matcher shared memory");
    static_assert(BM == kMatchTile && BN == kMatchTile && kCand == kMatchCand, "planner and kernel tile sizes");
    static_assert(kMatchGuidedRowBytes == kMatchRowBytes + sizeof(float2), "pooled guided row: hi + lo, norm, position");
    if constexpr (guided) cudaFuncSetAttribute(match_tc_guided_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    else cudaFuncSetAttribute(match_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM);
    const int sms = sm_count();
    for (size_t gi = 0; gi < plan.groups.size(); ++gi) {
        const MatchGroup& g = plan.groups[gi];
        const RerankPair* d_pairs = ws.at<const RerankPair>(meta[gi].pairs);
        int32_t* cand = nullptr;
        if (!g.items.empty()) {
            const int rows = (int)g.rows;
            uint8_t* plane = ws.at<uint8_t>(o_planes);
            float* hi = reinterpret_cast<float*>(plane);
            float* lo = reinterpret_cast<float*>(plane + (size_t)rows * 512);
            float* norm = reinterpret_cast<float*>(plane + (size_t)rows * 1024);
            cand = reinterpret_cast<int32_t*>(plane + (size_t)rows * row_bytes);
            // one tensor map per plane: a left tile and a right tile are both row offsets into it
            CUtensorMap m_hi, m_lo;
            if (!make_tmap_2d(&m_hi, hi, 128, rows, 512, KB, BM, true) || !make_tmap_2d(&m_lo, lo, 128, rows, 512, KB, BM, true))
                return ws.fail("cuTensorMapEncodeTiled failed (matcher)", err);
            match_split_kernel<<<(rows + 3) / 4, 128, 0, st>>>(ws.at<const SplitSet>(meta[gi].sets), (int)g.sets.size(), rows, hi, lo, norm);
            const int n_items = (int)g.items.size();
            const MatchItem* d_items = ws.at<const MatchItem>(meta[gi].items);
            if constexpr (guided) {
                float2* pos = reinterpret_cast<float2*>(plane + (size_t)rows * kMatchRowBytes);
                launch_match_coords(ws.at<const MatchCoordSet>(meta[gi].csets), (int)g.sets.size(), rows, pos, st);
                match_tc_guided_kernel<MODE><<<std::min(sms, n_items), TC_THREADS, TC_SMEM, st>>>(
                    m_hi, m_lo, norm, pos, models, ws.at<const int32_t>(meta[gi].gpair), t2, d_items, n_items, cand);
                ++launches;
            } else {
                match_tc_kernel<<<std::min(sms, n_items), TC_THREADS, TC_SMEM, st>>>(m_hi, m_lo, norm, d_items, n_items, cand);
            }
            launches += 2;
        }
        match_rerank_kernel<<<(unsigned)((g.left_rows + 3) / 4), 128, 0, st>>>(d_pairs, (int)g.pairs.size(), g.left_rows, cand, out);
        ++launches;
    }
    return launches;
}

} // namespace

int run_match_batch(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs,
                    int32_t* out, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    if (n_pairs <= 0) return 0;
    return run_batch<kUnguided>(sets, nullptr, nullptr, n_desc, n_sets, pairs, n_pairs, nullptr, 0.0f, out, match_choice(flags), st, err);
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
    // a batch of one pair (one set when both sides are the same array)
    const ps_descriptor* sets[2] = {l, r};
    const int32_t n_desc[2] = {nl, nr};
    const bool same = l == r && nl == nr;
    const int32_t pair[2] = {0, same ? 0 : 1};
    return run_match_batch(sets, n_desc, same ? 1 : 2, pair, 1, out, PS_MATCH_TENSOR, st, err);
}

void launch_match_coords(const MatchCoordSet* d_sets, int n_sets, int rows, float2* out, cudaStream_t st)
{
    if (rows > 0) match_coords_kernel<<<(rows + 255) / 256, 256, 0, st>>>(d_sets, n_sets, rows, out);
}

int run_match_guided_batch(const ps_descriptor* const* sets, const ps_feature* const* feat, const int32_t* const* rev,
                           const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs, const float* models, int model,
                           float threshold, int32_t* out, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    if (n_pairs <= 0) return 0;
    flags = match_choice(flags);
    const float t2 = threshold * threshold;
    return model == kGuidedH ? run_batch<kGuidedH>(sets, feat, rev, n_desc, n_sets, pairs, n_pairs, models, t2, out, flags, st, err)
                             : run_batch<kGuidedF>(sets, feat, rev, n_desc, n_sets, pairs, n_pairs, models, t2, out, flags, st, err);
}

} // namespace psb
