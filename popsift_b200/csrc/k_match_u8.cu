// Exact brute-force 2-nearest-neighbour matcher for 8-bit descriptors, hand-written for sm_90a (integer wgmma + TMA +
// mbarrier).
//
// The 8-bit form is what the reference prints under --write-as-uchar (roundf of every component, features.cu:317-320;
// combined with --norm-multi=9 or similar, main.cpp:119).  For u8 vectors a and b every term of
//     |a - b|^2 = |a|^2 + |b|^2 - 2 a.b
// is an integer below 128 * 255^2 = 8 323 200 < 2^23, so the contraction S = A . B^T runs exactly on the integer tensor
// cores (wgmma m64n128k32 s32.u8.u8, one IGMMA per 32 bytes of K) and the 2-NN selection can be exact in the epilogue:
// no candidate list, no re-rank.
//
// Pipeline (ps_match_u8_batch, per group of pairs planned by k_match_plan.h with 132-byte rows):
//   1. match_u8_pack_kernel      every set of the group once into one pooled u8 plane (each set's rows padded with zero
//                                rows to a multiple of 128) and one int32 norm key per pooled row,
//                                    nkey = (|b|^2 + 2^23) << 5 | e,
//                                e = the row's position among the 32 columns one consumer thread holds of a tile.
//                                Padding rows have |b|^2 = 2^24: their a.b is 0, so their key is above every real key.
//   2. match_u8_kernel           persistent, one CTA (three warpgroups) per SM over the same MatchItems as match_tc_kernel.
//                                A u8 descriptor is exactly one 128-byte swizzle span, so a 128-row tile is one 16 KB TMA
//                                box (UINT8, SWIZZLE_128B, K-major).  The A tile stays resident while consecutive items
//                                share it; right tiles stream through an 8-stage ring.  Warpgroup 0 is the TMA producer;
//                                warpgroups 1 and 2 each own 64 left rows and issue four m64n128k32 IGMMAs per right
//                                tile, then form  nkey - 64 a.b = (key + 2^23) << 5 | e  with key = |b|^2 - 2 a.b  (one
//                                IMAD per element) and take the minimum with an IMNMX tree: ties within a thread's 32
//                                columns go to the lower column.  Across tiles, quad lanes and chunks entries are compared
//                                as (key, right index), never as packed words.  Two (key, index) pairs per (row, chunk).
//   3. match_u8_finalize_kernel  one thread per (pair, left row) merges its chunks' pairs lexicographically, adds |a|^2
//                                (from the norm key) and writes (best, second, accept).
// Rows equal ps_match_batch(..., PS_MATCH_EXACT) on float32 copies of the same sets, bit for bit: that kernel is exact on
// these integers (a lane's partial sum <= 4 * 255^2, the total < 2^24), its strict-< scan in index order keeps the
// lexicographically smallest (distance, index) pairs, and accept = float(d1) / float(d2) < 0.8 in both.
// match_u8_exact_kernel is the CUDA-core form (one warp per left row, __dp4a), pair by pair: PS_MATCH_EXACT.
#include "ps_internal.h"
#include "k_match_common.h"
#include "k_match_plan.h"
#include "k_guided.h"
#include "tma_util.h"
#include "workspace.h"

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kKeyBias = 1 << 23;         // key + 2^23 > 0 for every key (|key| <= 128 * 255^2 < 2^23)
constexpr int kPadNorm = 1 << 24;         // |b|^2 of a padding row
constexpr int kNone = INT_MAX;            // no entry (key and index)

// ------------------------------------------------------------------------------------------------ quantisation

// q = roundf(min(max(v, 0), 255)); fmaxf turns NaN into 0
__global__ void __launch_bounds__(256)
to_u8_kernel(const float* __restrict__ in, size_t n, uint8_t* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint8_t)roundf(fminf(fmaxf(__ldg(in + i), 0.0f), 255.0f));
}

// ------------------------------------------------------------------------------------------------ exact (CUDA cores)

__device__ __forceinline__ float dist_f(int d) { return d == kNone ? INFINITY : (float)d; }

// (best, second, accept) of one row from its two smallest (distance, index) pairs; kNone distance: no such descriptor
// (index 0 and distance +inf, as the float scan leaves them)
__device__ __forceinline__ void store_row(int32_t* out, int d1, int i1, int d2, int i2)
{
    out[0] = d1 == kNone ? 0 : i1;
    out[1] = d2 == kNone ? 0 : i2;
    out[2] = (__fdiv_rn(dist_f(d1), dist_f(d2)) < 0.8f) ? 1 : 0;
}

// one warp per left row: lane holds bytes 4 lane .. 4 lane + 3; |a - b|^2 = sum of the byte-wise |a - b| squared
__global__ void __launch_bounds__(128)
match_u8_exact_kernel(const uint8_t* __restrict__ l, int nl, const uint8_t* __restrict__ r, int nr, int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= nl) return;
    const unsigned a = __ldg(reinterpret_cast<const unsigned*>(l + (size_t)row * 128) + lane);
    int d1 = kNone, d2 = kNone, i1 = 0, i2 = 0;
    for (int i = 0; i < nr; ++i) {
        const unsigned df = __vabsdiffu4(a, __ldg(reinterpret_cast<const unsigned*>(r + (size_t)i * 128) + lane));
        const int d = (int)__reduce_add_sync(0xffffffffu, __dp4a(df, df, 0u));
        if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = i; }            // the reference's scan rule: strict <, index order
        else if (d < d2) { d2 = d; i2 = i; }
    }
    if (lane == 0) store_row(out + 3 * (size_t)row, d1, i1, d2, i2);
}

// ------------------------------------------------------------------------------------------------ pack

// one set of a group: its descriptors and its first row in the pooled plane (its padded rows run up to the next set's)
struct PackSet { const uint8_t* d; int32_t n; int32_t row; };

// one warp per pooled row: the row (zeros for padding) and its norm key
__global__ void __launch_bounds__(128)
match_u8_pack_kernel(const PackSet* __restrict__ sets, int n_sets, int rows, uint8_t* __restrict__ plane, int32_t* __restrict__ nkey)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= rows) return;
    int a = 0, b = n_sets - 1;                                    // the last set that starts at or before `row`
    while (a < b) { const int m = (a + b + 1) >> 1; if (sets[m].row <= row) a = m; else b = m - 1; }
    const PackSet ps = sets[a];
    const int local = row - ps.row;
    unsigned v = 0;
    if (local < ps.n) v = __ldg(reinterpret_cast<const unsigned*>(ps.d + (size_t)local * 128) + lane);
    reinterpret_cast<unsigned*>(plane + (size_t)row * 128)[lane] = v;
    const int nn = (int)__reduce_add_sync(0xffffffffu, __dp4a(v, v, 0u));
    if (lane == 0) {
        const int c = row & 127;                                  // column within its tile (sets start at multiples of 128)
        nkey[row] = (((local < ps.n ? nn : kPadNorm) + kKeyBias) << 5) | (2 * (c >> 3) + (c & 1));
    }
}

// ------------------------------------------------------------------------------------------------ integer tensor-core pass

constexpr int BM = 128, BN = 128;            // left descriptors per CTA, right descriptors per tile (= N of one wgmma)
constexpr int MMA_K = 32;                    // u8: 32 bytes per instruction
constexpr int TILE_BYTES = 128 * 128;        // 16 KB: 128 descriptors x 128 bytes, one TMA box
constexpr int STAGES = 8;                    // B ring: one right tile per stage
constexpr int TC_THREADS = 384;              // warpgroup 0 = TMA producer, warpgroups 1 and 2 = MMA + epilogue
// A resident (16 KB) + the ring (128 KB) + slack to align the dynamic buffer to 1024 bytes
constexpr size_t U8_SMEM = (size_t)(1 + STAGES) * TILE_BYTES + 1024;

// D[64 x 128] (+)= A[64 x 32] . B[128 x 32]^T, u8 in, s32 accumulate, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_u8(int (&d)[64], uint64_t a_desc, uint64_t b_desc, int accumulate)
{
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}

// The two lexicographically smallest (key, right index) pairs seen so far of one left row
struct Top2 {
    int k1 = kNone, i1 = kNone, k2 = kNone, i2 = kNone;
    __device__ __forceinline__ bool beats2(int k, int i) const { return k < k2 || (k == k2 && i < i2); }
    __device__ __forceinline__ void insert(int k, int i)          // beats2(k, i)
    {
        if (k < k1 || (k == k1 && i < i1)) { k2 = k1; i2 = i1; k1 = k; i1 = i; }
        else { k2 = k; i2 = i; }
    }
    __device__ __forceinline__ void offer(int k, int i) { if (beats2(k, i)) insert(k, i); }
    // the two best of this pair of entries and lane (lane ^ x)'s, whose columns are disjoint from ours
    __device__ __forceinline__ void merge_xor(int x)
    {
        const int pk1 = __shfl_xor_sync(0xffffffffu, k1, x), pi1 = __shfl_xor_sync(0xffffffffu, i1, x);
        const int pk2 = __shfl_xor_sync(0xffffffffu, k2, x), pi2 = __shfl_xor_sync(0xffffffffu, i2, x);
        offer(pk1, pi1);
        offer(pk2, pi2);
    }
};

// One row of the accumulator fragment, keys already packed: in the m64nNk32 layout a thread holds, for its row, the
// columns 8b + 2q + u (b = 0..15, u = 0..1, q = lane % 4) in d[4b + 2h + u] (h = 0: row lane / 4, h = 1: that row + 8);
// e = 2b + u is the column's position among the thread's 32 and grows with the column.  col0: right index of the tile's
// first column.
template <int HALF>
__device__ __forceinline__ void top2_row(Top2& T, const int (&d)[64], int col0, int q)
{
    int m[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) m[i] = min(d[4 * (i >> 1) + 2 * HALF + (i & 1)], d[4 * ((i + 16) >> 1) + 2 * HALF + (i & 1)]);
    // constant bounds at every level, so that m[] stays in registers
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = min(m[i], m[i + 8]);
#pragma unroll
    for (int i = 0; i < 4; ++i) m[i] = min(m[i], m[i + 4]);
    m[0] = min(m[0], m[2]); m[1] = min(m[1], m[3]);
    const int best = min(m[0], m[1]);
    const int k = (best >> 5) - kKeyBias, e = best & 31;
    const int idx = col0 + 8 * (e >> 1) + 2 * q + (e & 1);
    // rare after the first tiles: the 2nd best of n random items improves about 2 / n of the time
    if (T.beats2(k, idx)) {
        T.insert(k, idx);
        int nxt = INT_MAX;                                       // the tile's next packed key (all 32 are distinct)
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int v = d[4 * (i >> 1) + 2 * HALF + (i & 1)];
            nxt = v > best ? min(nxt, v) : nxt;
        }
        const int e2 = nxt & 31;
        T.offer((nxt >> 5) - kKeyBias, col0 + 8 * (e2 >> 1) + 2 * q + (e2 & 1));
    }
}

// Persistent: CTA b runs the work items b, b + gridDim.x, ... (k_match_plan.h), each one 128-row left tile (A) against a
// contiguous run of right tiles (B), both addressed as rows of the same pooled plane.  The producer and the consumers walk
// the same item sequence; the ring's stage / phase carries across items, and A is reloaded only when the next item's
// left tile differs (a_empty: both consumer warpgroups' MMAs on the old A have completed).  cand: (key1, index1, key2,
// index2) per (left row, chunk), keys relative to |a|^2.
__global__ void __launch_bounds__(TC_THREADS, 1)
match_u8_kernel(const __grid_constant__ CUtensorMap tm, const int32_t* __restrict__ nkey, const MatchItem* __restrict__ items,
                int n_items, int4* __restrict__ cand)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t a_full, a_empty, b_full[STAGES], b_empty[STAGES];
    // SWIZZLE_128B tiles: 1024-byte aligned
    uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
    uint8_t* A = smem;
    uint8_t* B_st = smem + TILE_BYTES;                           // [STAGES]
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
                    mb_expect(&a_full, TILE_BYTES);
                    tma_tile(A, &tm, 0, w.a_row, &a_full);
                }
                for (int j = 0; j < w.b_tiles; ++j) {
                    mb_wait(&b_empty[s], ph ^ 1u);                   // the MMAs that read this slot have completed
                    mb_expect(&b_full[s], TILE_BYTES);
                    tma_tile(B_st + s * TILE_BYTES, &tm, 0, w.b_row + j * BN, &b_full[s]);
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
    const uint64_t a_desc = gmma_desc(A + 64 * c * 128);               // 64 rows x 128 bytes into the A tile
    int d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0;
    int s = 0; unsigned ph = 0;
    int a_cur = -1; unsigned a_ph = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const MatchItem w = items[it];
        if (w.a_row != a_cur) { mb_wait(&a_full, a_ph); a_ph ^= 1u; a_cur = w.a_row; }
        const int32_t* __restrict__ rkey = nkey + w.b_row;
        Top2 T0, T1;
        for (int j = 0; j < w.b_tiles; ++j) {
            const int nb0 = j * BN;
            // the norm keys of the thread's 32 columns are on their way while the MMAs run
            int2 nk[16];
#pragma unroll
            for (int b = 0; b < 16; ++b) nk[b] = __ldg(reinterpret_cast<const int2*>(rkey + nb0 + 8 * b + 2 * q));
            mb_wait(&b_full[s], ph);
            wg_fence();
            const uint64_t b_desc = gmma_desc(B_st + s * TILE_BYTES);
#pragma unroll
            for (int k = 0; k < 128 / MMA_K; ++k)
                wgmma_u8(d, a_desc + 2 * k, b_desc + 2 * k, k != 0);          // +32 bytes inside the swizzle span
            wg_commit();
            wg_wait<0>();
            __syncwarp();
            if (lane == 0) mb_arrive(&b_empty[s]);
            if (++s == STAGES) { s = 0; ph ^= 1u; }
            // (key + 2^23) << 5 | e = nkey - 64 a.b: the subtrahend's low 6 bits are zero, so e is untouched
#pragma unroll
            for (int b = 0; b < 16; ++b)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int i = 4 * b + 2 * h + u;
                        d[i] = (u ? nk[b].y : nk[b].x) - 64 * d[i];
                    }
            top2_row<0>(T0, d, w.b_col0 + nb0, q);
            top2_row<1>(T1, d, w.b_col0 + nb0, q);
        }
        // the four lanes of a quad hold disjoint columns of the same two rows
        T0.merge_xor(1); T1.merge_xor(1);
        T0.merge_xor(2); T1.merge_xor(2);
        if (q == 0) {
            int4* cw = cand + w.cand + (int64_t)r0 * w.stride;
            if (w.l_row0 + r0 < w.nl) *cw = make_int4(T0.k1, T0.i1, T0.k2, T0.i2);
            if (w.l_row0 + r0 + 8 < w.nl) cw[(int64_t)8 * w.stride] = make_int4(T1.k1, T1.i1, T1.k2, T1.i2);
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

// the finalize pass's view of one pair of a group
struct FinalPair {
    int64_t out_row;      // first output row of the pair
    int64_t row;          // first row of the pair among the group's rows (ascending over the group's pairs)
    int64_t cand;         // first candidate slot; row i, chunk c: cand + i * chunks + c
    int32_t a_row;        // pooled row of the left set's first descriptor (when chunks > 0)
    int32_t nr, chunks, pad_;
};

// one thread per (pair, left row): the lexicographic merge of the chunks' (key, index) pairs, padding columns (index >= nr)
// dropped, then distances = |a|^2 + key
__global__ void __launch_bounds__(128)
match_u8_finalize_kernel(const FinalPair* __restrict__ pairs, int n_pairs, int64_t rows, const int32_t* __restrict__ nkey,
                         const int4* __restrict__ cand, int32_t* __restrict__ out)
{
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= rows) return;
    int a = 0, b = n_pairs - 1;                                   // the last pair that starts at or before row g
    while (a < b) { const int m = (a + b + 1) >> 1; if (pairs[m].row <= g) a = m; else b = m - 1; }
    const FinalPair P = pairs[a];
    const int64_t row = g - P.row;
    Top2 T;
    for (int c = 0; c < P.chunks; ++c) {
        const int4 v = cand[P.cand + row * P.chunks + c];
        if (v.y < P.nr) T.offer(v.x, v.y);
        if (v.w < P.nr) T.offer(v.z, v.w);
    }
    const int na = T.k1 == kNone ? 0 : (nkey[P.a_row + row] >> 5) - kKeyBias;
    store_row(out + 3 * (size_t)(P.out_row + row), T.k1 == kNone ? kNone : na + T.k1, T.i1,
              T.k2 == kNone ? kNone : na + T.k2, T.i2);
}

// ------------------------------------------------------------------------------------------------ guided matching
//
// ps_match_u8_guided_batch (include/popsift_b200_guided.h): the exact 2-NN restricted per left row to the right descriptors
// that pass the pair's geometric test (k_guided.h).  In match_u8_guided_kernel an ineligible element's packed key becomes
// kMasked | e: above every real key (< (2^24 + 2^23) << 5) and every padding key (= that), still distinct in its low 5
// bits, so the min tree and the "next key" scan work unchanged.  Unpacked, its key is above kPadNorm, like a padding
// column's is equal to it, and the guided finalize drops every entry whose key is >= kPadNorm.

constexpr int kMasked = 0x7fffffe0;

// launched only for pairs with a non-empty right set (the model is read unconditionally)
template <int MODEL>
__global__ void __launch_bounds__(128, 8)
match_u8_exact_guided_kernel(const uint8_t* __restrict__ l, const ps_feature* __restrict__ fl, const int32_t* __restrict__ revl, int nl,
                             const uint8_t* __restrict__ r, const ps_feature* __restrict__ fr, const int32_t* __restrict__ revr, int nr,
                             const float* __restrict__ model, float t2, int32_t* __restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= nl) return;
    const unsigned a = __ldg(reinterpret_cast<const unsigned*>(l + (size_t)row * 128) + lane);
    float m[9];
    load_model(m, model);
    const float2 p = feat_xy(fl, revl, row);
    const GuidedRow gr = guided_row<MODEL>(m, t2, p.x, p.y);
    int d1 = kNone, d2 = kNone, i1 = 0, i2 = 0;
    for (int i = 0; i < nr; ++i) {
        const float2 P = feat_xy(fr, revr, i);                            // the same for every lane
        if (!guided_ok<MODEL>(gr, guided_col<MODEL>(m, P.x, P.y), t2, P.x, P.y)) continue;
        const unsigned df = __vabsdiffu4(a, __ldg(reinterpret_cast<const unsigned*>(r + (size_t)i * 128) + lane));
        const int d = (int)__reduce_add_sync(0xffffffffu, __dp4a(df, df, 0u));
        if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = i; }
        else if (d < d2) { d2 = d; i2 = i; }
    }
    if (lane == 0) store_row(out + 3 * (size_t)row, d1, i1, d2, i2);
}

// match_u8_kernel plus the geometric test.  coords: the group's pooled pixel positions; models: the caller's 9 floats per
// pair; gpair: group pair -> caller pair.  A right tile's 128 positions (1 KB) travel with the tile in the same ring stage
// (same b_full barrier), and the stage is released after the epilogue instead of after the MMAs.
template <int MODEL>
__global__ void __launch_bounds__(TC_THREADS, 1)
match_u8_guided_kernel(const __grid_constant__ CUtensorMap tm, const int32_t* __restrict__ nkey, const float2* __restrict__ coords,
                       const float* __restrict__ models, const int32_t* __restrict__ gpair, float t2,
                       const MatchItem* __restrict__ items, int n_items, int4* __restrict__ cand)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t a_full, a_empty, b_full[STAGES], b_empty[STAGES];
    uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
    uint8_t* A = smem;
    uint8_t* B_st = smem + TILE_BYTES;                           // [STAGES]
    float2* C_st = reinterpret_cast<float2*>(smem + (1 + STAGES) * TILE_BYTES);   // [STAGES][BN]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        mb_init(&a_full, 1);
        mb_init(&a_empty, 8);
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
                    if (a_cur >= 0) { mb_wait(&a_empty, a_ph); a_ph ^= 1u; }
                    a_cur = w.a_row;
                    mb_expect(&a_full, TILE_BYTES);
                    tma_tile(A, &tm, 0, w.a_row, &a_full);
                }
                for (int j = 0; j < w.b_tiles; ++j) {
                    mb_wait(&b_empty[s], ph ^ 1u);                   // the epilogue that read this slot is done
                    mb_expect(&b_full[s], TILE_BYTES + BN * sizeof(float2));
                    tma_tile(B_st + s * TILE_BYTES, &tm, 0, w.b_row + j * BN, &b_full[s]);
                    bulk_copy(C_st + s * BN, coords + w.b_row + j * BN, BN * sizeof(float2), &b_full[s]);
                    if (++s == STAGES) { s = 0; ph ^= 1u; }
                }
            }
        }
        return;
    }
    // ===== consumers: warpgroup c owns rows 64c .. 64c+63 of each item's 128 =====
    const int c = (warp >> 2) - 1;
    const int q = lane & 3;
    const int r0 = 64 * c + 16 * (warp & 3) + (lane >> 2);
    const uint64_t a_desc = gmma_desc(A + 64 * c * 128);
    int d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0;
    int s = 0; unsigned ph = 0;
    int a_cur = -1; unsigned a_ph = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const MatchItem w = items[it];
        if (w.a_row != a_cur) { mb_wait(&a_full, a_ph); a_ph ^= 1u; a_cur = w.a_row; }
        const int32_t* __restrict__ rkey = nkey + w.b_row;
        // the pair's model, and the per-row part of the test for the thread's two left rows (NaN rows: nothing eligible)
        float m[9];
        load_model(m, models + 9 * (size_t)__ldg(gpair + w.pair));
        const float2 p0 = __ldg(coords + w.a_row + r0), p1 = __ldg(coords + w.a_row + r0 + 8);
        const GuidedRow g0 = guided_row<MODEL>(m, t2, p0.x, p0.y), g1 = guided_row<MODEL>(m, t2, p1.x, p1.y);
        Top2 T0, T1;
        for (int j = 0; j < w.b_tiles; ++j) {
            const int nb0 = j * BN;
            int2 nk[16];
#pragma unroll
            for (int b = 0; b < 16; ++b) nk[b] = __ldg(reinterpret_cast<const int2*>(rkey + nb0 + 8 * b + 2 * q));
            mb_wait(&b_full[s], ph);
            wg_fence();
            const uint64_t b_desc = gmma_desc(B_st + s * TILE_BYTES);
#pragma unroll
            for (int k = 0; k < 128 / MMA_K; ++k)
                wgmma_u8(d, a_desc + 2 * k, b_desc + 2 * k, k != 0);
            wg_commit();
            wg_wait<0>();
            // packed keys as in match_u8_kernel; an ineligible element gets kMasked | e.  Columns 8b + 2q and 8b + 2q + 1
            // are one float4 of the stage's positions; the per-column part of the test serves both rows.
            const float4* cp = reinterpret_cast<const float4*>(C_st + s * BN);
#pragma unroll
            for (int b = 0; b < 16; ++b) {
                const float4 xy = cp[4 * b + q];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const float X = u ? xy.z : xy.x, Y = u ? xy.w : xy.y;
                    const float cb = guided_col<MODEL>(m, X, Y);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * b + 2 * h + u;
                        const bool ok = guided_ok<MODEL>(h ? g1 : g0, cb, t2, X, Y);
                        d[i] = ok ? (u ? nk[b].y : nk[b].x) - 64 * d[i] : (kMasked | (2 * b + u));
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mb_arrive(&b_empty[s]);
            if (++s == STAGES) { s = 0; ph ^= 1u; }
            top2_row<0>(T0, d, w.b_col0 + nb0, q);
            top2_row<1>(T1, d, w.b_col0 + nb0, q);
        }
        T0.merge_xor(1); T1.merge_xor(1);
        T0.merge_xor(2); T1.merge_xor(2);
        if (q == 0) {
            int4* cw = cand + w.cand + (int64_t)r0 * w.stride;
            if (w.l_row0 + r0 < w.nl) *cw = make_int4(T0.k1, T0.i1, T0.k2, T0.i2);
            if (w.l_row0 + r0 + 8 < w.nl) cw[(int64_t)8 * w.stride] = make_int4(T1.k1, T1.i1, T1.k2, T1.i2);
        }
        const int nx = it + gridDim.x;
        if (nx < n_items && items[nx].a_row != a_cur) {
            __syncwarp();
            if (lane == 0) mb_arrive(&a_empty);
        }
    }
}

// match_u8_finalize_kernel for guided rows: entries whose key is >= kPadNorm (padding columns and ineligible ones) dropped
__global__ void __launch_bounds__(128)
match_u8_guided_finalize_kernel(const FinalPair* __restrict__ pairs, int n_pairs, int64_t rows, const int32_t* __restrict__ nkey,
                                const int4* __restrict__ cand, int32_t* __restrict__ out)
{
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= rows) return;
    int a = 0, b = n_pairs - 1;
    while (a < b) { const int m = (a + b + 1) >> 1; if (pairs[m].row <= g) a = m; else b = m - 1; }
    const FinalPair P = pairs[a];
    const int64_t row = g - P.row;
    Top2 T;
    for (int c = 0; c < P.chunks; ++c) {
        const int4 v = cand[P.cand + row * P.chunks + c];
        if (v.x < kPadNorm) T.offer(v.x, v.y);
        if (v.z < kPadNorm) T.offer(v.z, v.w);
    }
    const int na = T.k1 == kNone ? 0 : (nkey[P.a_row + row] >> 5) - kKeyBias;
    store_row(out + 3 * (size_t)(P.out_row + row), T.k1 == kNone ? kNone : na + T.k1, T.i1,
              T.k2 == kNone ? kNone : na + T.k2, T.i2);
}

constexpr int kUnguided = -1;

// The host side of the batched 8-bit matcher: plan, metadata upload, workspace, launches.  MODE = kUnguided:
// ps_match_u8_batch; MODE = kGuidedH / kGuidedF: ps_match_u8_guided_batch, which also uses feat, rev, models and t2, and
// whose pooled rows carry the row's pixel position (8 more bytes per row).  Arguments already validated, flags resolved.
template <int MODE>
int run_u8_batch(const uint8_t* const* sets, const ps_feature* const* feat, const int32_t* const* rev, const int32_t* n_desc,
                 int n_sets, const int32_t* pairs, int n_pairs, const float* models, float t2, int32_t* out, int flags,
                 cudaStream_t st, const char** err)
{
    constexpr bool guided = MODE != kUnguided;
    constexpr size_t row_bytes = guided ? kMatchU8GuidedRowBytes : kMatchU8RowBytes;
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
                        cudaGetLastError(); *err = "guided u8 matcher: cudaMemsetAsync failed"; return -1;
                    }
                    continue;
                }
                match_u8_exact_guided_kernel<MODE><<<(n_desc[l] + 3) / 4, 128, 0, st>>>(sets[l], feat[l], rev[l], n_desc[l], sets[r], feat[r],
                                                                                     rev[r], n_desc[r], models + 9 * (size_t)p, t2, o);
            } else {
                match_u8_exact_kernel<<<(n_desc[l] + 3) / 4, 128, 0, st>>>(sets[l], n_desc[l], sets[r], n_desc[r], o);
            }
            ++launches;
        }
        return launches;
    }
    if (plan.groups.empty()) return 0;
    // every group's sets, pairs and items (guided: also its position sets and its group pair -> caller pair map), uploaded
    // once; one workspace for the largest group's plane, reused in turn
    struct Meta { size_t sets, csets, pairs, gpair, items; };
    std::vector<Meta> meta;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (u8 matcher workspace)", "u8 matcher: plan upload failed");
    size_t planes = 0;
    for (const MatchGroup& g : plan.groups) {
        if (g.rows > 0x7fffff80) { *err = "matcher: a group of pairs has more than 2^31 rows"; return -1; }
        std::vector<PackSet> hs(g.sets.size());
        std::vector<MatchCoordSet> hc(guided ? g.sets.size() : 0);
        for (size_t k = 0; k < g.sets.size(); ++k) {
            const int si = g.sets[k].set;
            hs[k] = {sets[si], n_desc[si], (int32_t)g.sets[k].row};
            if (guided) hc[k] = {feat[si], rev[si], n_desc[si], (int32_t)g.sets[k].row};
        }
        std::vector<FinalPair> hp(g.pairs.size());
        std::vector<int32_t> hg(guided ? g.pairs.size() : 0);
        for (size_t k = 0; k < g.pairs.size(); ++k) {
            const MatchGroupPair& gp = g.pairs[k];
            const int l = pairs[2 * gp.pair], r = pairs[2 * gp.pair + 1];
            int64_t a_row = 0;
            for (const MatchGroupSet& s : g.sets) if (s.set == l) a_row = s.row;
            hp[k] = {plan.out_row[gp.pair], gp.row, gp.cand, (int32_t)a_row, n_desc[r], gp.chunks, 0};
            if (guided) hg[k] = gp.pair;
        }
        Meta m;
        m.sets = ws.put(hs.data(), hs.size() * sizeof(PackSet), 16);
        m.csets = ws.put(hc.data(), hc.size() * sizeof(MatchCoordSet), 16);
        m.pairs = ws.put(hp.data(), hp.size() * sizeof(FinalPair), 16);
        m.gpair = ws.put(hg.data(), hg.size() * sizeof(int32_t), 16);
        m.items = ws.put(g.items.data(), g.items.size() * sizeof(MatchItem), 16);
        meta.push_back(m);
        planes = std::max(planes, g.bytes());
    }
    const size_t o_plane = ws.take(planes, 1024);
    if (!ws.alloc(err)) return -1;
    // the guided kernel's ring stages carry a right tile's 128 positions next to the tile
    constexpr size_t smem_bytes = U8_SMEM + (guided ? (size_t)STAGES * BN * sizeof(float2) : 0);
    static_assert(smem_bytes + 1024 <= 227 * 1024, "u8 matcher shared memory");
    static_assert(BM == kMatchTile && BN == kMatchTile && sizeof(int4) == kMatchCand * 4, "planner and kernel tile / slot sizes");
    static_assert(kMatchU8RowBytes == 128 + sizeof(int32_t), "pooled u8 row: descriptor + norm key");
    static_assert(kMatchU8GuidedRowBytes == kMatchU8RowBytes + sizeof(float2), "pooled guided u8 row: descriptor, norm key, position");
    static_assert(kMasked > ((kPadNorm + kKeyBias) << 5 | 31) && (kMasked & 31) == 0, "masked keys above padding keys");
    if constexpr (guided) cudaFuncSetAttribute(match_u8_guided_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    else cudaFuncSetAttribute(match_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    const int sms = sm_count();
    for (size_t gi = 0; gi < plan.groups.size(); ++gi) {
        const MatchGroup& g = plan.groups[gi];
        const FinalPair* d_pairs = ws.at<const FinalPair>(meta[gi].pairs);
        const int32_t* nkey = nullptr;
        const int4* cand = nullptr;
        if (!g.items.empty()) {
            const int rows = (int)g.rows;
            uint8_t* plane = ws.at<uint8_t>(o_plane);
            int32_t* nk = reinterpret_cast<int32_t*>(plane + (size_t)rows * 128);
            int4* cd = reinterpret_cast<int4*>(plane + (size_t)rows * row_bytes);
            // one tensor map: a left tile and a right tile are both row offsets into it
            CUtensorMap tm;
            if (!make_tmap_2d(&tm, plane, 128, rows, 128, 128, BM, true)) return ws.fail("cuTensorMapEncodeTiled failed (u8 matcher)", err);
            match_u8_pack_kernel<<<(rows + 3) / 4, 128, 0, st>>>(ws.at<const PackSet>(meta[gi].sets), (int)g.sets.size(), rows, plane, nk);
            const int n_items = (int)g.items.size();
            const MatchItem* d_items = ws.at<const MatchItem>(meta[gi].items);
            if constexpr (guided) {
                float2* pos = reinterpret_cast<float2*>(plane + (size_t)rows * kMatchU8RowBytes);
                launch_match_coords(ws.at<const MatchCoordSet>(meta[gi].csets), (int)g.sets.size(), rows, pos, st);
                match_u8_guided_kernel<MODE><<<std::min(sms, n_items), TC_THREADS, smem_bytes, st>>>(
                    tm, nk, pos, models, ws.at<const int32_t>(meta[gi].gpair), t2, d_items, n_items, cd);
                ++launches;
            } else {
                match_u8_kernel<<<std::min(sms, n_items), TC_THREADS, smem_bytes, st>>>(tm, nk, d_items, n_items, cd);
            }
            launches += 2;
            nkey = nk; cand = cd;
        }
        const unsigned blocks = (unsigned)((g.left_rows + 127) / 128);
        if constexpr (guided) match_u8_guided_finalize_kernel<<<blocks, 128, 0, st>>>(d_pairs, (int)g.pairs.size(), g.left_rows, nkey, cand, out);
        else match_u8_finalize_kernel<<<blocks, 128, 0, st>>>(d_pairs, (int)g.pairs.size(), g.left_rows, nkey, cand, out);
        ++launches;
    }
    return launches;
}

} // namespace

int run_descriptors_to_u8(const ps_descriptor* in, int n, uint8_t* out, cudaStream_t st)
{
    if (n <= 0) return 0;
    const size_t total = (size_t)n * 128;
    to_u8_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float*>(in), total, out);
    return 1;
}

int run_match_u8_batch(const uint8_t* const* sets, const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs,
                       int32_t* out, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    if (n_pairs <= 0) return 0;
    return run_u8_batch<kUnguided>(sets, nullptr, nullptr, n_desc, n_sets, pairs, n_pairs, nullptr, 0.0f, out, match_choice(flags), st, err);
}

int run_match_u8_guided_batch(const uint8_t* const* sets, const ps_feature* const* feat, const int32_t* const* rev,
                              const int32_t* n_desc, int n_sets, const int32_t* pairs, int n_pairs, const float* models, int model,
                              float threshold, int32_t* out, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    if (n_pairs <= 0) return 0;
    flags = match_choice(flags);
    const float t2 = threshold * threshold;
    return model == kGuidedH ? run_u8_batch<kGuidedH>(sets, feat, rev, n_desc, n_sets, pairs, n_pairs, models, t2, out, flags, st, err)
                             : run_u8_batch<kGuidedF>(sets, feat, rev, n_desc, n_sets, pairs, n_pairs, models, t2, out, flags, st, err);
}

} // namespace psb
