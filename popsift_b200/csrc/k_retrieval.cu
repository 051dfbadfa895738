// Image retrieval (include/popsift_b200_retrieval.h): the k-means / VLAD aggregation, the VLAD normalisation and the
// all-vs-all inner products with a top-m per row.  Assignment to the nearest centroid is the batched matcher's best column
// (run_match_batch with the centroids as the right set).
#include "ps_internal.h"
#include "k_match_common.h"
#include "k_retrieval.h"
#include "k_verify_sample.h"
#include "tma_util.h"
#include "workspace.h"

#include <algorithm>
#include <cstring>
#include <vector>

namespace psb {

namespace {

// ---- aggregation

constexpr int kAggChunk = 2048;   // consecutive descriptors of one set per aggregation item

// a chunk of one set: its descriptors, their match rows (3 int32 each, best first)
struct AggItem { const float* x; const int32_t* match; int32_t n; int32_t pad_; };

// Item q, centroid c (blockIdx.y): part[q][c][d] = sum over the chunk's members of c, in descriptor order, of x[d]
// (train) or x[d] - mu_c[d] (encode), in double; cnt[q][c] = the number of members.  Thread d owns dimension d; the
// members are listed in shared memory first (ballot compaction, so in descriptor order).
__global__ void __launch_bounds__(128) vlad_aggregate_kernel(const AggItem* __restrict__ items, const float* __restrict__ mu,
                                                             int sub_mu, int k, double* __restrict__ part, int32_t* __restrict__ cnt)
{
    __shared__ int32_t list[kAggChunk];
    __shared__ int32_t warp_n[4];
    const AggItem it = items[blockIdx.x];
    const int c = blockIdx.y;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    int total = 0;
    for (int i0 = 0; i0 < it.n; i0 += 128) {
        const int i = i0 + t;
        const bool mine = i < it.n && __ldg(it.match + 3 * (size_t)i) == c;
        const unsigned b = __ballot_sync(0xffffffffu, mine);
        if (lane == 0) warp_n[w] = __popc(b);
        __syncthreads();
        int base = total;
        for (int q = 0; q < w; ++q) base += warp_n[q];
        if (mine) list[base + __popc(b & ((1u << lane) - 1u))] = i;
        total += warp_n[0] + warp_n[1] + warp_n[2] + warp_n[3];
        __syncthreads();
    }
    const double m = sub_mu ? (double)__ldg(mu + (size_t)c * 128 + t) : 0.0;
    const float* x = it.x + t;
    double acc = 0.0;
    int j = 0;
    for (; j + 4 <= total; j += 4) {
        // four independent loads in flight, added in order
        const float a0 = __ldg(x + (size_t)list[j] * 128), a1 = __ldg(x + (size_t)list[j + 1] * 128);
        const float a2 = __ldg(x + (size_t)list[j + 2] * 128), a3 = __ldg(x + (size_t)list[j + 3] * 128);
        acc += (double)a0 - m;
        acc += (double)a1 - m;
        acc += (double)a2 - m;
        acc += (double)a3 - m;
    }
    for (; j < total; ++j) acc += (double)__ldg(x + (size_t)list[j] * 128) - m;
    part[((size_t)blockIdx.x * k + c) * 128 + t] = acc;
    if (t == 0) cnt[(size_t)blockIdx.x * k + c] = total;
}

// Segment s (blockIdx.x: a set when encoding, the group's whole pool when training), centroid c (blockIdx.y): the partial
// sums of items seg_first[s] .. seg_first[s+1]-1 added in item order.  accumulate (training): the chain starts from the
// running sum of the earlier groups, so that over all groups it is one chain over the pool's chunks in pool order, the
// same for any grouping; else it starts from zero.
__global__ void __launch_bounds__(128) vlad_merge_kernel(const int32_t* __restrict__ seg_first, const double* __restrict__ part,
                                                         const int32_t* __restrict__ cnt, int k, int accumulate,
                                                         double* __restrict__ sum, long long* __restrict__ count)
{
    const int s = blockIdx.x, c = blockIdx.y, t = threadIdx.x;
    double* o = sum + ((size_t)s * k + c) * 128 + t;
    double acc = accumulate ? *o : 0.0;
    long long n = 0;
    for (int q = seg_first[s]; q < seg_first[s + 1]; ++q) {
        acc += part[((size_t)q * k + c) * 128 + t];
        n += cnt[(size_t)q * k + c];
    }
    *o = acc;
    if (t == 0 && count) count[(size_t)s * k + c] = accumulate ? count[(size_t)s * k + c] + n : n;
}

// k-means update: centroid c = sum / count rounded once to float, unchanged without members
__global__ void __launch_bounds__(128) vlad_update_kernel(const double* __restrict__ sum, const long long* __restrict__ count,
                                                          float* __restrict__ centroids)
{
    const int c = blockIdx.x, t = threadIdx.x;
    const long long n = count[c];
    if (n > 0) centroids[(size_t)c * 128 + t] = (float)(sum[(size_t)c * 128 + t] / (double)n);
}

// deterministic sum over the block's 128 threads (a fixed tree; every thread gets the same value)
__device__ __forceinline__ double block_sum128(double v, double* red)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();                                   // red is free (an earlier call's readers are done)
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    return ((red[0] + red[1]) + red[2]) + red[3];
}

// VLAD normalisation of set blockIdx.x (v: k x 128 doubles, modified in place): every 128-block by its L2 norm, signed
// square root, the whole vector by its L2 norm; written as float
__global__ void __launch_bounds__(128) vlad_normalize_kernel(double* __restrict__ vall, int k, float* __restrict__ out)
{
    __shared__ double red[4];
    const int t = threadIdx.x;
    double* v = vall + (size_t)blockIdx.x * k * 128;
    double ss = 0.0;
    for (int c = 0; c < k; ++c) {
        const double x = v[(size_t)c * 128 + t];
        const double n2 = block_sum128(x * x, red);
        double y = n2 > 0.0 ? x / sqrt(n2) : 0.0;
        y = y < 0.0 ? -sqrt(-y) : sqrt(y);
        v[(size_t)c * 128 + t] = y;
        ss += y * y;
    }
    const double g2 = block_sum128(ss, red);
    const double g = sqrt(g2);
    float* o = out + (size_t)blockIdx.x * k * 128;
    for (int c = 0; c < k; ++c) o[(size_t)c * 128 + t] = g2 > 0.0 ? (float)(v[(size_t)c * 128 + t] / g) : 0.0f;
}

// d_assign[i] = the best column of match row i
__global__ void vlad_assign_kernel(const int32_t* __restrict__ match, int n, int32_t* __restrict__ assign)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) assign[i] = match[3 * (size_t)i];
}

// initial centroids: row c = *src[c]
__global__ void vlad_gather_kernel(const float* const* __restrict__ src, float* __restrict__ centroids)
{
    centroids[(size_t)blockIdx.x * 128 + threadIdx.x] = src[blockIdx.x][threadIdx.x];
}

// ---- similarity + top-m

constexpr int kRT = 128;                        // rows (and columns) of a score tile
constexpr int kRK = 32;                         // floats of a row per k-step: one 128-byte swizzled smem row
constexpr int kRStages = 4;
constexpr int kRThreads = 256;                  // 16 x 16 threads, 8 x 8 scores each
constexpr unsigned kRTileBytes = kRT * kRK * 4; // 16 KB
constexpr size_t kRSmem = (size_t)kRStages * 2 * kRTileBytes + 1024;

struct RTile { int32_t bi, bj; };

// float offset of (row, float quad q) in a SWIZZLE_128B tile of 128-byte rows (base 1024-byte aligned)
__device__ __forceinline__ int swz(int row, int q) { return row * kRK + ((q ^ (row & 7)) << 2); }

// One 128 x 128 tile of scores per block: S[i - r0][j] for rows bi*128.. and columns bj*128.. (mirror: also S[j][i],
// the tile list then holding bj >= bi only).  Each score is one fma chain over d = 0 .. dim-1 (retrieve_fma), no split.
// The tiles of both operands arrive by TMA (SWIZZLE_128B, so that the 16-byte reads of 8 consecutive rows hit distinct
// banks) into a 4-stage ring on full barriers; one __syncthreads per k-step releases a stage.
__global__ void __launch_bounds__(kRThreads, 1) retrieve_score_kernel(const __grid_constant__ CUtensorMap map,
                                                                      const RTile* __restrict__ tiles, int n, int dim, int r0,
                                                                      int mirror, float* __restrict__ S)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    __shared__ __align__(8) uint64_t full[kRStages];
    const RTile tile = tiles[blockIdx.x];
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int nk = (dim + kRK - 1) / kRK;
    if (t == 0) {
        for (int s = 0; s < kRStages; ++s) mb_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](int kt) {
        const int s = kt % kRStages;
        float* a = reinterpret_cast<float*>(smem + (size_t)s * 2 * kRTileBytes);
        mb_expect(&full[s], 2 * kRTileBytes);
        tma_tile(a, &map, kt * kRK, tile.bi * kRT, &full[s]);
        tma_tile(a + kRT * kRK, &map, kt * kRK, tile.bj * kRT, &full[s]);
    };
    if (t == 0)
        for (int kt = 0; kt < kRStages && kt < nk; ++kt) issue(kt);
    float acc[8][8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = 0.0f;
    for (int kt = 0; kt < nk; ++kt) {
        const int s = kt % kRStages;
        mb_wait(&full[s], (kt / kRStages) & 1);
        const float* a = reinterpret_cast<const float*>(smem + (size_t)s * 2 * kRTileBytes);
        const float* b = a + kRT * kRK;
        const int nq = min(kRK / 4, (dim - kt * kRK) >> 2);   // the last step may be partial: no padded fma
#pragma unroll
        for (int q = 0; q < kRK / 4; ++q) {
            if (q < nq) {
                float4 av[8], bv[8];
#pragma unroll
                for (int r = 0; r < 8; ++r) av[r] = *reinterpret_cast<const float4*>(a + swz(ty + 16 * r, q));
#pragma unroll
                for (int c = 0; c < 8; ++c) bv[c] = *reinterpret_cast<const float4*>(b + swz(tx + 16 * c, q));
#pragma unroll
                for (int r = 0; r < 8; ++r)
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        float v = acc[r][c];
                        v = retrieve_fma(av[r].x, bv[c].x, v);
                        v = retrieve_fma(av[r].y, bv[c].y, v);
                        v = retrieve_fma(av[r].z, bv[c].z, v);
                        v = retrieve_fma(av[r].w, bv[c].w, v);
                        acc[r][c] = v;
                    }
            }
        }
        __syncthreads();                                  // every thread is done with stage s
        if (t == 0 && kt + kRStages < nk) issue(kt + kRStages);
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int i = tile.bi * kRT + ty + 16 * r;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int j = tile.bj * kRT + tx + 16 * c;
            if (i < n && j < n) {
                S[(size_t)(i - r0) * n + j] = acc[r][c];
                if (mirror && tile.bi != tile.bj) S[(size_t)j * n + i] = acc[r][c];
            }
        }
    }
}

constexpr int kTopBuf = 2048;                   // candidate buffer of the top-m kernel (u64 keys)
constexpr int kTopThreads = 256;

// ascending bitonic sort of kTopBuf keys in shared memory
__device__ void bitonic_sort(unsigned long long* buf)
{
    for (int size = 2; size <= kTopBuf; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int idx = threadIdx.x; idx < kTopBuf; idx += kTopThreads) {
                const int o = idx ^ stride;
                if (o > idx) {
                    const unsigned long long x = buf[idx], y = buf[o];
                    if ((x > y) == ((idx & size) == 0)) { buf[idx] = y; buf[o] = x; }
                }
            }
            __syncthreads();
        }
}

// Row i = r0 + blockIdx.x of S: the m smallest retrieve_key(S[i][j], j) over j != i.  buf[0, m) is the current top m,
// sorted; candidates below the m-th key are appended after it, and when the buffer could overflow (and at the end) the
// whole buffer is sorted and its first m kept.  Keys are unique (j), so the order of appends does not matter.
__global__ void __launch_bounds__(kTopThreads) retrieve_topm_kernel(const float* __restrict__ S, int n, int r0, int m,
                                                                    int32_t* __restrict__ nbr, float* __restrict__ score)
{
    __shared__ unsigned long long buf[kTopBuf];
    __shared__ int cnt;
    __shared__ unsigned long long thr;
    const int t = threadIdx.x;
    const int i = r0 + blockIdx.x;
    const float* row = S + (size_t)blockIdx.x * n;
    for (int q = t; q < kTopBuf; q += kTopThreads) buf[q] = ~0ull;
    if (t == 0) { cnt = 0; thr = ~0ull; }
    __syncthreads();
    for (int j0 = 0; j0 < n; j0 += kTopThreads) {
        const int j = j0 + t;
        if (j < n && j != i) {
            const unsigned long long key = retrieve_key(row[j], j);
            if (key < thr) buf[m + atomicAdd(&cnt, 1)] = key;
        }
        __syncthreads();
        const int c = cnt;
        __syncthreads();
        if (m + c + kTopThreads > kTopBuf || (j0 + kTopThreads >= n && c > 0)) {
            bitonic_sort(buf);
            for (int q = m + t; q < kTopBuf; q += kTopThreads) buf[q] = ~0ull;
            if (t == 0) { cnt = 0; thr = buf[m - 1]; }
            __syncthreads();
        }
    }
    for (int q = t; q < m; q += kTopThreads) {
        const unsigned long long key = buf[q];
        const int j = (int)(uint32_t)key;
        const bool empty = key == ~0ull;
        nbr[(size_t)i * m + q] = empty ? -1 : j;
        score[(size_t)i * m + q] = empty ? -INFINITY : row[j];
    }
}

} // namespace

// ---- host side

namespace {

// Groups of consecutive sets whose workspace stays under the cap (a set larger than the cap forms a group of its own).
// per_set(n) is the workspace one set of n descriptors needs.
template <class F>
std::vector<std::pair<int, int>> set_groups(int n_sets, const int32_t* n_desc, F per_set)
{
    std::vector<std::pair<int, int>> g;
    const size_t cap = match_workspace_cap();
    int a = 0;
    size_t bytes = 0;
    for (int i = 0; i < n_sets; ++i) {
        const size_t b = per_set(n_desc[i]);
        if (i > a && bytes + b > cap) { g.push_back({a, i}); a = i; bytes = 0; }
        bytes += b;
    }
    if (n_sets > a) g.push_back({a, n_sets});
    return g;
}

size_t chunks_of(int n) { return (size_t)(n + kAggChunk - 1) / kAggChunk; }

// One group's aggregation: items (chunks of the group's sets) and segments (encode: one per set; train: one)
struct AggPlan {
    std::vector<AggItem> items;
    std::vector<int32_t> seg_first;
};

AggPlan agg_plan(const ps_descriptor* const* sets, const int32_t* n_desc, int a, int b, const int32_t* match, bool per_set)
{
    AggPlan p;
    size_t row = 0;
    p.seg_first.push_back(0);
    for (int s = a; s < b; ++s) {
        for (int q0 = 0; q0 < n_desc[s]; q0 += kAggChunk)
            p.items.push_back({reinterpret_cast<const float*>(sets[s]) + (size_t)q0 * 128, match + 3 * (row + q0),
                               std::min(kAggChunk, n_desc[s] - q0), 0});
        row += n_desc[s];
        if (per_set) p.seg_first.push_back((int32_t)p.items.size());
    }
    if (!per_set) p.seg_first.push_back((int32_t)p.items.size());
    return p;
}

// assignment of sets [a, b) to the centroids: match rows of every set against the centroid set
int assign_group(const ps_descriptor* const* sets, const int32_t* n_desc, int a, int b, const float* centroids, int k,
                 int32_t* match, int flags, cudaStream_t st, const char** err)
{
    std::vector<const ps_descriptor*> gs(sets + a, sets + b);
    std::vector<int32_t> gn(n_desc + a, n_desc + b);
    gs.push_back(reinterpret_cast<const ps_descriptor*>(centroids));
    gn.push_back(k);
    std::vector<int32_t> pairs;
    for (int s = 0; s < b - a; ++s) { pairs.push_back(s); pairs.push_back(b - a); }
    return run_match_batch(gs.data(), gn.data(), (int)gs.size(), pairs.data(), b - a, match, flags, st, err);
}

// The workspace regions of the group of sets [a, b), laid out from the start of the workspace (the groups reuse them in
// turn): match rows, partial sums and counts, segment sums, metadata
struct AggWs { size_t rows, match, part, cnt, sum, items, seg_first; };

AggWs agg_layout(Workspace& ws, const int32_t* n_desc, int a, int b, size_t segs, int k)
{
    AggWs L{};
    size_t items = 0;
    for (int s = a; s < b; ++s) { L.rows += n_desc[s]; items += chunks_of(n_desc[s]); }
    ws.rewind(0);
    L.match = ws.take(L.rows * 12);
    L.part = ws.take(items * k * 128 * sizeof(double));
    L.cnt = ws.take(items * k * sizeof(int32_t));
    L.sum = ws.take(segs * k * 128 * sizeof(double));
    L.items = ws.take(items * sizeof(AggItem));
    L.seg_first = ws.take((segs + 1) * sizeof(int32_t));
    return L;
}

} // namespace

static void vlad_draw(uint64_t seed, uint32_t N, int k, uint32_t* idx)
{
    const uint64_t key = verify_mix(seed);
    std::vector<uint32_t> seen;                       // the indices drawn so far, sorted (k <= 1024 of them)
    seen.reserve(k);
    int got = 0;
    for (uint64_t c = 0; got < k; ++c) {
        const uint32_t v = verify_draw(key, (int)c, N);
        const auto at = std::lower_bound(seen.begin(), seen.end(), v);
        if (at != seen.end() && *at == v) continue;
        seen.insert(at, v);
        idx[got++] = v;
    }
}

// the aggregation of one group on `st`: assignment, items, merge, in the group's regions L of ws
static int aggregate_group(const ps_descriptor* const* sets, const int32_t* n_desc, int a, int b, const float* centroids, int k,
                           bool encode, Workspace& ws, const AggWs& L, double* train_sum, long long* train_cnt, int flags,
                           cudaStream_t st, const char** err)
{
    int32_t* match = ws.at<int32_t>(L.match);
    int launches = L.rows > 0 ? assign_group(sets, n_desc, a, b, centroids, k, match, flags, st, err) : 0;
    if (launches < 0) return -1;
    AggPlan plan = agg_plan(sets, n_desc, a, b, match, encode);
    const size_t segs = plan.seg_first.size() - 1;
    ws.stage(L.items, plan.items.data(), plan.items.size() * sizeof(AggItem));
    ws.stage(L.seg_first, plan.seg_first.data(), (segs + 1) * sizeof(int32_t));
    if (!ws.upload()) { *err = "vlad: plan upload failed"; return -1; }
    double* part = ws.at<double>(L.part);
    int32_t* cnt = ws.at<int32_t>(L.cnt);
    if (!plan.items.empty()) {
        vlad_aggregate_kernel<<<dim3((unsigned)plan.items.size(), k), 128, 0, st>>>(ws.at<const AggItem>(L.items), centroids, encode ? 1 : 0,
                                                                                   k, part, cnt);
        ++launches;
    }
    if (encode) {
        if (segs > 0) {
            vlad_merge_kernel<<<dim3((unsigned)segs, k), 128, 0, st>>>(ws.at<const int32_t>(L.seg_first), part, cnt, k, 0, ws.at<double>(L.sum),
                                                                      nullptr);
            ++launches;
        }
    } else {
        vlad_merge_kernel<<<dim3(1, k), 128, 0, st>>>(ws.at<const int32_t>(L.seg_first), part, cnt, k, 1, train_sum, train_cnt);
        ++launches;
    }
    return launches;
}

int run_vlad_train(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, int k, int iters, uint64_t seed,
                   float* centroids, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    flags = match_choice(flags);
    long long N = 0;
    for (int i = 0; i < n_sets; ++i) N += n_desc[i];
    // initialisation: the drawn pool rows
    std::vector<uint32_t> idx(k);
    vlad_draw(seed, (uint32_t)N, k, idx.data());
    std::vector<int64_t> start(n_sets + 1, 0);
    for (int i = 0; i < n_sets; ++i) start[i + 1] = start[i] + n_desc[i];
    std::vector<const float*> src(k);
    for (int c = 0; c < k; ++c) {
        const int s = (int)(std::upper_bound(start.begin(), start.end(), (int64_t)idx[c]) - start.begin()) - 1;
        src[c] = reinterpret_cast<const float*>(sets[s]) + (size_t)(idx[c] - start[s]) * 128;
    }
    const auto groups = set_groups(n_sets, n_desc, [k](int n) { return (size_t)n * 12 + chunks_of(n) * k * (128 * 8 + 4) + 256; });
    // one workspace for the largest group, plus the running sums and counts
    Workspace ws(st, "cudaMallocFromPoolAsync failed (vlad)", "vlad: upload failed");
    for (const auto& g : groups) agg_layout(ws, n_desc, g.first, g.second, 1, k);
    ws.rewind(ws.size());
    const size_t o_sum = ws.take((size_t)k * 128 * 8), o_cnt = ws.take((size_t)k * 8);
    const size_t o_src = ws.put(src.data(), src.size() * sizeof(const float*));
    if (!ws.alloc(err)) return -1;
    vlad_gather_kernel<<<k, 128, 0, st>>>(ws.at<const float* const>(o_src), centroids);
    int launches = 1;
    double* sum = ws.at<double>(o_sum);
    long long* cnt = ws.at<long long>(o_cnt);
    for (int it = 0; it < iters; ++it) {
        if (cudaMemsetAsync(sum, 0, o_src - o_sum, st) != cudaSuccess) return ws.fail("vlad: memset failed", err);
        for (const auto& g : groups) {
            const AggWs L = agg_layout(ws, n_desc, g.first, g.second, 1, k);
            const int n = aggregate_group(sets, n_desc, g.first, g.second, centroids, k, false, ws, L, sum, cnt, flags, st, err);
            if (n < 0) return -1;
            launches += n;
        }
        vlad_update_kernel<<<k, 128, 0, st>>>(sum, cnt, centroids);
        ++launches;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

int run_vlad_encode(const ps_descriptor* const* sets, const int32_t* n_desc, int n_sets, int k, const float* centroids,
                    float* vlad, int32_t* assign, int flags, cudaStream_t st, const char** err)
{
    *err = nullptr;
    flags = match_choice(flags);
    const size_t dim = (size_t)k * 128;
    const auto groups = set_groups(n_sets, n_desc, [k](int n) {
        return (size_t)n * 12 + chunks_of(n) * k * (128 * 8 + 4) + (size_t)k * 128 * 8 + 256; });
    Workspace ws(st, "cudaMallocFromPoolAsync failed (vlad)", "vlad: plan upload failed");
    for (const auto& g : groups) agg_layout(ws, n_desc, g.first, g.second, g.second - g.first, k);
    if (!ws.alloc(err)) return -1;
    int launches = 0;
    size_t row0 = 0;
    for (const auto& g : groups) {
        const int segs = g.second - g.first;
        const AggWs L = agg_layout(ws, n_desc, g.first, g.second, segs, k);
        const int n = aggregate_group(sets, n_desc, g.first, g.second, centroids, k, true, ws, L, nullptr, nullptr, flags, st, err);
        if (n < 0) return -1;
        launches += n;
        vlad_normalize_kernel<<<segs, 128, 0, st>>>(ws.at<double>(L.sum), k, vlad + (size_t)g.first * dim);
        ++launches;
        if (assign && L.rows > 0) {
            vlad_assign_kernel<<<(unsigned)((L.rows + 255) / 256), 256, 0, st>>>(ws.at<const int32_t>(L.match), (int)L.rows, assign + row0);
            ++launches;
        }
        row0 += L.rows;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

int run_retrieve_pairs(int n, const float* vec, int dim, int m, int32_t* nbr, float* score, cudaStream_t st, const char** err)
{
    *err = nullptr;
    if (n <= 0) return 0;
    const int T = (n + kRT - 1) / kRT;
    const size_t row_bytes = (size_t)n * sizeof(float);
    const size_t cap = match_workspace_cap();
    // the whole score matrix when it fits (then only tiles bj >= bi, mirrored); else groups of 128-row blocks, full width
    const bool mirror = (size_t)n * row_bytes <= cap;
    const int grp_tiles = mirror ? T : (int)std::max<size_t>(1, cap / (row_bytes * kRT));
    std::vector<std::vector<RTile>> gtiles;
    for (int b0 = 0; b0 < T; b0 += grp_tiles) {
        gtiles.emplace_back();
        for (int bi = b0; bi < std::min(T, b0 + grp_tiles); ++bi)
            for (int bj = mirror ? bi : 0; bj < T; ++bj) gtiles.back().push_back({bi, bj});
    }
    Workspace ws(st, "cudaMallocFromPoolAsync failed (retrieval)", "retrieval: plan upload failed");
    std::vector<size_t> toff;
    for (const auto& g : gtiles) toff.push_back(ws.put(g.data(), g.size() * sizeof(RTile)));
    const size_t s_rows = std::min<size_t>((size_t)grp_tiles * kRT, (size_t)n);
    const size_t o_S = ws.take(s_rows * row_bytes);
    if (!ws.alloc(err)) return -1;
    CUtensorMap map;
    if (!make_tmap_2d(&map, vec, dim, n, (size_t)dim * sizeof(float), kRK, kRT, true)) return ws.fail("cuTensorMapEncodeTiled failed (retrieval)", err);
    static_assert(kRSmem + kRStages * 8 <= 227 * 1024, "retrieval shared memory");
    cudaFuncSetAttribute(retrieve_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRSmem);
    float* S = ws.at<float>(o_S);
    int launches = 0;
    for (size_t q = 0; q < gtiles.size(); ++q) {
        const int r0 = gtiles[q].front().bi * kRT;
        const int rows = std::min(n, r0 + grp_tiles * kRT) - r0;
        retrieve_score_kernel<<<(unsigned)gtiles[q].size(), kRThreads, kRSmem, st>>>(map, ws.at<const RTile>(toff[q]), n, dim, r0,
                                                                                    mirror ? 1 : 0, S);
        retrieve_topm_kernel<<<rows, kTopThreads, 0, st>>>(S, n, r0, m, nbr, score);
        launches += 2;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

} // namespace psb
