// Feature tracks (include/popsift_b200_tracks.h): connected components of match edges over all features of all sets, with
// the components that hold two features of one set (forks) and the short ones dropped.
//
//   hook      lock-free union-find over an int32 parent array: every edge finds both roots (path halving) and links the
//             larger root under the smaller with atomicCAS(&parent[hi], hi, lo), retrying until both ends share a root.
//             A root only ever gets a smaller parent, so each component's final root is its smallest id, whatever the
//             schedule: the labels are deterministic by construction.
//   compress  parent[v] = root(v): a halving pass, then a read-only pass that writes each node's own entry
//   size      cnt[root] = the component's size (one warp-aggregated atomicAdd per run of equal roots)
//   compact   the active nodes (component size >= 2) in gid order: flags, an exclusive scan, a scatter
//   group     a stable LSD radix sort of the active gids by root (8-bit digits, ceil(bits(N-1) / 8) passes); the key is
//             read through parent[] in every pass, so only the gids move
//   classify  adjacent sorted entries with one root and one set mark the root conflicting (bit 31 of cnt[root])
//   emit      an exclusive scan over the segment heads (the head of a segment is its root, its smallest gid) packs
//             (track index, member position) into one uint64; the heads write d_track_start, the members d_members and
//             d_track_of
// No library sort or scan: both are in k_scan.h.
#include "ps_internal.h"
#include "k_scan.h"
#include "popsift_b200_tracks.h"
#include "workspace.h"

#include <algorithm>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kT = 256;                 // threads of the element-wise kernels
constexpr uint32_t kConflict = 0x80000000u;

__device__ __forceinline__ long long gtid() { return (long long)blockIdx.x * blockDim.x + threadIdx.x; }

// ---- union-find

// the root of x, halving the path on the way (each store replaces a parent by one of its ancestors: safe under
// concurrent finds and links, since a node that is not a root never becomes one again)
__device__ __forceinline__ int find_root(int* parent, int x)
{
    volatile int* p = parent;
    for (;;) {
        const int px = p[x];
        if (px == x) return x;
        const int ppx = p[px];
        if (ppx == px) return px;
        p[x] = ppx;
        x = ppx;
    }
}

// The edge of list entry t: (u, v) of d_edges.  An endpoint outside [0, N) sets *bad and gives no edge.
struct ListEdges {
    const int32_t* edges;
    int32_t N;
    __device__ __forceinline__ bool operator()(long long t, int& u, int& v, int* bad) const
    {
        u = __ldg(edges + 2 * t);
        v = __ldg(edges + 2 * t + 1);
        if ((unsigned)u >= (unsigned)N || (unsigned)v >= (unsigned)N) { *bad = 1; return false; }
        return true;
    }
};

// The edge of correspondence t of the concatenated pairs (TrackPair below): pair p = the last with first[p] <= t, row
// k = row0 + t - first[p] of d_src / d_inlier_mask, i = src[k], b = match[3 (row0 + i)],
// edge = (off_l + rev_l[i], off_r + rev_r[b]).  An index outside its set sets *bad and gives no edge.
struct PairEdges {
    const TrackPair* pairs;
    int n_pairs;
    const int32_t* match;
    const int32_t* src;
    const uint8_t* mask;
    __device__ __forceinline__ bool operator()(long long t, int& u, int& v, int* bad) const
    {
        int lo = 0, hi = n_pairs - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (__ldg(&pairs[mid].first) <= t) lo = mid; else hi = mid - 1;
        }
        const TrackPair& P = pairs[lo];
        const long long k = P.row0 + (t - P.first);
        if (mask && __ldg(mask + k) == 0) return false;
        const int i = __ldg(src + k);
        if ((unsigned)i >= (unsigned)P.n_l) { *bad = 1; return false; }
        const int b = __ldg(match + 3 * (P.row0 + i));
        if ((unsigned)b >= (unsigned)P.n_r) { *bad = 1; return false; }
        const int fu = __ldg(P.rev_l + i), fv = __ldg(P.rev_r + b);
        if ((unsigned)fu >= (unsigned)P.nf_l || (unsigned)fv >= (unsigned)P.nf_r) { *bad = 1; return false; }
        u = P.off_l + fu;
        v = P.off_r + fv;
        return true;
    }
};

template <class Src>
__global__ void __launch_bounds__(kT) tracks_hook_kernel(Src src, long long n, int* __restrict__ parent, int* __restrict__ bad)
{
    const long long t = gtid();
    if (t >= n) return;
    int u, v;
    if (!src(t, u, v, bad) || u == v) return;
    int ru = find_root(parent, u), rv = find_root(parent, v);
    while (ru != rv) {
        const int lo = min(ru, rv), hi = max(ru, rv);
        if (atomicCAS(parent + hi, hi, lo) == hi) break;
        // hi was linked meanwhile: both ends again
        ru = find_root(parent, lo);
        rv = find_root(parent, hi);
    }
}

__global__ void __launch_bounds__(kT) tracks_init_kernel(int* __restrict__ parent, int* __restrict__ cnt, int N)
{
    const long long v = gtid();
    if (v >= N) return;
    parent[v] = (int)v;
    cnt[v] = 0;
}

// Two passes.  The first shortens every path by halving, but a halving store of one thread may land after another
// thread has written its node's root, so an entry may still name a non-root ancestor.  The second walks without storing
// (the paths are short by then) and each thread writes only its own node's root: afterwards parent[v] is v's root.
__global__ void __launch_bounds__(kT) tracks_compress_kernel(int* parent, int N)
{
    const long long v = gtid();
    if (v >= N) return;
    find_root(parent, (int)v);
}

__global__ void __launch_bounds__(kT) tracks_label_kernel(int* parent, int N)
{
    const long long v = gtid();
    if (v >= N) return;
    volatile int* p = parent;
    int x = p[v];
    for (int px = p[x]; px != x; px = p[x]) x = px;
    parent[v] = x;
}

// cnt[root] += the nodes with that root; lanes of a warp with equal roots add once (paths and stars are runs of them)
__global__ void __launch_bounds__(kT) tracks_size_kernel(const int* __restrict__ parent, int* __restrict__ cnt, int N)
{
    const long long v = gtid();
    const int r = v < N ? parent[v] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, r);
    if (r >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cnt + r, __popc(peers));
}

__global__ void __launch_bounds__(kT) tracks_active_kernel(const int* __restrict__ parent, const int* __restrict__ cnt,
                                                           int* __restrict__ flag, int N)
{
    const long long v = gtid();
    if (v >= N) return;
    flag[v] = cnt[parent[v]] >= 2 ? 1 : 0;
}

__global__ void __launch_bounds__(kT) tracks_gather_kernel(const int* __restrict__ parent, const int* __restrict__ cnt,
                                                           const int* __restrict__ pos, int* __restrict__ out, int N)
{
    const long long v = gtid();
    if (v >= N) return;
    if (cnt[parent[v]] >= 2) out[pos[v]] = (int)v;
}

// the radix sort's key of an active gid: its root
struct RootKey {
    const int* parent;
    __device__ __forceinline__ int operator()(int v) const { return parent[v]; }
};

// ---- classify and emit

__device__ __forceinline__ int set_of(const int32_t* __restrict__ off, int n_sets, int g)
{
    int lo = 0, hi = n_sets - 1;    // the last set with off[s] <= g (an empty set shares its offset with the next)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(off + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kT) tracks_conflict_kernel(const int* __restrict__ sorted, int A, const int* __restrict__ parent,
                                                             const int32_t* __restrict__ off, int n_sets, int* __restrict__ cnt)
{
    const long long j = gtid();
    if (j == 0 || j >= A) return;
    const int g = sorted[j], gp = sorted[j - 1];
    const int r = parent[g];
    if (parent[gp] == r && set_of(off, n_sets, g) == set_of(off, n_sets, gp)) atomicOr(reinterpret_cast<unsigned*>(cnt + r), kConflict);
}

// Segment heads (the root itself: the smallest gid of its component) of kept components get (1 << 32 | size), every
// other entry 0; the heads are counted into stat[0..2] (components, conflicting, short).
__global__ void __launch_bounds__(kT) tracks_heads_kernel(const int* __restrict__ sorted, int A, const int* __restrict__ parent,
                                                          const int* __restrict__ cnt, int min_length, unsigned long long* __restrict__ key,
                                                          unsigned* __restrict__ stat)
{
    const long long j = gtid();
    bool head = false, conflict = false, shortc = false;
    unsigned long long k = 0;
    if (j < A) {
        const int g = sorted[j];
        head = parent[g] == g;
        if (head) {
            const unsigned c = (unsigned)cnt[g];
            const unsigned size = c & ~kConflict;
            conflict = (c & kConflict) != 0;
            shortc = !conflict && size < (unsigned)min_length;
            if (!conflict && !shortc) k = (1ull << 32) | size;
        }
        key[j] = k;
    }
    const unsigned nh = __reduce_add_sync(0xffffffffu, head ? 1u : 0u);
    const unsigned nc = __reduce_add_sync(0xffffffffu, conflict ? 1u : 0u);
    const unsigned ns = __reduce_add_sync(0xffffffffu, shortc ? 1u : 0u);
    if ((threadIdx.x & 31) == 0 && nh) {
        atomicAdd(stat + 0, nh);
        if (nc) atomicAdd(stat + 1, nc);
        if (ns) atomicAdd(stat + 2, ns);
    }
}

// after the scan of key: a kept head j of root r writes track_start[t] and leaves cnt[r] = t, base[r] = m0 - j (a
// member at sorted position j' goes to m0 + j' - j); a dropped head leaves cnt[r] = -1.  Thread 0 closes track_start.
__global__ void __launch_bounds__(kT) tracks_start_kernel(const int* __restrict__ sorted, int A, const int* __restrict__ parent,
                                                          int* __restrict__ cnt, const unsigned long long* __restrict__ key,
                                                          const unsigned long long* __restrict__ total, int min_length,
                                                          int* __restrict__ base, int32_t* __restrict__ track_start)
{
    const long long j = gtid();
    if (j == 0) {
        const unsigned long long T = *total;
        track_start[T >> 32] = (int)(uint32_t)T;
    }
    if (j >= A) return;
    const int g = sorted[j];
    if (parent[g] != g) return;
    const unsigned c = (unsigned)cnt[g];
    if ((c & kConflict) || c < (unsigned)min_length) { cnt[g] = -1; return; }
    const unsigned long long s = key[j];
    const int t = (int)(s >> 32), m0 = (int)(uint32_t)s;
    track_start[t] = m0;
    cnt[g] = t;
    base[g] = m0 - (int)j;
}

__global__ void __launch_bounds__(kT) tracks_members_kernel(const int* __restrict__ sorted, int A, const int* __restrict__ parent,
                                                            const int* __restrict__ cnt, const int* __restrict__ base,
                                                            int32_t* __restrict__ members, int32_t* __restrict__ track_of)
{
    const long long j = gtid();
    if (j >= A) return;
    const int g = sorted[j], r = parent[g];
    const int t = cnt[r];
    if (t < 0) return;
    members[base[r] + j] = g;
    track_of[g] = t;
}

// What the host reads back: the bad-edge flag, the active count, the head statistics, the packed totals (and the sum of
// a radix pass's histograms, which nothing reads).
struct Stat {
    int32_t bad, active;
    uint32_t heads[3];
    int32_t hist_total;
    unsigned long long total;
};

template <class MakeSrc>
int run_tracks(int n_sets, const int32_t* n_feat, long long n_items, const std::vector<uint8_t>& plan, MakeSrc make_src, int min_length,
               int32_t* track_of, int32_t* track_start, int32_t* members, ps_track_counts* counts, bool* bad_edge,
               cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad_edge = false;
    std::memset(counts, 0, sizeof(*counts));
    std::vector<int32_t> off(n_sets + 1, 0);
    for (int i = 0; i < n_sets; ++i) off[i + 1] = off[i] + n_feat[i];
    const int N = off[n_sets];
    // workspace: parent, cnt, two gid buffers (4 N bytes each), the scan keys (8 N), the radix histograms, the scan
    // partial sums; then the set offsets, the pair plan and the statistics
    const int nbt = (int)blocks_for(std::max(N, 1), kRadixTile);
    const long long n_hist = 256ll * nbt;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (tracks)", "tracks: upload failed");
    const size_t o_parent = ws.take(4ull * N), o_cnt = ws.take(4ull * N), o_va = ws.take(4ull * N), o_vb = ws.take(4ull * N);
    const size_t o_key = ws.take(8ull * N), o_hist = ws.take(4ull * n_hist);
    const size_t o_part = ws.take(8ull * scan_partials(std::max<long long>({(long long)N, n_hist, 1})));
    const size_t o_off = ws.put(off.data(), 4ull * off.size()), o_plan = ws.put(plan.data(), plan.size());
    const size_t o_stat = ws.take(sizeof(Stat));
    if (!ws.alloc(err)) return -1;
    int* parent = ws.at<int>(o_parent);
    int* cnt = ws.at<int>(o_cnt);
    int* va = ws.at<int>(o_va);
    int* vb = ws.at<int>(o_vb);
    unsigned long long* key = ws.at<unsigned long long>(o_key);
    int* hist = ws.at<int>(o_hist);
    void* part = ws.at<void>(o_part);
    int32_t* d_off = ws.at<int32_t>(o_off);
    Stat* stat = ws.at<Stat>(o_stat);

    if (cudaMemsetAsync(stat, 0, sizeof(Stat), st) != cudaSuccess) return ws.fail("tracks: memset failed", err);
    int launches = 0;
    if (N > 0) {
        tracks_init_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, cnt, N);
        ++launches;
        if (n_items > 0) {
            tracks_hook_kernel<<<blocks_for(n_items, kT), kT, 0, st>>>(make_src(ws.at<uint8_t>(o_plan), N), n_items, parent, &stat->bad);
            ++launches;
        }
        tracks_compress_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, N);
        tracks_label_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, N);
        tracks_size_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, cnt, N);
        tracks_active_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, cnt, vb, N);
        launches += 4 + scan_exclusive(vb, (long long)N, static_cast<int*>(part), &stat->active, st);
        tracks_gather_kernel<<<blocks_for(N, kT), kT, 0, st>>>(parent, cnt, vb, va, N);
        ++launches;
    } else if (n_items > 0) {
        tracks_hook_kernel<<<blocks_for(n_items, kT), kT, 0, st>>>(make_src(ws.at<uint8_t>(o_plan), N), n_items, parent, &stat->bad);
        ++launches;
    }
    Stat h{};
    if (!read_back(&h, stat, sizeof(Stat), st)) return ws.fail("tracks: read-back failed", err);
    if (h.bad) {
        *bad_edge = true;
        return launches;
    }
    const int A = h.active;
    if (N > 0 && cudaMemsetAsync(track_of, 0xff, 4ull * N, st) != cudaSuccess) return ws.fail("tracks: memset failed", err);
    if (A == 0) {
        if (cudaMemsetAsync(track_start, 0, 4, st) != cudaSuccess) return ws.fail("tracks: memset failed", err);
    } else {
        int bits = 0;
        while (bits < 31 && ((N - 1) >> bits) != 0) ++bits;
        const int passes = (bits + 7) / 8;
        const int nb = (int)blocks_for(A, kRadixTile);
        int* src = va;
        int* dst = vb;
        for (int p = 0; p < passes; ++p) {
            radix_hist_kernel<<<nb, kRadixT, 0, st>>>(src, A, RootKey{parent}, 8 * p, hist, nb);
            launches += 1 + scan_exclusive(hist, 256ll * nb, static_cast<int*>(part), &stat->hist_total, st);
            radix_scatter_kernel<<<nb, kRadixT, 0, st>>>(src, dst, A, RootKey{parent}, 8 * p, hist, nb);
            ++launches;
            std::swap(src, dst);
        }
        int* spare = dst;
        tracks_conflict_kernel<<<blocks_for(A, kT), kT, 0, st>>>(src, A, parent, d_off, n_sets, cnt);
        tracks_heads_kernel<<<blocks_for(A, kT), kT, 0, st>>>(src, A, parent, cnt, min_length, key, stat->heads);
        launches += 2 + scan_exclusive(key, (long long)A, static_cast<unsigned long long*>(part), &stat->total, st);
        tracks_start_kernel<<<blocks_for(A, kT), kT, 0, st>>>(src, A, parent, cnt, key, &stat->total, min_length, spare, track_start);
        tracks_members_kernel<<<blocks_for(A, kT), kT, 0, st>>>(src, A, parent, cnt, spare, members, track_of);
        launches += 2;
        if (!read_back(&h, stat, sizeof(Stat), st)) return ws.fail("tracks: read-back failed", err);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    counts->n_tracks = (int32_t)(h.total >> 32);
    counts->n_members = (int32_t)(uint32_t)h.total;
    counts->n_components = (int32_t)h.heads[0];
    counts->n_conflicting = (int32_t)h.heads[1];
    counts->n_short = (int32_t)h.heads[2];
    return launches;
}

} // namespace

int run_tracks_from_edges(int n_sets, const int32_t* n_feat, int n_edges, const int32_t* edges, int min_length, int32_t* track_of,
                          int32_t* track_start, int32_t* members, ps_track_counts* counts, bool* bad_edge, cudaStream_t st,
                          const char** err)
{
    return run_tracks(n_sets, n_feat, n_edges, {}, [edges](uint8_t*, int N) { return ListEdges{edges, N}; }, min_length,
                      track_of, track_start, members, counts, bad_edge, st, err);
}

int run_tracks_from_matches(int n_sets, const int32_t* n_feat, const std::vector<TrackPair>& pairs, const int32_t* match,
                            const int32_t* src, const uint8_t* mask, int min_length, int32_t* track_of, int32_t* track_start,
                            int32_t* members, ps_track_counts* counts, bool* bad_edge, cudaStream_t st, const char** err)
{
    long long n = 0;
    std::vector<TrackPair> live;    // the pairs with correspondences, each with its first index in their concatenation
    for (const TrackPair& p : pairs)
        if (p.n_corr > 0) { live.push_back(p); live.back().first = n; n += p.n_corr; }
    std::vector<uint8_t> plan(live.size() * sizeof(TrackPair));
    if (!live.empty()) std::memcpy(plan.data(), live.data(), plan.size());
    const int np = (int)live.size();
    return run_tracks(n_sets, n_feat, n, plan,
                      [=](uint8_t* d_plan, int) { return PairEdges{reinterpret_cast<const TrackPair*>(d_plan), np, match, src, mask}; },
                      min_length, track_of, track_start, members, counts, bad_edge, st, err);
}

} // namespace psb
