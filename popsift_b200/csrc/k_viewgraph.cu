// View-graph cleaning, hand-written for sm_90a: ps_view_graph_filter (contract in include/popsift_b200_viewgraph.h).  The
// cycle error is in k_viewgraph.h, the scan and the radix sort in k_scan.h.
//
// Triangle counting in the usual GPU shape, each triangle found exactly once:
//   vg_used_kernel     per pair: the step-1 rule, the orthonormal rotation in double, each endpoint's degree, the
//                      statistics reset to (0, 0, +inf)
//   vg_orient_kernel   per used pair: oriented from its lower-ranked end u to its higher-ranked end v, rank = (degree,
//                      set id), so every out-list has O(sqrt(pairs)) entries; u's out-degree counted
//   scan of the out-degrees (the CSR offsets), two stable radix sorts of the pair ids (by v, then by u), so each out-list
//   is sorted by set id, and vg_gather_kernel writes each entry's v
//   vg_enum_kernel     one warp per oriented entry u -> v: the lanes take the entries of the shorter of out(u) and
//                      out(v) and binary-search the longer; every common w is the triangle {u, v, w}, found from its
//                      lowest-ranked edge only.  Its cycle error (named a < b < c, not by rank) goes to its three pairs
//                      by integer atomics (u -> v's aggregated over the warp first); the totals by warp-aggregated 64-bit
//                      atomics
//   vg_decide_kernel   per pair: step 5, the counts of the report
//   scan of the keep flags and vg_compact_kernel, when d_kept is given
// Nothing here is a floating-point reduction: counts are integer sums and the smallest error an atomicMin on the bit
// pattern of a non-negative float, so the results do not depend on the order of the updates.
#include "k_scan.h"
#include "k_viewgraph.h"
#include "ps_internal.h"
#include "popsift_b200_viewgraph.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace psb {

namespace {

constexpr int kVgT = 256;                       // threads of every kernel here
constexpr int kVgWarps = kVgT / 32;
constexpr unsigned kVgEnumBlocks = 4096;        // the enumeration's grid (warps stride over the oriented entries)
constexpr unsigned kInfBits = 0x7f800000u;      // +inf as float bits

__global__ void __launch_bounds__(kVgT) vg_used_kernel(const ps_two_view* __restrict__ tv, const int2* __restrict__ ends, int P, int S,
                                                       int min_inliers, double* __restrict__ Rd, int32_t* __restrict__ keys,
                                                       int32_t* __restrict__ deg, ps_cycle_stats* __restrict__ stats)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int2 lr = ends[p];
    float R[9];
    bool fin = true;
    for (int k = 0; k < 9; ++k) {
        R[k] = tv[p].R[k];
        fin = fin && isfinite(R[k]);
    }
    const bool used = tv[p].n_front >= min_inliers && fin && lr.x != lr.y;
    if (used) {
        gl_orthonormal(R, Rd + 9 * (size_t)p);
        atomicAdd(deg + lr.x, 1);
        atomicAdd(deg + lr.y, 1);
    }
    keys[p] = used ? 0 : S;
    stats[p].n_triangles = 0;
    stats[p].n_consistent = 0;
    stats[p].min_error = __uint_as_float(kInfBits);
}

// keys[p] / keyd[p]: the ends u -> v of a used pair, S for an unused one; vals the identity
__global__ void __launch_bounds__(kVgT) vg_orient_kernel(const int2* __restrict__ ends, int P, int S, const int32_t* __restrict__ deg,
                                                         int32_t* __restrict__ keys, int32_t* __restrict__ keyd, int32_t* __restrict__ cnt,
                                                         int32_t* __restrict__ vals)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    vals[p] = p;
    if (keys[p] == S) {
        keyd[p] = S;
        return;
    }
    const int2 lr = ends[p];
    const int dl = deg[lr.x], dr = deg[lr.y];
    const bool l_low = dl < dr || (dl == dr && lr.x < lr.y);
    const int u = l_low ? lr.x : lr.y, v = l_low ? lr.y : lr.x;
    keys[p] = u;
    keyd[p] = v;
    atomicAdd(cnt + u, 1);
}

__global__ void __launch_bounds__(kVgT) vg_gather_kernel(const int32_t* __restrict__ vals, int P, const int32_t* __restrict__ keyd,
                                                         int32_t* __restrict__ adj)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < P) adj[j] = keyd[vals[j]];
}

struct KeyArr {
    const int32_t* key;
    __device__ __forceinline__ int operator()(int k) const { return key[k]; }
};

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the cycle error of the triangle {u, v, w} joined by the pairs p_uv, p_uw, p_vw, with the sets named a < b < c
__device__ __forceinline__ double vg_triangle(int u, int v, int w, int p_uv, int p_uw, int p_vw, const int2* __restrict__ ends,
                                              const double* __restrict__ Rd)
{
    const int a = min(u, min(v, w)), c = max(u, max(v, w)), b = u + v + w - a - c;
    // the pair joining the two sets other than s
    auto other = [&](int s) { return s == w ? p_uv : (s == v ? p_uw : p_vw); };
    const int pab = other(c), pbc = other(a), pca = other(b);
    return vg_cycle_error(Rd + 9 * (size_t)pab, ends[pab].x != a, Rd + 9 * (size_t)pbc, ends[pbc].x != b, Rd + 9 * (size_t)pca,
                          ends[pca].x != c);
}

// off[S + 1]: the out-list offsets (off[S] = the oriented entries); adj / vals: each entry's v and pair id
__global__ void __launch_bounds__(kVgT) vg_enum_kernel(const int32_t* __restrict__ off, int S, const int32_t* __restrict__ adj,
                                                       const int32_t* __restrict__ vals, const int32_t* __restrict__ keys,
                                                       const int32_t* __restrict__ keyd, const int2* __restrict__ ends,
                                                       const double* __restrict__ Rd, double max_err, ps_cycle_stats* __restrict__ stats,
                                                       ps_view_graph_report* __restrict__ rep)
{
    const int lane = threadIdx.x & 31;
    const int n_warps = gridDim.x * kVgWarps;
    const int m = off[S];
    unsigned long long nt = 0, nc = 0;
    for (int j = blockIdx.x * kVgWarps + (threadIdx.x >> 5); j < m; j += n_warps) {
        const int p = vals[j];
        const int u = keys[p], v = keyd[p];
        const int ua = off[u], un = off[u + 1] - ua, va = off[v], vn = off[v + 1] - va;
        const bool u_short = un <= vn;
        const int sa = u_short ? ua : va, sn = u_short ? un : vn;
        const int la = u_short ? va : ua, ln = u_short ? vn : un;
        int t_uv = 0, c_uv = 0;
        unsigned m_uv = kInfBits;
        for (int i = lane; i < sn; i += 32) {
            const int w = adj[sa + i];
            int lo = 0, hi = ln;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (adj[la + mid] < w) lo = mid + 1; else hi = mid;
            }
            if (lo == ln || adj[la + lo] != w) continue;
            const int ps = vals[sa + i], pl = vals[la + lo];
            const int p_uw = u_short ? ps : pl, p_vw = u_short ? pl : ps;
            const double e = vg_triangle(u, v, w, p, p_uw, p_vw, ends, Rd);
            const bool ok = e <= max_err;
            const unsigned bits = __float_as_uint((float)e);
            ++t_uv;
            c_uv += ok;
            m_uv = min(m_uv, bits);
            ++nt;
            nc += ok;
            for (const int q : {p_uw, p_vw}) {
                atomicAdd(&stats[q].n_triangles, 1);
                if (ok) atomicAdd(&stats[q].n_consistent, 1);
                atomicMin(reinterpret_cast<unsigned*>(&stats[q].min_error), bits);
            }
        }
        t_uv = __reduce_add_sync(0xffffffffu, t_uv);
        c_uv = __reduce_add_sync(0xffffffffu, c_uv);
        m_uv = __reduce_min_sync(0xffffffffu, m_uv);
        if (lane == 0 && t_uv > 0) {
            atomicAdd(&stats[p].n_triangles, t_uv);
            if (c_uv) atomicAdd(&stats[p].n_consistent, c_uv);
            atomicMin(reinterpret_cast<unsigned*>(&stats[p].min_error), m_uv);
        }
    }
    nt = warp_sum_u64(nt);
    nc = warp_sum_u64(nc);
    if (lane == 0 && nt) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&rep->n_triangles), nt);
        if (nc) atomicAdd(reinterpret_cast<unsigned long long*>(&rep->n_consistent_triangles), nc);
    }
}

// step 5; flag[p] = keep[p] for the compaction's scan
__global__ void __launch_bounds__(kVgT) vg_decide_kernel(int P, int S, const int32_t* __restrict__ keys, const ps_cycle_stats* __restrict__ stats,
                                                         int min_consistent, double min_fraction, int keep_untested,
                                                         uint8_t* __restrict__ keep, int32_t* __restrict__ flag,
                                                         ps_view_graph_report* __restrict__ rep)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    bool used = false, kept = false, untested = false;
    if (p < P) {
        used = keys[p] < S;
        const int nt = stats[p].n_triangles, nc = stats[p].n_consistent;
        untested = used && nt == 0;
        kept = used && (nt > 0 ? nc >= min_consistent && (double)nc >= min_fraction * (double)nt : keep_untested != 0);
        keep[p] = kept ? 1 : 0;
        flag[p] = kept ? 1 : 0;
    }
    const unsigned nu = __reduce_add_sync(0xffffffffu, used ? 1u : 0u);
    const unsigned nk = __reduce_add_sync(0xffffffffu, kept ? 1u : 0u);
    const unsigned nn = __reduce_add_sync(0xffffffffu, untested ? 1u : 0u);
    if ((threadIdx.x & 31) == 0) {
        if (nu) atomicAdd(&rep->n_used, (int)nu);
        if (nk) atomicAdd(&rep->n_kept, (int)nk);
        if (nn) atomicAdd(&rep->n_untested, (int)nn);
    }
}

__global__ void __launch_bounds__(kVgT) vg_compact_kernel(const ps_two_view* __restrict__ tv, int P, const uint8_t* __restrict__ keep,
                                                          const int32_t* __restrict__ pos, ps_two_view* __restrict__ out)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < P && keep[p]) out[pos[p]] = tv[p];
}

} // namespace

int run_view_graph_filter(int n_sets, int n_pairs, const int32_t* pairs, const ps_two_view* d_two_view, const ps_view_graph_params& prm,
                          uint8_t* keep, ps_cycle_stats* stats, ps_two_view* d_kept, ps_view_graph_report* report, cudaStream_t st,
                          const char** err)
{
    *err = nullptr;
    const int S = n_sets, P = n_pairs;
    const int nb = (int)blocks_for(P, kVgT);
    const int nbr = (int)blocks_for(P, kRadixTile);
    Workspace ws(st, "cudaMallocFromPoolAsync failed (view-graph filter)", "view-graph filter: upload failed");
    // staged: the ends, the zeroed degrees and out-degrees; then the report, the statistics and keep, read back in one copy
    const size_t o_ends = ws.put(pairs, (size_t)P * 8), o_deg = ws.put(nullptr, (size_t)S * 4), o_cnt = ws.put(nullptr, ((size_t)S + 1) * 4);
    const size_t o_rep = ws.put(nullptr, sizeof(ps_view_graph_report));
    const size_t o_stats = ws.take((size_t)P * sizeof(ps_cycle_stats), 4), o_keep = ws.take(P, 1);
    const size_t o_R = ws.take((size_t)P * 72), o_flag = ws.take((size_t)P * 4), o_keys = ws.take((size_t)P * 4), o_keyd = ws.take((size_t)P * 4);
    const size_t o_la = ws.take((size_t)P * 4), o_lb = ws.take((size_t)P * 4), o_adj = ws.take((size_t)P * 4);
    const size_t o_hist = ws.take(4ull * 256 * nbr);
    // the partials of the largest scan (the histograms, the offsets or the keep flags), then one slot for the totals
    const long long n_part = scan_partials(std::max<long long>(256ll * nbr, std::max<long long>((long long)S + 1, P)));
    const size_t o_spart = ws.take(4ull * (n_part + 1));
    if (!ws.alloc(err)) return -1;
    const int2* ends = ws.at<const int2>(o_ends);
    int32_t* deg = ws.at<int32_t>(o_deg);
    int32_t* off = ws.at<int32_t>(o_cnt);
    ps_view_graph_report* rep = ws.at<ps_view_graph_report>(o_rep);
    ps_cycle_stats* d_stats = ws.at<ps_cycle_stats>(o_stats);
    uint8_t* d_keep = ws.at<uint8_t>(o_keep);
    double* Rd = ws.at<double>(o_R);
    int32_t* flag = ws.at<int32_t>(o_flag);
    int32_t* keys = ws.at<int32_t>(o_keys);
    int32_t* keyd = ws.at<int32_t>(o_keyd);
    int32_t* la = ws.at<int32_t>(o_la);
    int32_t* lb = ws.at<int32_t>(o_lb);
    int32_t* adj = ws.at<int32_t>(o_adj);
    int32_t* hist = ws.at<int32_t>(o_hist);
    int32_t* spart = ws.at<int32_t>(o_spart);
    int32_t* stotal = spart + n_part;

    int launches = 0;
    vg_used_kernel<<<nb, kVgT, 0, st>>>(d_two_view, ends, P, S, prm.min_inliers, Rd, keys, deg, d_stats);
    vg_orient_kernel<<<nb, kVgT, 0, st>>>(ends, P, S, deg, keys, keyd, off, la);
    launches += 2;
    launches += scan_exclusive(off, (long long)S + 1, spart, stotal, st);
    int bits = 0;
    while (bits < 31 && (S >> bits) != 0) ++bits;      // keys 0 .. S
    for (const int32_t* key : {(const int32_t*)keyd, (const int32_t*)keys}) {
        for (int q = 0; q < (bits + 7) / 8; ++q) {
            radix_hist_kernel<<<nbr, kRadixT, 0, st>>>(la, P, KeyArr{key}, 8 * q, hist, nbr);
            launches += 1 + scan_exclusive(hist, 256ll * nbr, spart, stotal, st);
            radix_scatter_kernel<<<nbr, kRadixT, 0, st>>>(la, lb, P, KeyArr{key}, 8 * q, hist, nbr);
            ++launches;
            std::swap(la, lb);
        }
    }
    vg_gather_kernel<<<nb, kVgT, 0, st>>>(la, P, keyd, adj);
    const unsigned nbe = std::min<unsigned>(blocks_for(P, kVgWarps), kVgEnumBlocks);
    vg_enum_kernel<<<nbe, kVgT, 0, st>>>(off, S, adj, la, keys, keyd, ends, Rd, prm.max_cycle_error, d_stats, rep);
    vg_decide_kernel<<<nb, kVgT, 0, st>>>(P, S, keys, d_stats, prm.min_consistent, prm.min_fraction, prm.keep_untested, d_keep, flag, rep);
    launches += 3;
    if (d_kept) {
        launches += scan_exclusive(flag, (long long)P, spart, stotal, st);
        vg_compact_kernel<<<nb, kVgT, 0, st>>>(d_two_view, P, d_keep, flag, d_kept);
        ++launches;
    }
    // the report, the statistics and keep in one copy
    std::vector<uint8_t> host(o_keep + P - o_rep);
    if (!read_back(host.data(), rep, host.size(), st)) return ws.fail("view-graph filter: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    std::memcpy(report, host.data(), sizeof(ps_view_graph_report));
    if (stats) std::memcpy(stats, host.data() + (o_stats - o_rep), (size_t)P * sizeof(ps_cycle_stats));
    std::memcpy(keep, host.data() + (o_keep - o_rep), P);
    return launches;
}

} // namespace psb
