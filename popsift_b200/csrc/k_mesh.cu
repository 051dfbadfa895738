// Surface meshes, hand-written for sm_90a: ps_tsdf_integrate and ps_tsdf_mesh (contract in include/popsift_b200_mesh.h).
// The per-voxel math is in k_mesh.h.
//
// ps_tsdf_integrate, one workspace (the views) and one launch:
//   ts_integrate_kernel  one CTA per 32 x 4 x 4 block of grid points, one thread per point, so each row access is 128
//                        bytes.  The views go to shared memory 64 at a time; for each, 8 lanes project the block's 8
//                        corners and AND their frustum codes (k_mesh.h), a CTA-uniform decision that skips the views that
//                        cannot see the block, so the cost scales with the views that see it.  A point reads its three
//                        values at its first update, folds every view in order in registers and writes them once: at
//                        most 24 bytes per grid point.  The totals: a warp sum, one integer atomic per warp and counter.
// ps_tsdf_mesh, memory O(surface) (no per-voxel scratch):
//   ts_count_kernel      one CTA per 2048 consecutive grid points (cells by their corner 0): the active cells, their
//                        sign-changing edges and their triangles per block.
//   scan_exclusive x 3   k_scan.h's integer scans of the block counts; one read-back of the three totals sizes the rest.
//   ts_emit_kernel       the same classification again, a CTA scan per round: the active cells in cell order with their
//                        first triangle, and their edge keys (8 g + d).
//   radix passes         k_scan.h's stable radix sort of the key indices by the 64-bit keys, one pass per 8 bits of the
//                        largest possible key (5 below 2^34).
//   ts_unique_kernel / scan / ts_unique_compact_kernel   the distinct keys in order: the vertices; their count is the
//                        second read-back.
//   ts_vertex_kernel     one thread per vertex: the edge vertex from its lower endpoint.
//   ts_triangle_kernel   one thread per active cell: its triangles in (tetrahedron, triangle) order, each corner found by
//                        binary search in the vertex keys.
#include "k_mesh.h"
#include "k_scan.h"
#include "ps_internal.h"
#include "popsift_b200_mesh.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kBX = 32, kBY = 4, kBZ = 4, kIntT = kBX * kBY * kBZ;   // one thread per grid point of a block
constexpr int kViewChunk = kIntT / 8;                                 // views per shared-memory chunk: 8 lanes per view
constexpr int kMeshT = 512, kMeshRounds = 4;
constexpr long long kCellBlock = (long long)kMeshT * kMeshRounds;    // grid points per classification CTA
constexpr int kFlatT = 256;

static_assert(sizeof(TsView) == 168 && sizeof(TsView) % 8 == 0, "view layout");

struct TsIntArgs {
    const TsView* views;
    int n_views;
    int nx, ny, nz;
    double origin[3], voxel;
    float* T;
    float* W;
    float* G;
    float trunc;
    int min_consistent;
    unsigned long long* totals;    // updates, points touched
};

__global__ void __launch_bounds__(kIntT) ts_integrate_kernel(const TsIntArgs a)
{
    __shared__ TsView sv[kViewChunk];
    __shared__ uint8_t unseen[kViewChunk];
    const int tid = threadIdx.x;
    const int i0 = blockIdx.x * kBX, j0 = blockIdx.y * kBY, k0 = blockIdx.z * kBZ;
    const int i = i0 + (tid & (kBX - 1)), j = j0 + ((tid / kBX) & (kBY - 1)), k = k0 + tid / (kBX * kBY);
    const int i1 = min(i0 + kBX, a.nx) - 1, j1 = min(j0 + kBY, a.ny) - 1, k1 = min(k0 + kBZ, a.nz) - 1;
    const bool in = i < a.nx && j < a.ny && k < a.nz;
    const size_t g = (size_t)i + (size_t)a.nx * ((size_t)j + (size_t)a.ny * (size_t)k);
    double X[3];
    ts_point(a.origin, a.voxel, i, j, k, X);
    float T = 0.0f, W = 0.0f, G = 0.0f;
    int n_upd = 0;
    for (int v0 = 0; v0 < a.n_views; v0 += kViewChunk) {
        const int nv = min(kViewChunk, a.n_views - v0);
        __syncthreads();   // the previous chunk is no longer read
        const uint64_t* src = reinterpret_cast<const uint64_t*>(a.views + v0);
        uint64_t* dst = reinterpret_cast<uint64_t*>(sv);
        for (int w = tid; w < nv * (int)(sizeof(TsView) / 8); w += kIntT) dst[w] = src[w];
        __syncthreads();
        {
            const int v = tid >> 3, c = tid & 7;
            unsigned code = 0;
            if (v < nv) {
                double Xk[3];
                ts_point(a.origin, a.voxel, (c & 1) ? i1 : i0, (c & 2) ? j1 : j0, (c & 4) ? k1 : k0, Xk);
                code = ts_corner_code(sv[v], Xk);
            }
            code &= __shfl_xor_sync(0xffffffffu, code, 1);
            code &= __shfl_xor_sync(0xffffffffu, code, 2);
            code &= __shfl_xor_sync(0xffffffffu, code, 4);
            if (c == 0 && v < nv) unseen[v] = ts_block_unseen(code) ? 1 : 0;
        }
        __syncthreads();
        if (!in) continue;
        for (int v = 0; v < nv; ++v) {
            if (unseen[v]) continue;
            const TsView& V = sv[v];
            double Xc[3];
            ts_to_camera(V.R, V.t, X, Xc);
            int qx, qy;
            if (!ts_pixel(V.K, V.w, V.h, Xc, qx, qy)) continue;
            const size_t p = (size_t)qy * V.w + qx;
            const float D = __ldg(V.depth + p);
            if (!(D > 0.0f)) continue;
            if (a.min_consistent > 0 && (int)__ldg(V.ncons + p) < a.min_consistent) continue;
            float tau;
            if (!ts_tau(D, Xc[2], a.trunc, tau)) continue;
            if (n_upd == 0) {
                T = a.T[g];
                W = a.W[g];
                G = a.G[g];
            }
            ts_update(T, W, G, tau, (float)__ldg(V.img + (size_t)qy * V.pitch + qx));
            ++n_upd;
        }
    }
    if (in && n_upd) {
        a.T[g] = T;
        a.W[g] = W;
        a.G[g] = G;
    }
    int s = n_upd, t = n_upd > 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    if ((tid & 31) == 0 && s) {
        atomicAdd(a.totals, (unsigned long long)s);
        atomicAdd(a.totals + 1, (unsigned long long)t);
    }
}

struct TsMeshArgs {
    const float* T;
    const float* W;
    const float* G;
    int nx, ny, nz;
    int n;                         // grid points
    float min_weight;
    float o[3], h;
};

// grid point of corner c of the cell at g
__device__ __forceinline__ int ts_corner(const TsMeshArgs& a, int g, int c)
{
    return g + (c & 1) + a.nx * (((c >> 1) & 1) + a.ny * ((c >> 2) & 1));
}

// step 1 for the cell at grid point g (g < n): true when it is active, with the inside corners in mask
__device__ __forceinline__ bool ts_cell(const TsMeshArgs& a, int g, unsigned& mask)
{
    const int i = g % a.nx, r = g / a.nx, j = r % a.ny, k = r / a.ny;
    if (i >= a.nx - 1 || j >= a.ny - 1 || k >= a.nz - 1) return false;
    bool meshed = true;
    mask = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int q = ts_corner(a, g, c);
        meshed &= __ldg(a.W + q) >= a.min_weight;
        mask |= (__ldg(a.T + q) < 0.0f ? 1u : 0u) << c;
    }
    return meshed && mask != 0u && mask != 255u;
}

// one CTA's (active cells, edge entries, triangles) over kCellBlock grid points: cnt[q * nb + block]
__global__ void __launch_bounds__(kMeshT) ts_count_kernel(const TsMeshArgs a, long long* __restrict__ cnt, int nb)
{
    __shared__ int sum[3];
    if (threadIdx.x < 3) sum[threadIdx.x] = 0;
    __syncthreads();
    int v[3] = {0, 0, 0};
    const long long base = blockIdx.x * kCellBlock;
    for (int r = 0; r < kMeshRounds; ++r) {
        const long long g = base + r * kMeshT + threadIdx.x;
        unsigned mask;
        if (g < a.n && ts_cell(a, (int)g, mask)) {
            int ne, nt;
            ts_cell_counts(mask, ne, nt);
            v[0] += 1;
            v[1] += ne;
            v[2] += nt;
        }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        int s = v[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(&sum[q], s);   // integer sums: the order does not matter
    }
    __syncthreads();
    if (threadIdx.x < 3) cnt[(size_t)threadIdx.x * nb + blockIdx.x] = sum[threadIdx.x];
}

// exclusive CTA scan of three counts per thread: ex the thread's offsets, tot the CTA's totals
__device__ __forceinline__ void cta_scan3(const int (&v)[3], int (&ex)[3], int (&tot)[3])
{
    constexpr int NW = kMeshT / 32;
    __shared__ int ws[3][NW];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        int x = v[q];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        inc[q] = x;
        if (lane == 31) ws[q][w] = x;
    }
    __syncthreads();
    if (w == 0) {
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            int x = lane < NW ? ws[q][lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (lane < NW) ws[q][lane] = x;
        }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        ex[q] = (w ? ws[q][w - 1] : 0) + inc[q] - v[q];
        tot[q] = ws[q][NW - 1];
    }
    __syncthreads();   // ws is rewritten by the next call
}

// the active cells of each CTA in cell order (cells, their first triangle in cell_tri) and their edge keys; off: the
// exclusive scans of ts_count_kernel's counts
__global__ void __launch_bounds__(kMeshT) ts_emit_kernel(const TsMeshArgs a, const long long* __restrict__ off, int nb,
                                                         int32_t* __restrict__ cells, long long* __restrict__ cell_tri,
                                                         unsigned long long* __restrict__ keys)
{
    long long o[3] = {off[blockIdx.x], off[(size_t)nb + blockIdx.x], off[2 * (size_t)nb + blockIdx.x]};
    const long long base = blockIdx.x * kCellBlock;
    for (int r = 0; r < kMeshRounds; ++r) {
        const long long g = base + r * kMeshT + threadIdx.x;
        unsigned mask = 0;
        int v[3] = {0, 0, 0};
        if (g < a.n && ts_cell(a, (int)g, mask)) {
            v[0] = 1;
            ts_cell_counts(mask, v[1], v[2]);
        }
        int ex[3], tot[3];
        cta_scan3(v, ex, tot);
        if (v[0]) {
            const long long c = o[0] + ex[0];
            cells[c] = (int32_t)g;
            cell_tri[c] = o[2] + ex[2];
            long long kp = o[1] + ex[1];
            for (int e = 0; e < 19; ++e) {
                const int ca = kCellEdge[e] >> 3, d = kCellEdge[e] & 7;
                if (((mask >> ca) ^ (mask >> (ca + d))) & 1u)
                    keys[kp++] = (unsigned long long)ts_corner(a, (int)g, ca) * 8ull + (unsigned long long)d;
            }
        }
#pragma unroll
        for (int q = 0; q < 3; ++q) o[q] += tot[q];
    }
}

// the 64-bit key of entry v, signed so that the radix kernels' digit stays an int (keys are below 2^34)
struct KeyOf64 {
    const unsigned long long* key;
    __device__ __forceinline__ long long operator()(int v) const { return (long long)key[v]; }
};

__global__ void __launch_bounds__(kFlatT) ts_iota_kernel(int* __restrict__ v, int n)
{
    const int i = blockIdx.x * kFlatT + threadIdx.x;
    if (i < n) v[i] = i;
}

// 1 where the sorted key differs from the one before it
__global__ void __launch_bounds__(kFlatT) ts_unique_kernel(const int* __restrict__ order, const unsigned long long* __restrict__ keys,
                                                           int n, int* __restrict__ flag)
{
    const int i = blockIdx.x * kFlatT + threadIdx.x;
    if (i < n) flag[i] = (i == 0 || keys[order[i]] != keys[order[i - 1]]) ? 1 : 0;
}

__global__ void __launch_bounds__(kFlatT) ts_unique_compact_kernel(const int* __restrict__ order, const unsigned long long* __restrict__ keys,
                                                                   int n, const int* __restrict__ pos, unsigned long long* __restrict__ ukeys)
{
    const int i = blockIdx.x * kFlatT + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = keys[order[i]];
    if (i == 0 || k != keys[order[i - 1]]) ukeys[pos[i]] = k;
}

__global__ void __launch_bounds__(kFlatT) ts_vertex_kernel(const TsMeshArgs a, const unsigned long long* __restrict__ ukeys, int nv,
                                                           ps_mesh_vertex* __restrict__ out)
{
    const int i = blockIdx.x * kFlatT + threadIdx.x;
    if (i >= nv) return;
    const unsigned long long key = ukeys[i];
    const int ga = (int)(key >> 3), d = (int)(key & 7);
    const int gb = ts_corner(a, ga, d);
    const int ax = ga % a.nx, r = ga / a.nx, ay = r % a.ny, az = r / a.ny;
    ps_mesh_vertex p;
    ts_vertex(a.o, a.h, ax, ay, az, d, __ldg(a.T + ga), __ldg(a.T + gb), __ldg(a.G + ga), __ldg(a.G + gb), p.X, p.grey);
    out[i] = p;
}

__device__ __forceinline__ int ts_find(const unsigned long long* __restrict__ ukeys, int nv, unsigned long long key)
{
    int lo = 0, hi = nv - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ukeys[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kFlatT) ts_triangle_kernel(const TsMeshArgs a, const int32_t* __restrict__ cells,
                                                             const long long* __restrict__ cell_tri, int n_cells,
                                                             const unsigned long long* __restrict__ ukeys, int nv,
                                                             int32_t* __restrict__ tris)
{
    const int c = blockIdx.x * kFlatT + threadIdx.x;
    if (c >= n_cells) return;
    const int g = cells[c];
    unsigned mask = 0;
    ts_cell(a, g, mask);
    long long t = cell_tri[c];
    for (int q = 0; q < 6; ++q) {
        const int cs = ts_tet_case(q, mask);
        for (int s = 0; s < kTetTriCount[cs]; ++s, ++t)
            for (int m = 0; m < 3; ++m) {
                const int e = kTetTri[q][cs][s][m];
                const unsigned long long key = (unsigned long long)ts_corner(a, g, e >> 3) * 8ull + (unsigned long long)(e & 7);
                tris[3 * t + m] = ts_find(ukeys, nv, key);
            }
    }
}

TsMeshArgs mesh_args(const ps_volume& vol, float min_weight)
{
    TsMeshArgs a;
    a.T = vol.tsdf;
    a.W = vol.weight;
    a.G = vol.grey;
    a.nx = vol.nx;
    a.ny = vol.ny;
    a.nz = vol.nz;
    a.n = vol.nx * vol.ny * vol.nz;
    a.min_weight = min_weight;
    for (int c = 0; c < 3; ++c) a.o[c] = (float)vol.origin[c];
    a.h = (float)vol.voxel;
    return a;
}

} // namespace

int run_volume_clear(const ps_volume& vol, cudaStream_t st, const char** err)
{
    *err = nullptr;
    const size_t bytes = (size_t)vol.nx * vol.ny * vol.nz * sizeof(float);
    for (float* p : {vol.tsdf, vol.weight, vol.grey})
        if (cudaMemsetAsync(p, 0, bytes, st) != cudaSuccess) {
            cudaGetLastError();
            *err = "volume clear: cudaMemsetAsync failed";
            return -1;
        }
    return 0;
}

int run_tsdf_integrate(int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, const float* const* d_depth,
                       const uint8_t* const* d_n_consistent, const ps_tsdf_params& prm, const ps_volume& vol, ps_tsdf_report* report,
                       cudaStream_t st, const char** err)
{
    *err = nullptr;
    std::vector<TsView> views(n_views);
    for (int v = 0; v < n_views; ++v) {
        TsView& V = views[v];
        V.K[0] = cams[v].fx; V.K[1] = cams[v].fy; V.K[2] = cams[v].cx; V.K[3] = cams[v].cy;
        std::memcpy(V.R, poses[v].R, sizeof(V.R));
        std::memcpy(V.t, poses[v].t, sizeof(V.t));
        V.img = images[v].data;
        V.depth = d_depth[v];
        V.ncons = prm.min_consistent > 0 ? d_n_consistent[v] : nullptr;
        V.pitch = images[v].pitch;
        V.w = images[v].width;
        V.h = images[v].height;
    }
    Workspace ws(st, "cudaMallocFromPoolAsync failed (tsdf integrate)", "tsdf integrate: plan upload failed");
    const size_t o_views = ws.put(views.data(), views.size() * sizeof(TsView)), o_tot = ws.put(nullptr, 2 * sizeof(unsigned long long));
    if (!ws.alloc(err)) return -1;
    TsIntArgs a;
    a.views = ws.at<const TsView>(o_views);
    a.n_views = n_views;
    a.nx = vol.nx;
    a.ny = vol.ny;
    a.nz = vol.nz;
    for (int c = 0; c < 3; ++c) a.origin[c] = vol.origin[c];
    a.voxel = vol.voxel;
    a.T = vol.tsdf;
    a.W = vol.weight;
    a.G = vol.grey;
    a.trunc = prm.trunc;
    a.min_consistent = prm.min_consistent;
    a.totals = ws.at<unsigned long long>(o_tot);
    const dim3 grid((unsigned)((vol.nx + kBX - 1) / kBX), (unsigned)((vol.ny + kBY - 1) / kBY), (unsigned)((vol.nz + kBZ - 1) / kBZ));
    ts_integrate_kernel<<<grid, kIntT, 0, st>>>(a);
    unsigned long long tot[2];
    if (!read_back(tot, a.totals, sizeof(tot), st)) return ws.fail("tsdf integrate: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    report->n_updates = (int64_t)tot[0];
    report->n_voxels_touched = (int64_t)tot[1];
    return 1;
}

int run_tsdf_mesh(const ps_volume& vol, const ps_mesh_params& prm, int64_t max_vertices, int64_t max_triangles, ps_mesh_vertex* d_vertices,
                  int32_t* d_triangles, ps_mesh_report* report, bool* overflow, cudaStream_t st, const char** err)
{
    *err = nullptr;
    *overflow = false;
    const TsMeshArgs a = mesh_args(vol, prm.min_weight);
    const long long n = a.n;
    const int nb = (int)((n + kCellBlock - 1) / kCellBlock);
    // the block counts, their scans' partials (one region, the three scans run in turn) and the totals
    Workspace ws(st, "cudaMallocFromPoolAsync failed (tsdf mesh)", "tsdf mesh: plan upload failed");
    const size_t o_tot = ws.put(nullptr, 3 * sizeof(long long));
    const size_t o_cnt = ws.take(3 * (size_t)nb * sizeof(long long)), o_part = ws.take((size_t)scan_partials(nb) * sizeof(long long));
    if (!ws.alloc(err)) return -1;
    long long* cnt = ws.at<long long>(o_cnt);
    long long* tot = ws.at<long long>(o_tot);
    ts_count_kernel<<<nb, kMeshT, 0, st>>>(a, cnt, nb);
    int launches = 1;
    for (int q = 0; q < 3; ++q) launches += scan_exclusive<long long>(cnt + (size_t)q * nb, nb, ws.at<long long>(o_part), tot + q, st);
    long long h_tot[3];
    if (!read_back(h_tot, tot, sizeof(h_tot), st)) return ws.fail("tsdf mesh: read-back failed", err);
    const long long n_cells = h_tot[0], n_keys = h_tot[1], n_tris = h_tot[2];
    report->n_cells = n_cells;
    report->n_triangles = n_tris;
    report->n_vertices = 0;
    if (n_cells == 0) return launches;
    if (n_keys > 0x7fffffffLL) {
        report->n_vertices = -1;
        *overflow = true;
        return launches;
    }
    const int nk = (int)n_keys;
    const int nbr = (int)((nk + kRadixTile - 1) / kRadixTile);
    int passes = 0;
    for (unsigned long long top = (unsigned long long)n * 8ull - 1ull; top; top >>= 8) ++passes;
    Workspace ws2(st, "cudaMallocFromPoolAsync failed (tsdf mesh surface)", "tsdf mesh: upload failed");
    const size_t o_nv = ws2.put(nullptr, sizeof(int));
    const size_t o_cells = ws2.take((size_t)n_cells * sizeof(int32_t)), o_ctri = ws2.take((size_t)n_cells * sizeof(long long));
    const size_t o_keys = ws2.take((size_t)nk * sizeof(unsigned long long)), o_ukeys = ws2.take((size_t)nk * sizeof(unsigned long long));
    const size_t o_va = ws2.take((size_t)nk * sizeof(int)), o_vb = ws2.take((size_t)nk * sizeof(int));
    const size_t o_hist = ws2.take((size_t)256 * nbr * sizeof(int));
    const size_t o_spart = ws2.take((size_t)scan_partials(std::max<long long>(256ll * nbr, nk)) * sizeof(int));
    if (!ws2.alloc(err)) return -1;
    int32_t* cells = ws2.at<int32_t>(o_cells);
    long long* ctri = ws2.at<long long>(o_ctri);
    unsigned long long* keys = ws2.at<unsigned long long>(o_keys);
    unsigned long long* ukeys = ws2.at<unsigned long long>(o_ukeys);
    int* la = ws2.at<int>(o_va);
    int* lb = ws2.at<int>(o_vb);
    int* hist = ws2.at<int>(o_hist);
    int* spart = ws2.at<int>(o_spart);
    int* d_nv = ws2.at<int>(o_nv);
    ts_emit_kernel<<<nb, kMeshT, 0, st>>>(a, cnt, nb, cells, ctri, keys);
    ts_iota_kernel<<<blocks_for(nk, kFlatT), kFlatT, 0, st>>>(la, nk);
    launches += 2;
    for (int p = 0; p < passes; ++p) {
        radix_hist_kernel<<<nbr, kRadixT, 0, st>>>(la, nk, KeyOf64{keys}, 8 * p, hist, nbr);
        launches += 1 + scan_exclusive(hist, 256ll * nbr, spart, d_nv, st);
        radix_scatter_kernel<<<nbr, kRadixT, 0, st>>>(la, lb, nk, KeyOf64{keys}, 8 * p, hist, nbr);
        ++launches;
        std::swap(la, lb);
    }
    ts_unique_kernel<<<blocks_for(nk, kFlatT), kFlatT, 0, st>>>(la, keys, nk, lb);
    launches += 1 + scan_exclusive(lb, (long long)nk, spart, d_nv, st);
    ts_unique_compact_kernel<<<blocks_for(nk, kFlatT), kFlatT, 0, st>>>(la, keys, nk, lb, ukeys);
    launches += 1;
    int nv = 0;
    if (!read_back(&nv, d_nv, sizeof(nv), st)) return ws2.fail("tsdf mesh: read-back failed", err);
    report->n_vertices = nv;
    if (nv > max_vertices || n_tris > max_triangles) {
        *overflow = true;
        return launches;
    }
    ts_vertex_kernel<<<blocks_for(nv, kFlatT), kFlatT, 0, st>>>(a, ukeys, nv, d_vertices);
    ts_triangle_kernel<<<blocks_for(n_cells, kFlatT), kFlatT, 0, st>>>(a, cells, ctri, (int)n_cells, ukeys, nv, d_triangles);
    launches += 2;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    return launches;
}

} // namespace psb
