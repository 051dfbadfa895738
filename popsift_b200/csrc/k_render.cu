// Mesh rendering and texturing, hand-written for sm_90a: ps_mesh_render and ps_mesh_texture (contract in
// include/popsift_b200_render.h).  The per-element math is in k_render.h.
//
// ps_mesh_render, one workspace (views, flags, z-buffer keys, big-triangle list):
//   rd_check_kernel      one thread per triangle: a vertex index outside [0, n_vertices) sets a flag, read back before
//                        anything else runs.
//   memset               every key to kEmptyKey.
//   rd_raster_kernel     one thread per triangle; the views go to shared memory kViewChunk at a time.  Per view: projection,
//                        culling (behind z_near, zero area, empty box) and, when the box has at most kBigTri pixels, the
//                        thread rasterises it itself: a 64-bit atomicMin of (float bits of z) << 32 | m per covered pixel.
//                        Positive floats order like their bit patterns, so the winner does not depend on the order.
//                        Marching-tetrahedra triangles are about one voxel, a few pixels.  Larger boxes are appended to
//                        a list, so that a triangle next to a camera does not stall a warp.
//   rd_big_kernel        a fixed grid of CTAs over the list, one entry per CTA at a time, walking its box in 16 x 16 tiles.
//   rd_resolve_kernel    one launch per view: the keys into d_depth and d_tri, and the covered pixels.
//   The list holds at most one pass of views (max(1, kBigListCap / n_triangles) views), so its memory stays bounded;
//   passes repeat the raster and big kernels over the next views.
// ps_mesh_texture, one workspace (views, flags):
//   rd_check_kernel      as above.
//   tx_select_kernel     one thread per triangle over the views in shared-memory chunks: the facing test, four probes
//                        with a nearest-pixel depth gather each, and the projected area; the best view to d_view.
//   tx_fill_kernel       one thread per texel; a CTA covers kFillT consecutive texels of one atlas row, so rows are
//                        written in contiguous spans rather than cell by cell.
// No floating-point atomics anywhere; the totals are integer warp sums and one atomicAdd per warp.
#include "k_render.h"
#include "ps_internal.h"
#include "popsift_b200_render.h"
#include "workspace.h"

#include <algorithm>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kRasterT = 256;
constexpr int kViewChunk = 64;                 // views per shared-memory chunk
constexpr int kBigTri = 64;                    // box pixels above which a triangle goes to rd_big_kernel
constexpr int kTile = 16, kBigT = kTile * kTile;
constexpr long long kBigListCap = (long long)1 << 24;   // big-list entries of one pass, at least n_triangles
constexpr int kFlatT = 256;
constexpr int kFillT = 256;

static_assert(sizeof(RdView) == 144 && sizeof(TxView) == 184 && sizeof(RdView) % 8 == 0 && sizeof(TxView) % 8 == 0, "view layout");

__device__ __forceinline__ void load_vertex(const ps_mesh_vertex* __restrict__ V, int i, double* X)
{
    for (int k = 0; k < 3; ++k) X[k] = (double)__ldg(&V[i].X[k]);
}

__device__ __forceinline__ void warp_total(unsigned long long* dst, unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, v);
}

template <class T>
__device__ __forceinline__ void load_chunk(T* dst, const T* src, int n)
{
    const uint64_t* s = reinterpret_cast<const uint64_t*>(src);
    uint64_t* d = reinterpret_cast<uint64_t*>(dst);
    for (int w = threadIdx.x; w < n * (int)(sizeof(T) / 8); w += blockDim.x) d[w] = s[w];
}

__global__ void __launch_bounds__(kFlatT) rd_check_kernel(const int32_t* __restrict__ T, int n_tri, long long n_vertices, int* flag)
{
    const int m = blockIdx.x * kFlatT + threadIdx.x;
    if (m >= n_tri) return;
    for (int k = 0; k < 3; ++k) {
        const long long i = __ldg(T + 3 * (size_t)m + k);
        if (i < 0 || i >= n_vertices) *flag = 1;
    }
}

struct RdArgs {
    const RdView* views;
    const ps_mesh_vertex* V;
    const int32_t* T;
    int n_tri;
    double z_near;
    unsigned long long* keys;
    unsigned long long* totals;    // drawn, big, covered
    int2* list;                    // (view, triangle) of the big boxes of this pass
    int* list_n;
};

// steps 1-2 of triangle m in view W: false when it is not drawn
__device__ __forceinline__ bool rd_triangle(const RdView& W, const double (*X)[3], double z_near, double (*p)[2], double* z, double& A,
                                            int* box)
{
    for (int k = 0; k < 3; ++k)
        if (!rd_project(W.K, W.R, W.t, X[k], z_near, p[k], z[k])) return false;
    return rd_setup(p, W.w, W.h, A, box);
}

__device__ __forceinline__ void rd_pixel(const RdArgs& a, const RdView& W, const double (*p)[2], const double* z, double A, int m, int x, int y)
{
    float zf;
    if (rd_cover(p, z, A, x, y, zf)) atomicMin(a.keys + W.off + (size_t)y * W.w + x, rd_key(zf, m));
}

__global__ void __launch_bounds__(kRasterT) rd_raster_kernel(const RdArgs a, int v_begin, int v_end)
{
    __shared__ RdView sv[kViewChunk];
    const int m = blockIdx.x * kRasterT + threadIdx.x;
    const bool in = m < a.n_tri;
    double X[3][3];
    if (in)
        for (int k = 0; k < 3; ++k) load_vertex(a.V, __ldg(a.T + 3 * (size_t)m + k), X[k]);
    unsigned long long drawn = 0, big = 0;
    for (int v0 = v_begin; v0 < v_end; v0 += kViewChunk) {
        const int nv = min(kViewChunk, v_end - v0);
        __syncthreads();   // the previous chunk is no longer read
        load_chunk(sv, a.views + v0, nv);
        __syncthreads();
        if (!in) continue;
        for (int v = 0; v < nv; ++v) {
            const RdView& W = sv[v];
            double p[3][2], z[3], A;
            int box[4];
            if (!rd_triangle(W, X, a.z_near, p, z, A, box)) continue;
            ++drawn;
            if ((long long)(box[1] - box[0] + 1) * (box[3] - box[2] + 1) > kBigTri) {
                ++big;
                a.list[atomicAdd(a.list_n, 1)] = make_int2(v0 + v, m);
                continue;
            }
            for (int y = box[2]; y <= box[3]; ++y)
                for (int x = box[0]; x <= box[1]; ++x) rd_pixel(a, W, p, z, A, m, x, y);
        }
    }
    warp_total(a.totals, drawn);
    warp_total(a.totals + 1, big);
}

__global__ void __launch_bounds__(kBigT) rd_big_kernel(const RdArgs a)
{
    const int n = *a.list_n;
    const int tx = threadIdx.x % kTile, ty = threadIdx.x / kTile;
    for (int e = blockIdx.x; e < n; e += gridDim.x) {
        const int2 en = a.list[e];
        const RdView& W = a.views[en.x];
        double X[3][3];
        for (int k = 0; k < 3; ++k) load_vertex(a.V, __ldg(a.T + 3 * (size_t)en.y + k), X[k]);
        double p[3][2], z[3], A;
        int box[4];
        if (!rd_triangle(W, X, a.z_near, p, z, A, box)) continue;   // never: the raster kernel drew it
        const int ntx = (box[1] - box[0]) / kTile + 1, nty = (box[3] - box[2]) / kTile + 1;
        for (int t = 0; t < ntx * nty; ++t) {
            const int x = box[0] + (t % ntx) * kTile + tx, y = box[2] + (t / ntx) * kTile + ty;
            if (x <= box[1] && y <= box[3]) rd_pixel(a, W, p, z, A, en.y, x, y);
        }
    }
}

__global__ void __launch_bounds__(kFlatT) rd_resolve_kernel(const unsigned long long* __restrict__ keys, long long n, float* __restrict__ depth,
                                                            int32_t* __restrict__ tri, unsigned long long* covered)
{
    const long long i = (long long)blockIdx.x * kFlatT + threadIdx.x;
    unsigned long long c = 0;
    if (i < n) {
        const unsigned long long k = keys[i];
        const bool hit = k != kEmptyKey;
        depth[i] = hit ? __uint_as_float((unsigned)(k >> 32)) : 0.0f;
        tri[i] = hit ? (int32_t)(uint32_t)k : -1;
        c = hit;
    }
    warp_total(covered, c);
}

struct TxArgs {
    const TxView* views;
    int n_views;
    const ps_mesh_vertex* V;
    const int32_t* T;
    int n_tri;
    double z_near, tol1;
    float min_cos;
    int cell, cpr, W;
    uint8_t* atlas;
    int32_t* view;
    unsigned long long* totals;    // viewed, fallback
};

__global__ void __launch_bounds__(kFlatT) tx_select_kernel(const TxArgs a)
{
    __shared__ TxView sv[kViewChunk];
    const int m = blockIdx.x * kFlatT + threadIdx.x;
    const bool in = m < a.n_tri;
    double P[4][3], n[3];
    if (in) {
        for (int k = 0; k < 3; ++k) load_vertex(a.V, __ldg(a.T + 3 * (size_t)m + k), P[k]);
        tx_frame(P[0], P[1], P[2], P[3], n);
    }
    int best = -1;
    double best_score = -1.0;
    for (int v0 = 0; v0 < a.n_views; v0 += kViewChunk) {
        const int nv = min(kViewChunk, a.n_views - v0);
        __syncthreads();
        load_chunk(sv, a.views + v0, nv);
        __syncthreads();
        if (!in) continue;
        for (int v = 0; v < nv; ++v) {
            const TxView& V = sv[v];
            if (!tx_facing(n, P[3], V.c, a.min_cos)) continue;
            double p[4][2];
            bool ok = true;
            for (int k = 0; k < 4 && ok; ++k) ok = tx_probe(V, P[k], a.z_near, a.tol1, p[k]);
            if (!ok) continue;
            const double score = fabs(rd_edge(p[0], p[1], p[2][0], p[2][1])) / 2.0;
            if (score > best_score) {
                best_score = score;
                best = v0 + v;
            }
        }
    }
    if (in) a.view[m] = best;
    warp_total(a.totals, in && best >= 0);
    warp_total(a.totals + 1, in && best < 0);
}

__global__ void __launch_bounds__(kFillT) tx_fill_kernel(const TxArgs a)
{
    const int X = blockIdx.x * kFillT + threadIdx.x, Y = blockIdx.y;
    if (X >= a.W) return;
    const int cx = X / a.cell, cy = Y / a.cell;
    const long long m = (long long)cy * a.cpr + cx;
    uint8_t out = 0;
    if (m < a.n_tri) {
        double u, v;
        tx_uv(X - cx * a.cell, Y - cy * a.cell, a.cell, u, v);
        const double b[3] = {1.0 - u - v, u, v};
        double Xw[3] = {0.0, 0.0, 0.0};
        float g[3];
        for (int k = 0; k < 3; ++k) {
            const ps_mesh_vertex* q = a.V + __ldg(a.T + 3 * (size_t)m + k);
            for (int c = 0; c < 3; ++c) Xw[c] += b[k] * (double)__ldg(&q->X[c]);
            g[k] = __ldg(&q->grey);
        }
        const int vi = a.view[m];
        double S;
        if (vi >= 0) {
            const TxView& V = a.views[vi];
            double p[2], z;
            rd_project(V.K, V.R, V.t, Xw, -INFINITY, p, z);
            S = tx_bilinear(V.img, V.pitch, V.w, V.h, p[0], p[1]);
        } else {
            S = b[0] * (double)g[0] + b[1] * (double)g[1] + b[2] * (double)g[2];
        }
        out = tx_round(S);
    }
    a.atlas[(size_t)Y * a.W + X] = out;
}

} // namespace

int run_mesh_render(int n_views, const int32_t* sizes, const ps_camera* cams, const ps_rigid* poses, const ps_mesh_vertex* d_vertices,
                    int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles, const ps_render_params& prm, float* const* d_depth,
                    int32_t* const* d_tri, ps_render_report* report, bool* bad, cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad = false;
    const int n_tri = (int)n_triangles;
    std::vector<RdView> views(n_views);
    long long total = 0;
    for (int v = 0; v < n_views; ++v) {
        RdView& V = views[v];
        V.K[0] = cams[v].fx; V.K[1] = cams[v].fy; V.K[2] = cams[v].cx; V.K[3] = cams[v].cy;
        std::memcpy(V.R, poses[v].R, sizeof(V.R));
        std::memcpy(V.t, poses[v].t, sizeof(V.t));
        V.off = total;
        V.w = sizes[2 * v];
        V.h = sizes[2 * v + 1];
        total += (long long)V.w * V.h;
    }
    const int per_pass = n_tri > 0 ? (int)std::max<long long>(1, std::min<long long>(n_views, kBigListCap / n_tri)) : n_views;
    const int n_pass = (n_views + per_pass - 1) / per_pass;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (mesh render)", "mesh render: plan upload failed");
    const size_t o_views = ws.put(views.data(), views.size() * sizeof(RdView));
    const size_t o_tot = ws.put(nullptr, 3 * sizeof(unsigned long long)), o_flag = ws.put(nullptr, sizeof(int));
    const size_t o_cnt = ws.put(nullptr, (size_t)n_pass * sizeof(int));
    const size_t o_keys = ws.take((size_t)total * sizeof(unsigned long long));
    const size_t o_list = ws.take((size_t)n_tri * per_pass * sizeof(int2));
    if (!ws.alloc(err)) return -1;
    int launches = 0;
    RdArgs a;
    a.views = ws.at<const RdView>(o_views);
    a.V = d_vertices;
    a.T = d_triangles;
    a.n_tri = n_tri;
    a.z_near = (double)prm.z_near;
    a.keys = ws.at<unsigned long long>(o_keys);
    a.totals = ws.at<unsigned long long>(o_tot);
    a.list = ws.at<int2>(o_list);
    if (n_tri > 0) {
        int flag = 0;
        rd_check_kernel<<<blocks_for(n_tri, kFlatT), kFlatT, 0, st>>>(d_triangles, n_tri, (long long)n_vertices, ws.at<int>(o_flag));
        ++launches;
        if (!read_back(&flag, ws.at<int>(o_flag), sizeof(int), st)) return ws.fail("mesh render: read-back failed", err);
        if (flag) {
            *bad = true;
            return launches;
        }
    }
    if (cudaMemsetAsync(a.keys, 0xff, (size_t)total * sizeof(unsigned long long), st) != cudaSuccess)
        return ws.fail("mesh render: cudaMemsetAsync failed", err);
    for (int q = 0; q < n_pass && n_tri > 0; ++q) {
        const int vb = q * per_pass, ve = std::min(n_views, vb + per_pass);
        a.list_n = ws.at<int>(o_cnt) + q;
        rd_raster_kernel<<<blocks_for(n_tri, kRasterT), kRasterT, 0, st>>>(a, vb, ve);
        rd_big_kernel<<<sm_count() * 4, kBigT, 0, st>>>(a);
        launches += 2;
    }
    for (int v = 0; v < n_views; ++v) {
        const long long n = (long long)views[v].w * views[v].h;
        rd_resolve_kernel<<<blocks_for(n, kFlatT), kFlatT, 0, st>>>(a.keys + views[v].off, n, d_depth[v], d_tri[v], a.totals + 2);
        ++launches;
    }
    unsigned long long tot[3];
    if (!read_back(tot, a.totals, sizeof(tot), st)) return ws.fail("mesh render: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    report->n_drawn = (int64_t)tot[0];
    report->n_big = (int64_t)tot[1];
    report->n_covered = (int64_t)tot[2];
    return launches;
}

int run_mesh_texture(int n_views, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, const float* const* d_depth,
                     const ps_mesh_vertex* d_vertices, int64_t n_vertices, const int32_t* d_triangles, int64_t n_triangles,
                     const ps_texture_params& prm, uint8_t* d_atlas, int32_t* d_view, ps_texture_report* report, bool* bad,
                     cudaStream_t st, const char** err)
{
    *err = nullptr;
    *bad = false;
    const int n_tri = (int)n_triangles;
    std::vector<TxView> views(n_views);
    for (int v = 0; v < n_views; ++v) {
        TxView& V = views[v];
        V.K[0] = cams[v].fx; V.K[1] = cams[v].fy; V.K[2] = cams[v].cx; V.K[3] = cams[v].cy;
        std::memcpy(V.R, poses[v].R, sizeof(V.R));
        std::memcpy(V.t, poses[v].t, sizeof(V.t));
        for (int k = 0; k < 3; ++k) V.c[k] = -(V.R[k] * V.t[0] + V.R[3 + k] * V.t[1] + V.R[6 + k] * V.t[2]);
        V.img = images[v].data;
        V.depth = d_depth[v];
        V.pitch = images[v].pitch;
        V.w = images[v].width;
        V.h = images[v].height;
    }
    Workspace ws(st, "cudaMallocFromPoolAsync failed (mesh texture)", "mesh texture: plan upload failed");
    const size_t o_views = ws.put(views.data(), views.size() * sizeof(TxView));
    const size_t o_tot = ws.put(nullptr, 2 * sizeof(unsigned long long)), o_flag = ws.put(nullptr, sizeof(int));
    if (!ws.alloc(err)) return -1;
    int flag = 0;
    rd_check_kernel<<<blocks_for(n_tri, kFlatT), kFlatT, 0, st>>>(d_triangles, n_tri, (long long)n_vertices, ws.at<int>(o_flag));
    if (!read_back(&flag, ws.at<int>(o_flag), sizeof(int), st)) return ws.fail("mesh texture: read-back failed", err);
    if (flag) {
        *bad = true;
        return 1;
    }
    TxArgs a;
    a.views = ws.at<const TxView>(o_views);
    a.n_views = n_views;
    a.V = d_vertices;
    a.T = d_triangles;
    a.n_tri = n_tri;
    a.z_near = (double)prm.z_near;
    a.tol1 = 1.0 + (double)prm.depth_tol;
    a.min_cos = prm.min_cos;
    a.cell = prm.cell;
    a.cpr = prm.cells_per_row;
    a.W = prm.cells_per_row * prm.cell;
    a.atlas = d_atlas;
    a.view = d_view;
    a.totals = ws.at<unsigned long long>(o_tot);
    const int H = (int)((n_triangles + prm.cells_per_row - 1) / prm.cells_per_row) * prm.cell;
    tx_select_kernel<<<blocks_for(n_tri, kFlatT), kFlatT, 0, st>>>(a);
    tx_fill_kernel<<<dim3(blocks_for(a.W, kFillT), (unsigned)H), kFillT, 0, st>>>(a);
    unsigned long long tot[2];
    if (!read_back(tot, a.totals, sizeof(tot), st)) return ws.fail("mesh texture: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    report->n_viewed = (int64_t)tot[0];
    report->n_fallback = (int64_t)tot[1];
    return 3;
}

} // namespace psb
