// Dense depth maps, hand-written for sm_90a: ps_depth_maps and ps_depth_filter (contract in include/popsift_b200_depth.h).
// The per-pixel math is in k_depth.h.
//
// ps_depth_maps, one workspace (workspace.h) and one launch:
//   dp_sweep_kernel  one CTA per 32 x 16 tile of reference pixels, all references' tiles in one grid from a tile table;
//                    one thread per pixel; two CTAs per SM (64 registers) up to K = 16, so that one computes while the
//                    other waits at a barrier.  The tile plus an r-pixel halo of the reference (minus 128) is read once, and
//                    each thread's A, AA and candidate test are computed once.  Then for each plane and, inside it, each
//                    source: the halo tile is warped into shared memory by the pair's homography and a manual bilinear
//                    interpolation from the u8 rows (NaN marks an invalid sample, so a window with one is NaN); the box
//                    sums of B, BB and AB run separably, rows then columns, in shared memory; each thread finishes its
//                    NCC in double and inserts the cost into its registers' K smallest (K = top_k rounded up to a power
//                    of two, a template parameter).  After the plane's sources each thread updates its running winner,
//                    keeping the previous plane's cost for C- and taking C+ at the next plane.  No cost volume is
//                    stored: the outputs are 9 bytes per pixel.  The totals: __syncthreads_count per CTA, one integer
//                    atomic per CTA and counter.
// ps_depth_filter, one workspace:
//   dp_filter_kernel   one thread per pixel of all references: the consistency count, a flag per pixel.
//   scan_exclusive     k_scan.h's integer scan of the flags: each point's position in (ref, y, x) order.
//   dp_compact_kernel  one thread per pixel: the records of the flagged pixels.
#include "k_depth.h"
#include "k_scan.h"
#include "ps_internal.h"
#include "popsift_b200_depth.h"
#include "workspace.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace psb {

namespace {

constexpr int kTW = 32, kTH = 16, kSweepThreads = kTW * kTH;   // a tile, one pixel per thread
constexpr int kRMax = 7;
constexpr int kHW = kTW + 2 * kRMax, kHH = kTH + 2 * kRMax;      // the largest halo tile
constexpr int kFilterThreads = 256;

// one reference of a ps_depth_maps call (64 bytes)
struct DpRef {
    const uint8_t* img;
    int64_t pitch;
    float* depth;
    float* cost;
    uint8_t* n_src;
    int32_t w, h;
    float iota0, diota;            // plane k: iota0 + k diota
    int32_t src0, n_srcs;          // its pairs
};

// one (reference, source) pair (80 bytes): the homography of step 3 rounded to float and the source image
struct DpPair {
    float H[9], b[3];
    const uint8_t* img;
    int64_t pitch;
    float w, h;
    int32_t iw, ih;
};

struct DpTile {
    int32_t ref;
    uint16_t tx, ty;
};

struct DpSweepArgs {
    const DpRef* refs;
    const DpPair* pairs;
    const DpTile* tiles;
    int n_depths, r, top_k, min_sources;
    float max_cost;
    double floor_m2;               // m^2 min_var
    unsigned long long* totals;    // candidates, depths
};

static_assert(sizeof(DpRef) == 64 && sizeof(DpPair) == 80 && sizeof(DpTile) == 8, "plan layouts");

template <int K>
__global__ void __launch_bounds__(kSweepThreads, K <= 16 ? 2 : 1) dp_sweep_kernel(const DpSweepArgs a)
{
    __shared__ float sR[kHH][kHW];         // the reference tile minus 128 (0 outside the image)
    __shared__ float sS[kHH][kHW];         // the warped source tile minus 128 (NaN where invalid)
    __shared__ float sB[kHH][kTW], sBB[kHH][kTW], sAB[kHH][kTW];   // row sums over 2r + 1 columns
    const DpTile T = a.tiles[blockIdx.x];
    const DpRef R = a.refs[T.ref];
    const int r = a.r, d = 2 * r + 1, hw = kTW + 2 * r, hh = kTH + 2 * r;
    const int tid = threadIdx.x;
    const int x0 = (int)T.tx * kTW - r, y0 = (int)T.ty * kTH - r;
    for (int i = tid; i < hw * hh; i += kSweepThreads) {
        const int hy = i / hw, hx = i - hy * hw;
        const int gx = x0 + hx, gy = y0 + hy;
        const bool in = gx >= 0 && gx < R.w && gy >= 0 && gy < R.h;
        sR[hy][hx] = in ? (float)__ldg(R.img + (size_t)gy * R.pitch + gx) - 128.0f : 0.0f;
    }
    __syncthreads();
    const int lx = tid % kTW, ly = tid / kTW;
    const int x = (int)T.tx * kTW + lx, y = (int)T.ty * kTH + ly;
    const bool cand = x >= r && x <= R.w - 1 - r && y >= r && y <= R.h - 1 - r;
    // A and AA are sums of integers below 2^24: exact in float
    float A = 0.0f, AA = 0.0f;
    for (int i = 0; i < d; ++i)
        for (int j = 0; j < d; ++j) {
            const float v = sR[ly + i][lx + j];
            A += v;
            AA += v * v;
        }
    const double m = (double)(d * d);
    const bool rok = cand && m * (double)AA - (double)A * (double)A > a.floor_m2;
    float best = INFINITY, c_minus = INFINITY, c_plus = INFINITY, prev = INFINITY;
    int k_best = -1, n_best = 0;
    bool want_plus = false;
    for (int k = 0; k < a.n_depths; ++k) {
        const float iota = R.iota0 + (float)k * R.diota;
        float top[K];
#pragma unroll
        for (int j = 0; j < K; ++j) top[j] = INFINITY;
        int nv = 0;
        for (int s = R.src0; s < R.src0 + R.n_srcs; ++s) {
            const DpPair& P = a.pairs[s];
            for (int i = tid; i < hw * hh; i += kSweepThreads) {
                const int hy = i / hw, hx = i - hy * hw;
                float u, v, val = NAN;
                if (dp_warp<float>(P.H, P.b, (float)(x0 + hx), (float)(y0 + hy), iota, P.w, P.h, u, v)) {
                    const int u0 = min((int)floorf(u), P.iw - 2), v0 = min((int)floorf(v), P.ih - 2);
                    const float fu = u - (float)u0, fv = v - (float)v0;
                    const uint8_t* row = P.img + (size_t)v0 * P.pitch + u0;
                    const float i00 = __ldg(row), i01 = __ldg(row + 1), i10 = __ldg(row + P.pitch), i11 = __ldg(row + P.pitch + 1);
                    val = ((1.0f - fv) * ((1.0f - fu) * i00 + fu * i01) + fv * ((1.0f - fu) * i10 + fu * i11)) - 128.0f;
                }
                sS[hy][hx] = val;
            }
            __syncthreads();
            for (int i = tid; i < hh * kTW; i += kSweepThreads) {
                const int hy = i / kTW, cx = i - hy * kTW;
                float b = 0.0f, bb = 0.0f, ab = 0.0f;
                for (int j = 0; j < d; ++j) {
                    const float sv = sS[hy][cx + j];
                    b += sv;
                    bb += sv * sv;
                    ab += sv * sR[hy][cx + j];
                }
                sB[hy][cx] = b;
                sBB[hy][cx] = bb;
                sAB[hy][cx] = ab;
            }
            __syncthreads();
            if (rok) {
                float B = 0.0f, BB = 0.0f, AB = 0.0f;
                for (int i = 0; i < d; ++i) {
                    B += sB[ly + i][lx];
                    BB += sBB[ly + i][lx];
                    AB += sAB[ly + i][lx];
                }
                double c;
                if (!isnan(B) && dp_ncc(m, A, AA, B, BB, AB, a.floor_m2, c)) {
                    dp_insert<K>(top, (float)c);
                    ++nv;
                }
            }
        }
        const float Ck = dp_mean<float, K>(top, nv, a.top_k, a.min_sources);
        if (want_plus) {
            c_plus = Ck;
            want_plus = false;
        }
        if (Ck < best) {
            best = Ck;
            k_best = k;
            n_best = nv;
            c_minus = prev;
            c_plus = INFINITY;
            want_plus = true;
        }
        prev = Ck;
    }
    float depth = 0.0f;
    if (k_best >= 0 && best <= a.max_cost) {
        const float delta = dp_parabola<float>(c_minus, best, c_plus, k_best, a.n_depths);
        depth = 1.0f / ((R.iota0 + (float)k_best * R.diota) + delta * R.diota);
    }
    const bool inside = x < R.w && y < R.h;
    if (inside) {
        const size_t i = (size_t)y * R.w + x;
        R.depth[i] = depth;
        R.cost[i] = k_best >= 0 ? best : INFINITY;
        R.n_src[i] = (uint8_t)(k_best >= 0 ? n_best : 0);
    }
    const int nc = __syncthreads_count(inside && cand), nd = __syncthreads_count(inside && depth > 0.0f);
    if (tid == 0) {
        if (nc) atomicAdd(a.totals, (unsigned long long)nc);
        if (nd) atomicAdd(a.totals + 1, (unsigned long long)nd);
    }
}

// one reference of a ps_depth_filter call (48 bytes)
struct DpFRef {
    const float* depth;
    uint8_t* n_cons;
    const uint8_t* img;
    int64_t pitch;
    int32_t off;                   // its first pixel in the call's pixel order
    int32_t src0, n_srcs;          // its sources that are references: list[src0 .. src0 + n_srcs - 1]
    int32_t pad_;
};

struct DpFilterArgs {
    const DpFRef* refs;
    const DpCam* cams;             // per reference
    const int32_t* list;           // source reference indices
    int n_refs, total, min_consistent;
    double max_reproj, max_diff;
    int32_t* flag;
    unsigned long long* tested;
};

__device__ __forceinline__ int dp_ref_of(const DpFRef* __restrict__ refs, int n_refs, int g)
{
    int lo = 0, hi = n_refs - 1;       // the last reference with off <= g (an empty one shares its offset with the next)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (refs[mid].off <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kFilterThreads) dp_filter_kernel(const DpFilterArgs a)
{
    const int g = blockIdx.x * kFilterThreads + threadIdx.x;
    bool has = false;
    if (g < a.total) {
        const int j = dp_ref_of(a.refs, a.n_refs, g);
        const DpFRef& F = a.refs[j];
        const DpCam& cr = a.cams[j];
        const int i = g - F.off, y = i / cr.w, x = i - y * cr.w;
        const float D = F.depth[i];
        int n = 0;
        if (D > 0.0f) {
            has = true;
            for (int k = F.src0; k < F.src0 + F.n_srcs; ++k) {
                const int js = a.list[k];
                const DpCam& cs = a.cams[js];
                int qx, qy;
                double zs;
                if (!dp_lookup(cr, cs, x, y, D, qx, qy, zs)) continue;
                const float Dq = a.refs[js].depth[(size_t)qy * cs.w + qx];
                if (Dq > 0.0f && dp_consistent(cr, cs, x, y, qx, qy, zs, Dq, a.max_reproj, a.max_diff)) ++n;
            }
        }
        F.n_cons[i] = (uint8_t)min(n, 255);
        a.flag[g] = n >= a.min_consistent ? 1 : 0;
    }
    const int nt = __syncthreads_count(has);
    if (threadIdx.x == 0 && nt) atomicAdd(a.tested, (unsigned long long)nt);
}

__global__ void __launch_bounds__(kFilterThreads) dp_compact_kernel(const DpFilterArgs a, const int32_t* __restrict__ pos,
                                                                    ps_dense_point* __restrict__ out)
{
    const int g = blockIdx.x * kFilterThreads + threadIdx.x;
    if (g >= a.total) return;
    const int j = dp_ref_of(a.refs, a.n_refs, g);
    const DpFRef& F = a.refs[j];
    const DpCam& cr = a.cams[j];
    const int i = g - F.off, y = i / cr.w, x = i - y * cr.w;
    const int n = F.n_cons[i];
    if (n < a.min_consistent) return;
    double X[3];
    dp_backproject(cr, x, y, F.depth[i], X);
    ps_dense_point p;
    p.X[0] = (float)X[0];
    p.X[1] = (float)X[1];
    p.X[2] = (float)X[2];
    p.ref = j;
    p.x = (uint16_t)x;
    p.y = (uint16_t)y;
    p.n_consistent = (uint8_t)n;
    p.grey = __ldg(F.img + (size_t)y * F.pitch + x);
    p.pad_ = 0;
    out[pos[g]] = p;
}

template <int K>
void dp_sweep_launch(unsigned n_tiles, const DpSweepArgs& a, cudaStream_t st)
{
    dp_sweep_kernel<K><<<n_tiles, kSweepThreads, 0, st>>>(a);
}

DpCam dp_cam(const ps_image& im, const ps_camera& c, const ps_rigid& p)
{
    DpCam k;
    k.K[0] = c.fx; k.K[1] = c.fy; k.K[2] = c.cx; k.K[3] = c.cy;
    std::memcpy(k.R, p.R, sizeof(k.R));
    std::memcpy(k.t, p.t, sizeof(k.t));
    k.w = im.width;
    k.h = im.height;
    return k;
}

} // namespace

int run_depth_maps(int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs, const int32_t* refs,
                   const float* ranges, const int32_t* src_start, const int32_t* src_sets, const ps_depth_params& prm,
                   float* const* d_depth, float* const* d_cost, uint8_t* const* d_n_src, ps_depth_report* report, cudaStream_t st,
                   const char** err)
{
    (void)n_sets;
    *err = nullptr;
    std::vector<DpRef> rf(n_refs);
    std::vector<DpPair> pr((size_t)src_start[n_refs]);
    std::vector<DpTile> tiles;
    for (int j = 0; j < n_refs; ++j) {
        const int ri = refs[j];
        const ps_image& im = images[ri];
        DpRef& R = rf[j];
        R.img = im.data;
        R.pitch = im.pitch;
        R.depth = d_depth[j];
        R.cost = d_cost[j];
        R.n_src = d_n_src[j];
        R.w = im.width;
        R.h = im.height;
        const double i0 = 1.0 / (double)ranges[2 * j], i1 = 1.0 / (double)ranges[2 * j + 1];
        R.iota0 = (float)i0;
        R.diota = (float)((i1 - i0) / (prm.n_depths - 1));
        R.src0 = src_start[j];
        R.n_srcs = src_start[j + 1] - src_start[j];
        const DpCam cr = dp_cam(im, cams[ri], poses[ri]);
        for (int s = src_start[j]; s < src_start[j + 1]; ++s) {
            const int si = src_sets[s];
            const DpCam cs = dp_cam(images[si], cams[si], poses[si]);
            double H[9], b[3];
            dp_homography(cr.K, cr.R, cr.t, cs.K, cs.R, cs.t, H, b);
            DpPair& P = pr[s];
            for (int k = 0; k < 9; ++k) P.H[k] = (float)H[k];
            for (int k = 0; k < 3; ++k) P.b[k] = (float)b[k];
            P.img = images[si].data;
            P.pitch = images[si].pitch;
            P.w = (float)images[si].width;
            P.h = (float)images[si].height;
            P.iw = images[si].width;
            P.ih = images[si].height;
        }
        const int ntx = (im.width + kTW - 1) / kTW, nty = (im.height + kTH - 1) / kTH;
        for (int ty = 0; ty < nty; ++ty)
            for (int tx = 0; tx < ntx; ++tx) tiles.push_back(DpTile{j, (uint16_t)tx, (uint16_t)ty});
    }
    // workspace: the plan (references, pairs, tiles) and the two totals
    Workspace ws(st, "cudaMallocFromPoolAsync failed (depth maps)", "depth maps: plan upload failed");
    const size_t o_refs = ws.put(rf.data(), rf.size() * sizeof(DpRef)), o_pairs = ws.put(pr.data(), pr.size() * sizeof(DpPair));
    const size_t o_tiles = ws.put(tiles.data(), tiles.size() * sizeof(DpTile));
    const size_t o_tot = ws.put(nullptr, 2 * sizeof(unsigned long long));
    if (!ws.alloc(err)) return -1;
    DpSweepArgs a;
    a.refs = ws.at<const DpRef>(o_refs);
    a.pairs = ws.at<const DpPair>(o_pairs);
    a.tiles = ws.at<const DpTile>(o_tiles);
    a.n_depths = prm.n_depths;
    a.r = prm.radius;
    a.top_k = prm.top_k;
    a.min_sources = prm.min_sources;
    a.max_cost = prm.max_cost;
    const double m = (double)((2 * prm.radius + 1) * (2 * prm.radius + 1));
    a.floor_m2 = m * m * (double)prm.min_var;
    a.totals = ws.at<unsigned long long>(o_tot);
    const unsigned nt = (unsigned)tiles.size();
    if (prm.top_k <= 1) dp_sweep_launch<1>(nt, a, st);
    else if (prm.top_k <= 2) dp_sweep_launch<2>(nt, a, st);
    else if (prm.top_k <= 4) dp_sweep_launch<4>(nt, a, st);
    else if (prm.top_k <= 8) dp_sweep_launch<8>(nt, a, st);
    else if (prm.top_k <= 16) dp_sweep_launch<16>(nt, a, st);
    else dp_sweep_launch<32>(nt, a, st);
    unsigned long long tot[2];
    if (!read_back(tot, a.totals, sizeof(tot), st)) return ws.fail("depth maps: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    report->n_candidates = (int64_t)tot[0];
    report->n_depths = (int64_t)tot[1];
    return 1;
}

int run_depth_filter(int n_sets, const ps_image* images, const ps_camera* cams, const ps_rigid* poses, int n_refs, const int32_t* refs,
                     const int32_t* src_start, const int32_t* src_sets, const float* const* d_depth, const ps_depth_filter_params& prm,
                     uint8_t* const* d_n_consistent, ps_dense_point* d_points, ps_depth_filter_report* report, cudaStream_t st,
                     const char** err)
{
    *err = nullptr;
    std::vector<int32_t> ref_index(n_sets, -1);
    for (int j = 0; j < n_refs; ++j) ref_index[refs[j]] = j;
    std::vector<DpFRef> rf(n_refs);
    std::vector<DpCam> cm(n_refs);
    std::vector<int32_t> list;
    int64_t total = 0;
    for (int j = 0; j < n_refs; ++j) {
        const int ri = refs[j];
        const ps_image& im = images[ri];
        cm[j] = dp_cam(im, cams[ri], poses[ri]);
        DpFRef& F = rf[j];
        F.depth = d_depth[j];
        F.n_cons = d_n_consistent[j];
        F.img = im.data;
        F.pitch = im.pitch;
        F.off = (int32_t)total;
        F.src0 = (int32_t)list.size();
        for (int s = src_start[j]; s < src_start[j + 1]; ++s)
            if (ref_index[src_sets[s]] >= 0) list.push_back(ref_index[src_sets[s]]);
        F.n_srcs = (int32_t)list.size() - F.src0;
        F.pad_ = 0;
        total += (int64_t)im.width * im.height;
    }
    const long long n = total;
    Workspace ws(st, "cudaMallocFromPoolAsync failed (depth filter)", "depth filter: plan upload failed");
    const size_t o_refs = ws.put(rf.data(), rf.size() * sizeof(DpFRef)), o_cams = ws.put(cm.data(), cm.size() * sizeof(DpCam));
    const size_t o_list = ws.put(list.data(), std::max<size_t>(list.size(), 1) * sizeof(int32_t));
    const size_t o_tot = ws.put(nullptr, 2 * sizeof(unsigned long long));
    const size_t o_flag = ws.take((size_t)n * sizeof(int32_t)), o_part = ws.take((size_t)scan_partials(n) * sizeof(int32_t));
    if (!ws.alloc(err)) return -1;
    DpFilterArgs a;
    a.refs = ws.at<const DpFRef>(o_refs);
    a.cams = ws.at<const DpCam>(o_cams);
    a.list = ws.at<const int32_t>(o_list);
    a.n_refs = n_refs;
    a.total = (int)n;
    a.min_consistent = prm.min_consistent;
    a.max_reproj = prm.max_reproj_error;
    a.max_diff = prm.max_depth_diff;
    a.flag = ws.at<int32_t>(o_flag);
    unsigned long long* tot = ws.at<unsigned long long>(o_tot);
    a.tested = tot;
    dp_filter_kernel<<<blocks_for(n, kFilterThreads), kFilterThreads, 0, st>>>(a);
    int32_t* n_points = reinterpret_cast<int32_t*>(tot + 1);
    const int launched = scan_exclusive<int32_t>(a.flag, n, ws.at<int32_t>(o_part), n_points, st);
    dp_compact_kernel<<<blocks_for(n, kFilterThreads), kFilterThreads, 0, st>>>(a, a.flag, d_points);
    unsigned long long h[2];
    if (!read_back(h, tot, sizeof(h), st)) return ws.fail("depth filter: read-back failed", err);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { *err = cudaGetErrorString(e); return -1; }
    int32_t np;
    std::memcpy(&np, &h[1], sizeof(np));
    report->n_tested = (int64_t)h[0];
    report->n_points = np;
    return launched + 2;
}

} // namespace psb
