// Device-wide exclusive scan and stable LSD radix sort (8-bit digits) without a library, shared by the track builder
// (k_tracks.cu), bundle adjustment's camera-major order (k_bundle.cu) and global positioning's (k_global.cu).  Both are
// deterministic: no floating point, and every entry's output position depends only on the input.  Also the CTA sum of
// doubles the solvers use, in a fixed order.
#pragma once
#include <cuda_runtime.h>

namespace psb {

namespace {

constexpr int kScanT = 1024;            // threads of a scan block
constexpr int kScanPer = 4;             // consecutive elements per scan thread
constexpr long long kScanChunk = (long long)kScanT * kScanPer;
constexpr int kRadixT = 256;            // threads of a radix block: one per digit
constexpr int kRadixRounds = 16;        // rounds of kRadixT elements per radix tile
constexpr long long kRadixTile = (long long)kRadixT * kRadixRounds;

// ---- deterministic CTA sums of doubles (bundle adjustment, global poses)

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// N values summed over a CTA of NT threads: xor butterflies within warps, then the warps in index order; the result is
// valid in thread 0
template <int N, int NT>
__device__ void cta_sum(double (&v)[N])
{
    __shared__ double part[NT / 32][N];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        const double s = warp_sum(v[k]);
        if (lane == 0) part[w][k] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            double s = part[0][k];
            for (int q = 1; q < NT / 32; ++q) s += part[q][k];
            v[k] = s;
        }
    }
    __syncthreads();
}

// ---- device-wide exclusive scan: blocks of kScanChunk elements, the block sums scanned recursively, then added back

template <class T>
__global__ void __launch_bounds__(kScanT) scan_block_kernel(T* data, long long n, T* __restrict__ sums)
{
    __shared__ T warp_sum[kScanT / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long base = blockIdx.x * kScanChunk + (long long)threadIdx.x * kScanPer;
    T v[kScanPer];
    T own = 0;
#pragma unroll
    for (int k = 0; k < kScanPer; ++k) {
        const T x = base + k < n ? data[base + k] : T(0);
        v[k] = own;
        own += x;
    }
    T inc = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sum[w] = inc;
    __syncthreads();
    if (w == 0) {
        const T x = warp_sum[lane];
        T xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, xi, o);
            if (lane >= o) xi += y;
        }
        warp_sum[lane] = xi - x;
    }
    __syncthreads();
    const T off = warp_sum[w] + inc - own;
#pragma unroll
    for (int k = 0; k < kScanPer; ++k)
        if (base + k < n) data[base + k] = v[k] + off;
    if (threadIdx.x == kScanT - 1) sums[blockIdx.x] = off + own;
}

template <class T>
__global__ void __launch_bounds__(kScanT) scan_add_kernel(T* __restrict__ data, long long n, const T* __restrict__ sums)
{
    const T s = sums[blockIdx.x];
    const long long base = blockIdx.x * kScanChunk + (long long)threadIdx.x * kScanPer;
#pragma unroll
    for (int k = 0; k < kScanPer; ++k)
        if (base + k < n) data[base + k] += s;
}

// elements of partial sums every level of a scan of n elements needs
inline long long scan_partials(long long n)
{
    long long total = 0;
    do {
        n = (n + kScanChunk - 1) / kScanChunk;
        total += n;
    } while (n > 1);
    return total;
}

// data[0, n) becomes its exclusive prefix sum; *total (device) the sum of all; partial: scan_partials(n) elements
template <class T>
int scan_exclusive(T* data, long long n, T* partial, T* total, cudaStream_t st)
{
    const unsigned nb = (unsigned)((n + kScanChunk - 1) / kScanChunk);
    if (nb <= 1) {
        scan_block_kernel<T><<<1, kScanT, 0, st>>>(data, n, total);
        return 1;
    }
    scan_block_kernel<T><<<nb, kScanT, 0, st>>>(data, n, partial);
    const int launches = scan_exclusive(partial, (long long)nb, partial + nb, total, st);
    scan_add_kernel<T><<<nb, kScanT, 0, st>>>(data, n, partial);
    return launches + 2;
}

// ---- stable LSD radix sort of int values by an int key, 8 bits per pass.  Key is a functor: key(v) is value v's key.
// One pass: radix_hist_kernel (a histogram per tile of kRadixTile entries, digit-major), scan_exclusive of the
// 256 * nb histogram entries, radix_scatter_kernel.

template <class Key>
__global__ void __launch_bounds__(kRadixT) radix_hist_kernel(const int* __restrict__ vals, int A, Key key, int shift, int* __restrict__ hist,
                                                             int nb)
{
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const long long base = blockIdx.x * kRadixTile;
    for (int r = 0; r < kRadixRounds; ++r) {
        const long long i = base + r * kRadixT + threadIdx.x;
        if (i < A) atomicAdd(&h[(key(vals[i]) >> shift) & 255], 1);
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * nb + blockIdx.x] = h[threadIdx.x];
}

// hist: the exclusive scan of the histograms, digit-major, so hist[d * nb + b] is where tile b's first digit-d entry goes.
// Each round of kRadixT entries ranks its entries per digit in index order (warp match + per-warp counts), so the pass is
// stable.
template <class Key>
__global__ void __launch_bounds__(kRadixT) radix_scatter_kernel(const int* __restrict__ vin, int* __restrict__ vout, int A, Key key,
                                                                int shift, const int* __restrict__ hist, int nb)
{
    constexpr int W = kRadixT / 32;
    __shared__ int next[256];      // the next output position of each digit
    __shared__ int wpos[W][256];   // per round: the entries of warp w with digit d, then their first position
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    next[t] = hist[(size_t)t * nb + blockIdx.x];
    const unsigned lt = (1u << lane) - 1u;
    const long long base = blockIdx.x * kRadixTile;
    for (int r = 0; r < kRadixRounds; ++r) {
        for (int k = t; k < W * 256; k += kRadixT) (&wpos[0][0])[k] = 0;
        __syncthreads();
        const long long i = base + r * kRadixT + t;
        const bool valid = i < A;
        const int v = valid ? vin[i] : 0;
        const int d = valid ? (key(v) >> shift) & 255 : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & lt);
        if (valid && rank == 0) wpos[w][d] = __popc(peers);
        __syncthreads();
        int run = next[t];
#pragma unroll
        for (int q = 0; q < W; ++q) {
            const int c = wpos[q][t];
            wpos[q][t] = run;
            run += c;
        }
        next[t] = run;
        __syncthreads();
        if (valid) vout[wpos[w][d] + rank] = v;
        __syncthreads();
    }
}

} // namespace

} // namespace psb
