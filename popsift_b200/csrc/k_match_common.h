// What both brute-force matchers (k_match.cu: float32 descriptors, k_match_u8.cu: 8-bit descriptors) share: the
// mbarrier / TMA / wgmma-descriptor helpers of their persistent tensor-core kernels and the guided matchers' position
// helpers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

#include "popsift_b200.h"

namespace psb {

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

// a plain 1-D bulk copy global -> shared, completing on `bar` (src, dst and bytes multiples of 16)
__device__ __forceinline__ void bulk_copy(void* dst, const void* src, unsigned bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(s32(dst)), "l"(src), "r"(bytes), "r"(s32(bar)) : "memory");
}

// Guided matching: the pixel position of every pooled row of a group, (feat[rev[i]].xpos, .ypos) for the set's row i and
// NaN for padding rows (k_match.cu), so that the kernels' epilogues read a right tile's 128 points as one 1 KB block.
struct MatchCoordSet { const ps_feature* f; const int32_t* rev; int32_t n; int32_t row; };
void launch_match_coords(const MatchCoordSet* d_sets, int n_sets, int rows, float2* out, cudaStream_t st);

// pixel position of descriptor i of a set: its Feature through the reverse map
__device__ __forceinline__ float2 feat_xy(const ps_feature* __restrict__ f, const int32_t* __restrict__ rev, int i)
{
    const ps_feature* p = f + __ldg(rev + i);
    return make_float2(__ldg(&p->xpos), __ldg(&p->ypos));
}

// a pair's 3 x 3 model (row-major)
__device__ __forceinline__ void load_model(float (&m)[9], const float* __restrict__ p)
{
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = __ldg(p + k);
}

} // namespace psb
