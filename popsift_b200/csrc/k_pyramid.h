// Shared between the two pyramid translation units.
#pragma once
#include "ps_internal.h"

#include <mutex>
#include <set>
#include <utility>

namespace psb {

// opt in to > 48 KB dynamic shared memory once per (kernel, device); safe from any thread
template <typename K>
inline void ensure_smem(K kernel, size_t bytes, bool prefer_max_carveout = false)
{
    static std::mutex mu;
    static std::set<std::pair<const void*, int>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    const std::pair<const void*, int> key(reinterpret_cast<const void*>(kernel), dev);
    std::lock_guard<std::mutex> g(mu);
    if (done.insert(key).second) {
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (prefer_max_carveout)
            cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
}


struct alignas(16) Taps { float g[PS_GAUSS_ALIGN]; };   // one half-kernel, passed by value (constant bank)

// column-marching fast path (k_pyramid_march.cu); return -1 when the radius is not instantiated
int march_blur_level(const OctaveView& o, int level, const Taps& t, int R, float* next0, int next_pitch,
                     const CandSink* sink, cudaStream_t st);
bool march_supports(int R);
// candidate list layout of a level kernel over a w x h plane
int march_cand_blocks(int w, int h);
int march_cand_region(int w, int h);
long long march_cand_entry_bound(int w, int h);
// How level 0 of octave 0 may be evaluated for one geometry (level0_plan, k_pyramid.cu): whether neighbouring outputs can
// share their texture fetches is decided by evaluating the texture unit's coordinate arithmetic for every (column, tap).
enum { LEVEL0_IDEAL_X2 = 0,   // exactly 2x: every fetch has fraction 0 or 1/2 at texels X>>1, (X+1)>>1 (the byte-tile kernel)
       LEVEL0_SHARED   = 1,   // tap `off` of output X fetches what output X+off fetches at its centre: separable staging
       LEVEL0_PER_TAP  = 2 }; // neither: every tap is fetched at its own coordinate
int march_level0_u8(const uint8_t* img, size_t img_pitch, int w, int h, float shift, const OctaveView& o0,
                    const Taps& dd, const Taps& inc0, int R, int plan, cudaStream_t st);
// levels 0 and 1 of octave 0 in one launch (march_level01x2_kernel): the exact-2x 8-bit path with R0 == R1 == 5; returns 0
// (nothing launched) anywhere else
int march_level01_u8(const uint8_t* img, size_t img_pitch, int w, int h, float shift, const OctaveView& o0,
                     const Taps& dd, const Taps& inc0, int R0, const Taps& t1, int R1, int plan, cudaStream_t st);
int march_level0_f32(const float* img, size_t img_pitch, int w, int h, float shift, const OctaveView& o0,
                     const Taps& dd, const Taps& inc0, int R, int plan, cudaStream_t st);

} // namespace psb
