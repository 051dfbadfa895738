// The order rules of ps_retrieve_pairs (include/popsift_b200_retrieval.h): one definition for the kernels (k_retrieval.cu)
// and the host check (tests/cpp/retrieval_host.cpp).
#pragma once
#include <stdint.h>
#include <math.h>
#if !defined(__CUDA_ARCH__)
#include <string.h>
#endif

#if defined(__CUDACC__)
#define PSR_HD __host__ __device__ __forceinline__
#else
#define PSR_HD inline
#endif

namespace psb {

// one step of a score's chain: acc + a * b, rounded once
PSR_HD float retrieve_fma(float a, float b, float acc) { return fmaf(a, b, acc); }

// score(i, j) of rows a and b, d = 0 .. dim-1 in order from 0 (the kernel's tiles run the same chain, 4 d at a time)
PSR_HD float retrieve_score(const float* a, const float* b, int dim)
{
    float acc = 0.0f;
    for (int d = 0; d < dim; ++d) acc = retrieve_fma(a[d], b[d], acc);
    return acc;
}

PSR_HD uint32_t retrieve_bits(float s)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(s);
#else
    uint32_t u;
    memcpy(&u, &s, 4);
    return u;
#endif
}

// The rank of candidate j with score s: smaller is better.  High word: the score's order, descending (-0 counts as +0,
// NaN is 0xffffffff, below every number); low word: j, so that equal scores go to the lower j.  ~0 (j = -1 below every
// NaN) marks an empty slot.
PSR_HD uint64_t retrieve_key(float s, int j)
{
    uint32_t hi = 0xffffffffu;
    if (s == s) {
        const uint32_t u = retrieve_bits(s == 0.0f ? 0.0f : s);
        const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
        hi = ~asc;
    }
    return ((uint64_t)hi << 32) | (uint32_t)j;
}

} // namespace psb
