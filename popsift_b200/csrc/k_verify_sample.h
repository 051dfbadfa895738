// The sample hash of ps_verify_batch (include/popsift_b200.h): which correspondences sample s of pair p draws.  One
// definition for the kernel (k_verify.cu) and the host check (tests/cpp/verify_sample_check.cpp).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PSV_HD __host__ __device__ __forceinline__
#else
#define PSV_HD inline
#endif

namespace psb {

constexpr int kVerifyDraws = 64;   // draws before a sample without enough distinct indices is invalid

// splitmix64's finaliser
PSV_HD uint64_t verify_mix(uint64_t z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

PSV_HD uint64_t verify_key(uint64_t seed, int p, int s)
{
    return verify_mix(seed ^ verify_mix(((uint64_t)(uint32_t)p << 32) | (uint32_t)s));
}

// draw c of a sample: an index in [0, n)
PSV_HD uint32_t verify_draw(uint64_t key, int c, uint32_t n)
{
    return (uint32_t)(((verify_mix(key + (uint64_t)c) >> 32) * (uint64_t)n) >> 32);
}

// M distinct indices in draw order; false when 64 draws do not give them.  Fully unrolled over M, so idx stays in
// registers in the kernel.
template <int M>
PSV_HD bool verify_sample(uint64_t seed, int p, int s, uint32_t n, uint32_t (&idx)[M])
{
    const uint64_t key = verify_key(seed, p, s);
    int got = 0;
#pragma unroll
    for (int j = 0; j < M; ++j) idx[j] = 0;
    for (int c = 0; c < kVerifyDraws && got < M; ++c) {
        const uint32_t v = verify_draw(key, c, n);
        bool dup = false;
#pragma unroll
        for (int j = 0; j < M; ++j) dup |= (j < got && idx[j] == v);
        if (dup) continue;
#pragma unroll
        for (int j = 0; j < M; ++j)
            if (j == got) idx[j] = v;
        ++got;
    }
    return got == M;
}

} // namespace psb
