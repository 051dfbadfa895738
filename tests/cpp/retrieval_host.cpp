// Host-only: the rules of ps_vlad_train's initial draw and of ps_retrieve_pairs' scores, computed by the same headers the
// kernels use (popsift_b200/csrc/k_verify_sample.h, k_retrieval.h).  No CUDA, no library.
//
//   retrieval_host draw <seed> <N> <k>         k distinct pool indices in draw order, one per line
//   retrieval_host score <in> <out> <fmaf> [rows]
//                                              in: int32 n, int32 dim, float32 v[n][dim]; out: float32 s[rows][n] (rows
//                                              default n); fmaf = 0: retrieve_score (k_retrieval.h); 1: a std::fmaf loop
#include "k_retrieval.h"
#include "k_verify_sample.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

int main(int argc, char** argv)
{
    if (argc == 5 && !strcmp(argv[1], "draw")) {
        const uint64_t seed = strtoull(argv[2], nullptr, 10);
        const uint32_t N = (uint32_t)strtoul(argv[3], nullptr, 10);
        const int k = atoi(argv[4]);
        const uint64_t key = psb::verify_mix(seed);
        std::vector<char> seen(N, 0);
        int got = 0;
        for (int c = 0; got < k; ++c) {
            const uint32_t v = psb::verify_draw(key, c, N);
            if (seen[v]) continue;
            seen[v] = 1;
            printf("%u\n", v);
            ++got;
        }
        return 0;
    }
    if ((argc == 5 || argc == 6) && !strcmp(argv[1], "score")) {
        FILE* f = fopen(argv[2], "rb");
        int32_t hd[2];
        if (!f || fread(hd, 4, 2, f) != 2) return 2;
        const int n = hd[0], dim = hd[1];
        const int rows = argc == 6 ? atoi(argv[5]) : n;
        std::vector<float> v((size_t)n * dim), s((size_t)rows * n);
        if (fread(v.data(), 4, v.size(), f) != v.size()) return 2;
        fclose(f);
        const bool plain = atoi(argv[4]) != 0;
        for (int i = 0; i < rows; ++i)
            for (int j = 0; j < n; ++j) {
                const float* a = &v[(size_t)i * dim];
                const float* b = &v[(size_t)j * dim];
                if (plain) {
                    float acc = 0.0f;
                    for (int d = 0; d < dim; ++d) acc = std::fmaf(a[d], b[d], acc);
                    s[(size_t)i * n + j] = acc;
                } else {
                    s[(size_t)i * n + j] = psb::retrieve_score(a, b, dim);
                }
            }
        FILE* o = fopen(argv[3], "wb");
        if (!o || fwrite(s.data(), 4, s.size(), o) != s.size()) return 3;
        fclose(o);
        return 0;
    }
    fprintf(stderr, "usage: retrieval_host draw <seed> <N> <k> | score <in> <out> <fmaf> [rows]\n");
    return 1;
}
