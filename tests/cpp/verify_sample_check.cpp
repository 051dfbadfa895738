// Host check of the RANSAC sample hash (popsift_b200/csrc/k_verify_sample.h), the same __host__ __device__ function the
// verify kernel calls.  `verify_sample_check IN OUT`: IN holds records {uint64 seed, int32 pair, int32 sample, uint32 n,
// int32 m} (24 bytes, m = 4 or 7); OUT receives per record {int32 valid, uint32 idx[7]} (32 bytes, unused entries 0).
#include "k_verify_sample.h"

#include <cstdio>
#include <cstring>
#include <vector>

struct Rec { uint64_t seed; int32_t p, s; uint32_t n; int32_t m; };
static_assert(sizeof(Rec) == 24, "record layout");

int main(int argc, char** argv)
{
    if (argc != 3) { std::fprintf(stderr, "usage: verify_sample_check IN OUT\n"); return 2; }
    FILE* fi = std::fopen(argv[1], "rb");
    if (!fi) return 2;
    std::vector<Rec> in;
    Rec r;
    while (std::fread(&r, sizeof r, 1, fi) == 1) in.push_back(r);
    std::fclose(fi);
    std::vector<uint32_t> out(in.size() * 8, 0);
    for (size_t i = 0; i < in.size(); ++i) {
        const Rec& q = in[i];
        uint32_t* o = &out[8 * i];
        bool ok = false;
        if (q.m == 4) {
            uint32_t idx[4];
            ok = psb::verify_sample<4>(q.seed, q.p, q.s, q.n, idx);
            std::memcpy(o + 1, idx, sizeof idx);
        } else if (q.m == 7) {
            uint32_t idx[7];
            ok = psb::verify_sample<7>(q.seed, q.p, q.s, q.n, idx);
            std::memcpy(o + 1, idx, sizeof idx);
        } else {
            return 2;
        }
        o[0] = ok ? 1u : 0u;
    }
    FILE* fo = std::fopen(argv[2], "wb");
    if (!fo || std::fwrite(out.data(), sizeof(uint32_t), out.size(), fo) != out.size()) return 2;
    std::fclose(fo);
    std::printf("OK %zu\n", in.size());
    return 0;
}
