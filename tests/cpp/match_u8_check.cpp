// popsift::matchPairsU8 through the C++ API: three frames extracted under Config::MatchingMode with norm_multi = 9, all
// nine ordered pairs (self pairs included) matched in one call under each flag (AUTO, EXACT, TENSOR).  Every entry must
// equal ps_match_batch(..., PS_MATCH_EXACT) on the same descriptors quantised with ps_descriptors_to_u8 and widened back
// to float32.
// Usage: match_u8_check W H a.raw b.raw c.raw      prints "OK <pairs> <rows> <accepted>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 6) { std::fprintf(stderr, "usage: match_u8_check W H a.raw b.raw c.raw\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    popsift::Config config;
    config.setNormalizationMultiplier(9);
    PopSift sift(config, popsift::Config::MatchingMode, PopSift::ByteImages, 0);
    std::vector<popsift::FeaturesDev*> sets;
    for (int k = 0; k < 3; ++k) {
        std::vector<unsigned char> img((size_t)w * h);
        std::ifstream in(argv[3 + k], std::ios::binary);
        in.read(reinterpret_cast<char*>(img.data()), img.size());
        if (!in) { std::fprintf(stderr, "short read\n"); return 2; }
        SiftJob* job = sift.enqueue(w, h, img.data());
        popsift::FeaturesDev* fd = job->getDev();
        delete job;
        if (!fd || fd->getDescriptorCount() <= 0) { std::printf("FAIL no descriptors in frame %d\n", k); return 1; }
        sets.push_back(fd);
    }
    // the expected rows: the quantised descriptors widened to float32, through the float matcher's CUDA-core kernel
    std::vector<const ps_descriptor*> wide(3);
    std::vector<int32_t> n(3);
    for (int k = 0; k < 3; ++k) {
        n[k] = sets[k]->getDescriptorCount();
        uint8_t* q = static_cast<uint8_t*>(ps_dev_alloc((size_t)n[k] * 128));
        if (!q || ps_descriptors_to_u8(0, reinterpret_cast<const ps_descriptor*>(sets[k]->getDescriptors()), n[k], q) != PS_OK) {
            std::printf("FAIL ps_descriptors_to_u8: %s\n", ps_last_error(nullptr)); return 1;
        }
        std::vector<uint8_t> hq((size_t)n[k] * 128);
        ps_dev_to_host(hq.data(), q, hq.size());
        ps_dev_free(q);
        std::vector<float> hf(hq.begin(), hq.end());
        void* d = ps_dev_alloc(hf.size() * sizeof(float));
        if (!d || ps_host_to_dev(d, hf.data(), hf.size() * sizeof(float)) != PS_OK) { std::printf("FAIL upload\n"); return 1; }
        wide[k] = static_cast<const ps_descriptor*>(d);
    }
    std::vector<std::pair<int, int>> pairs;
    std::vector<int32_t> flat;
    long rows = 0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { pairs.emplace_back(i, j); flat.push_back(i); flat.push_back(j); rows += n[i]; }
    std::vector<int32_t> want((size_t)rows * 3);
    int32_t* d_out = static_cast<int32_t*>(ps_dev_alloc(want.size() * sizeof(int32_t)));
    if (!d_out || ps_match_batch(0, 3, wide.data(), n.data(), (int)pairs.size(), flat.data(), d_out, PS_MATCH_EXACT) != PS_OK ||
        ps_dev_to_host(want.data(), d_out, want.size() * sizeof(int32_t)) != PS_OK) {
        std::printf("FAIL float exact matcher: %s\n", ps_last_error(nullptr)); return 1;
    }
    ps_dev_free(d_out);
    long accepted = 0;
    for (int flags : {PS_MATCH_AUTO, PS_MATCH_EXACT, PS_MATCH_TENSOR}) {
        const std::vector<std::vector<int>> got = popsift::matchPairsU8(sets, pairs, flags);
        if (got.size() != pairs.size()) { std::printf("FAIL %zu results for %zu pairs\n", got.size(), pairs.size()); return 1; }
        size_t row = 0;
        for (size_t p = 0; p < pairs.size(); ++p) {
            const size_t len = (size_t)n[pairs[p].first] * 3;
            if (got[p].size() != len || !std::equal(got[p].begin(), got[p].end(), want.begin() + row)) {
                std::printf("FAIL flags=%d pair (%d,%d)\n", flags, pairs[p].first, pairs[p].second); return 1;
            }
            row += len;
        }
    }
    for (size_t k = 2; k < want.size(); k += 3) accepted += want[k];
    std::printf("OK %zu %ld %ld\n", pairs.size(), rows, accepted);
    for (const ps_descriptor* d : wide) ps_dev_free(const_cast<ps_descriptor*>(d));
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
