// popsift::matchPairsGuided / matchPairsGuidedU8 through the C++ API against the C ABI on the same pairs: three frames
// extracted under Config::MatchingMode, all six ordered pairs of distinct frames plus one self pair, matched with matchPairs
// and verified with verifyPairs (homography and fundamental matrix).  The C path uploads the same models and runs
// ps_match_guided_batch / ps_match_u8_guided_batch itself (the u8 sets through ps_descriptors_to_u8); rows must be identical.
// Usage: guided_check W H a.raw b.raw c.raw      prints "OK <pairs> <accepted guided rows per model and path...>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>
#include <popsift_b200_guided.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 6) { std::fprintf(stderr, "usage: guided_check W H a.raw b.raw c.raw\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    popsift::Config config;
    config.setNormalizationMultiplier(9);               // descriptors scaled for 8 bits (no effect on the float distances' order)
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
    const std::vector<std::pair<int, int>> pairs = {{0, 1}, {0, 2}, {1, 0}, {1, 2}, {2, 0}, {2, 1}, {1, 1}};
    const std::vector<std::vector<int>> matches = popsift::matchPairs(sets, pairs);
    std::vector<const ps_descriptor*> desc(3);
    std::vector<const uint8_t*> desc8(3);
    std::vector<const ps_feature*> feat(3);
    std::vector<const int32_t*> rev(3);
    std::vector<int32_t> n(3), flat;
    for (int k = 0; k < 3; ++k) {
        desc[k] = reinterpret_cast<const ps_descriptor*>(sets[k]->getDescriptors());
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        rev[k] = sets[k]->getReverseMap();
        n[k] = sets[k]->getDescriptorCount();
        uint8_t* q = static_cast<uint8_t*>(ps_dev_alloc((size_t)n[k] * 128));
        if (!q || ps_descriptors_to_u8(0, desc[k], n[k], q) != PS_OK) { std::printf("FAIL u8 copy\n"); return 1; }
        desc8[k] = q;
    }
    size_t rows = 0;
    for (const auto& pq : pairs) { flat.push_back(pq.first); flat.push_back(pq.second); rows += n[pq.first]; }
    int32_t* d_out = static_cast<int32_t*>(ps_dev_alloc(rows * 3 * sizeof(int32_t)));
    float* d_models = static_cast<float*>(ps_dev_alloc(pairs.size() * 36));
    if (!d_out || !d_models) { std::printf("FAIL alloc\n"); return 1; }
    std::vector<int> report;
    for (int model : {popsift::VerifyParams::Homography, popsift::VerifyParams::Fundamental}) {
        popsift::VerifyParams vp;
        vp.model = model;
        vp.n_samples = 512;
        vp.seed = 3;
        const std::vector<popsift::PairGeometry> geo = popsift::verifyPairs(sets, pairs, matches, vp);
        std::vector<float> models(pairs.size() * 9);
        for (size_t p = 0; p < pairs.size(); ++p)
            for (int k = 0; k < 9; ++k) models[9 * p + k] = geo[p].model[k];
        ps_host_to_dev(d_models, models.data(), models.size() * 4);
        for (int u8 = 0; u8 < 2; ++u8) {
            const std::vector<std::vector<int>> got = u8 ? popsift::matchPairsGuidedU8(sets, pairs, geo, vp) : popsift::matchPairsGuided(sets, pairs, geo, vp);
            const int rc = u8 ? ps_match_u8_guided_batch(0, 3, desc8.data(), feat.data(), rev.data(), n.data(), (int)pairs.size(), flat.data(),
                                                         d_models, model, vp.threshold, d_out, 0)
                              : ps_match_guided_batch(0, 3, desc.data(), feat.data(), rev.data(), n.data(), (int)pairs.size(), flat.data(),
                                                      d_models, model, vp.threshold, d_out, 0);
            if (rc != PS_OK) { std::printf("FAIL C ABI: %s\n", ps_last_error(nullptr)); return 1; }
            std::vector<int32_t> want(rows * 3);
            ps_dev_to_host(want.data(), d_out, want.size() * 4);
            if (got.size() != pairs.size()) { std::printf("FAIL %zu results\n", got.size()); return 1; }
            size_t row = 0;
            int accepted = 0;
            for (size_t p = 0; p < pairs.size(); ++p) {
                const std::vector<int> w(want.begin() + 3 * row, want.begin() + 3 * (row + n[pairs[p].first]));
                if (got[p] != w) { std::printf("FAIL model %d u8 %d pair (%d,%d)\n", model, u8, pairs[p].first, pairs[p].second); return 1; }
                for (size_t i = 2; i < w.size(); i += 3) accepted += w[i];
                row += n[pairs[p].first];
            }
            report.push_back(accepted);
        }
    }
    std::printf("OK %zu", pairs.size());
    for (int v : report) std::printf(" %d", v);
    std::printf("\n");
    for (int k = 0; k < 3; ++k) ps_dev_free(const_cast<uint8_t*>(desc8[k]));
    ps_dev_free(d_out);
    ps_dev_free(d_models);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
