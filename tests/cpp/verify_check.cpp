// popsift::verifyPairs through the C++ API against the C ABI on the same pairs: three frames extracted under
// Config::MatchingMode, all six ordered pairs of distinct frames plus one self pair, matched with matchPairs, then verified
// with a homography (and with a fundamental matrix).  The C path uploads the same match rows and runs
// ps_match_correspondences + ps_verify_batch itself; models, counts and inlier rows must be identical.
// Usage: verify_check W H a.raw b.raw c.raw      prints "OK <pairs> <inliers per pair...>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 6) { std::fprintf(stderr, "usage: verify_check W H a.raw b.raw c.raw\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    popsift::Config config;
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
    std::vector<std::pair<int, int>> pairs = {{0, 1}, {0, 2}, {1, 0}, {1, 2}, {2, 0}, {2, 1}, {1, 1}};
    const std::vector<std::vector<int>> matches = popsift::matchPairs(sets, pairs);
    std::vector<const ps_feature*> feat(3);
    std::vector<const int32_t*> rev(3);
    std::vector<int32_t> n(3), flat, start;
    for (int k = 0; k < 3; ++k) {
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        rev[k] = sets[k]->getReverseMap();
        n[k] = sets[k]->getDescriptorCount();
    }
    size_t rows = 0;
    for (const auto& pq : pairs) { flat.push_back(pq.first); flat.push_back(pq.second); start.push_back((int32_t)rows); rows += n[pq.first]; }
    int32_t* d_match = static_cast<int32_t*>(ps_dev_alloc(rows * 3 * sizeof(int32_t)));
    float* d_corr = static_cast<float*>(ps_dev_alloc(rows * 16));
    int32_t* d_src = static_cast<int32_t*>(ps_dev_alloc(rows * sizeof(int32_t)));
    uint8_t* d_mask = static_cast<uint8_t*>(ps_dev_alloc(rows));
    float* d_models = static_cast<float*>(ps_dev_alloc(pairs.size() * 36));
    int32_t* d_n = static_cast<int32_t*>(ps_dev_alloc(pairs.size() * 4));
    if (!d_match || !d_corr || !d_src || !d_mask || !d_models || !d_n) { std::printf("FAIL alloc\n"); return 1; }
    for (size_t p = 0; p < pairs.size(); ++p)
        ps_host_to_dev(d_match + 3 * (size_t)start[p], matches[p].data(), matches[p].size() * sizeof(int32_t));
    std::vector<int32_t> n_corr(pairs.size());
    if (ps_match_correspondences(0, 3, feat.data(), rev.data(), n.data(), (int)pairs.size(), flat.data(), d_match, d_corr, d_src,
                                 n_corr.data()) != PS_OK) { std::printf("FAIL ps_match_correspondences: %s\n", ps_last_error(nullptr)); return 1; }
    std::vector<int32_t> src(rows);
    ps_dev_to_host(src.data(), d_src, rows * sizeof(int32_t));
    std::vector<int> report;
    for (int model : {popsift::VerifyParams::Homography, popsift::VerifyParams::Fundamental}) {
        popsift::VerifyParams vp;
        vp.model = model;
        vp.n_samples = model == popsift::VerifyParams::Homography ? 512 : 1024;
        vp.seed = 7;
        const std::vector<popsift::PairGeometry> got = popsift::verifyPairs(sets, pairs, matches, vp);
        ps_verify_params prm{model, vp.n_samples, vp.threshold, 1, 7};
        if (ps_verify_batch(0, (int)pairs.size(), d_corr, start.data(), n_corr.data(), &prm, d_models, d_n, d_mask, nullptr) != PS_OK) {
            std::printf("FAIL ps_verify_batch: %s\n", ps_last_error(nullptr)); return 1;
        }
        std::vector<float> models(pairs.size() * 9);
        std::vector<int32_t> cnt(pairs.size());
        std::vector<uint8_t> mask(rows);
        ps_dev_to_host(models.data(), d_models, models.size() * 4);
        ps_dev_to_host(cnt.data(), d_n, cnt.size() * 4);
        ps_dev_to_host(mask.data(), d_mask, rows);
        if (got.size() != pairs.size()) { std::printf("FAIL %zu results\n", got.size()); return 1; }
        for (size_t p = 0; p < pairs.size(); ++p) {
            std::vector<int> want_rows;
            for (int k = 0; k < n_corr[p]; ++k)
                if (mask[start[p] + k]) want_rows.push_back(src[start[p] + k]);
            if (std::memcmp(got[p].model, &models[9 * p], 36) != 0 || got[p].n_inliers != cnt[p] || got[p].inlier_rows != want_rows) {
                std::printf("FAIL model %d pair (%d,%d): %d vs %d inliers\n", model, pairs[p].first, pairs[p].second, got[p].n_inliers, cnt[p]);
                return 1;
            }
            report.push_back(cnt[p]);
        }
    }
    std::printf("OK %zu", pairs.size());
    for (int v : report) std::printf(" %d", v);
    std::printf("\n");
    for (void* p : {(void*)d_match, (void*)d_corr, (void*)d_src, (void*)d_mask, (void*)d_models, (void*)d_n}) ps_dev_free(p);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
