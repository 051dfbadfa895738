// popsift::vladCodebook / vladEncode / retrievePairs through the C++ API against the C ABI (popsift_b200_retrieval.h) on
// the same sets: frames extracted under Config::MatchingMode, a codebook of k = 8 centroids, their VLAD vectors and the
// pairs of m = 2 neighbours.  Codebook and vectors must be byte-identical, the pairs the union of the C ABI's neighbours.
// Usage: retrieval_check W H a.raw b.raw ...      prints "OK <frames> <pairs>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200_retrieval.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <set>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 5) { std::fprintf(stderr, "usage: retrieval_check W H a.raw b.raw ...\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    popsift::Config config;
    PopSift sift(config, popsift::Config::MatchingMode, PopSift::ByteImages, 0);
    std::vector<popsift::FeaturesDev*> sets;
    for (int a = 3; a < argc; ++a) {
        std::vector<unsigned char> img((size_t)w * h);
        std::ifstream in(argv[a], std::ios::binary);
        in.read(reinterpret_cast<char*>(img.data()), img.size());
        if (!in) { std::fprintf(stderr, "short read\n"); return 2; }
        SiftJob* job = sift.enqueue(w, h, img.data());
        popsift::FeaturesDev* fd = job->getDev();
        delete job;
        if (!fd || fd->getDescriptorCount() <= 0) { std::printf("FAIL no descriptors in frame %d\n", a - 3); return 1; }
        sets.push_back(fd);
    }
    const int n = (int)sets.size(), k = 8, m = 2;
    popsift::VladParams prm;
    prm.k = k;
    prm.iters = 3;
    prm.seed = 7;
    const std::vector<float> cb = popsift::vladCodebook(sets, prm);
    const std::vector<float> vl = popsift::vladEncode(sets, cb);
    const std::vector<std::pair<int, int>> pairs = popsift::retrievePairs(vl, n, m);

    std::vector<const ps_descriptor*> d_sets;
    std::vector<int32_t> n_desc;
    for (auto* s : sets) { d_sets.push_back(reinterpret_cast<const ps_descriptor*>(s->getDescriptors())); n_desc.push_back(s->getDescriptorCount()); }
    float* d_cb = static_cast<float*>(ps_dev_alloc((size_t)k * 512));
    float* d_vl = static_cast<float*>(ps_dev_alloc((size_t)n * k * 512));
    int32_t* d_nb = static_cast<int32_t*>(ps_dev_alloc((size_t)n * m * 4));
    float* d_sc = static_cast<float*>(ps_dev_alloc((size_t)n * m * 4));
    if (ps_vlad_train(0, n, d_sets.data(), n_desc.data(), k, 3, 7, d_cb, 0) != PS_OK ||
        ps_vlad_encode(0, n, d_sets.data(), n_desc.data(), k, d_cb, d_vl, nullptr, 0) != PS_OK ||
        ps_retrieve_pairs(0, n, d_vl, k * 128, m, d_nb, d_sc) != PS_OK) {
        std::printf("FAIL C ABI: %s\n", ps_last_error(nullptr));
        return 1;
    }
    std::vector<float> cb2((size_t)k * 128), vl2((size_t)n * k * 128);
    std::vector<int32_t> nb((size_t)n * m);
    ps_dev_to_host(cb2.data(), d_cb, cb2.size() * 4);
    ps_dev_to_host(vl2.data(), d_vl, vl2.size() * 4);
    ps_dev_to_host(nb.data(), d_nb, nb.size() * 4);
    for (void* p : {(void*)d_cb, (void*)d_vl, (void*)d_nb, (void*)d_sc}) ps_dev_free(p);
    if (cb.size() != cb2.size() || std::memcmp(cb.data(), cb2.data(), cb.size() * 4)) { std::printf("FAIL codebook differs\n"); return 1; }
    if (vl.size() != vl2.size() || std::memcmp(vl.data(), vl2.data(), vl.size() * 4)) { std::printf("FAIL vectors differ\n"); return 1; }
    std::set<std::pair<int, int>> want;
    for (int i = 0; i < n; ++i)
        for (int q = 0; q < m; ++q) {
            const int j = nb[(size_t)i * m + q];
            if (j >= 0) want.insert({std::min(i, j), std::max(i, j)});
        }
    if (std::vector<std::pair<int, int>>(want.begin(), want.end()) != pairs) { std::printf("FAIL pairs differ\n"); return 1; }
    for (auto* s : sets) delete s;
    std::printf("OK %d %zu\n", n, pairs.size());
    return 0;
}
