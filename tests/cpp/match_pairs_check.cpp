// popsift::matchPairs through the C++ API: three frames extracted under Config::MatchingMode, all nine ordered pairs
// (self pairs included) matched in one call, and every entry compared with FeaturesDev::matchIndices of the same pair
// under each flag (AUTO, EXACT, TENSOR).
// Usage: match_pairs_check W H a.raw b.raw c.raw      prints "OK <pairs> <rows>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 6) { std::fprintf(stderr, "usage: match_pairs_check W H a.raw b.raw c.raw\n"); return 2; }
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
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) pairs.emplace_back(i, j);
    long rows = 0;
    for (int flags : {0, 1, 2}) {
        const std::vector<std::vector<int>> got = popsift::matchPairs(sets, pairs, flags);
        if (got.size() != pairs.size()) { std::printf("FAIL %zu results for %zu pairs\n", got.size(), pairs.size()); return 1; }
        for (size_t p = 0; p < pairs.size(); ++p) {
            const std::vector<int> want = sets[pairs[p].first]->matchIndices(sets[pairs[p].second], flags);
            if (got[p] != want) { std::printf("FAIL flags=%d pair (%d,%d)\n", flags, pairs[p].first, pairs[p].second); return 1; }
            rows += (long)want.size() / 3;
        }
    }
    std::printf("OK %zu %ld\n", pairs.size(), rows);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
