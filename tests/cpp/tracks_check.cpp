// popsift::buildTracks (both overloads) through the C++ API against the C ABI (popsift_b200_tracks.h) on the same sets:
// frames extracted under Config::MatchingMode, all ordered pairs matched and verified with a homography, then
//   buildTracks(sets, pairs, matches, geometry)  against ps_match_correspondences + ps_verify_batch + ps_tracks_from_matches
//                                                with the inlier mask;
//   buildTracks(sets, pairs, guided rows)        against ps_match_correspondences + ps_tracks_from_matches without a mask.
// Tracks must be identical.
// Usage: tracks_check W H a.raw b.raw ...      prints "OK <tracks> <guided tracks>" or a FAIL line
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200_tracks.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <utility>
#include <vector>

namespace {

struct Abi {
    std::vector<const ps_feature*> feat;
    std::vector<const int32_t*> rev;
    std::vector<int32_t> n_desc, n_feat, flat;
    size_t rows = 0;
};

// the C ABI chain from host match rows: correspondences, optionally RANSAC (mask), then tracks as popsift::Tracks
bool abi_tracks(const Abi& a, const std::vector<std::vector<int>>& matches, bool verify, int min_length, popsift::Tracks& t)
{
    const int np = (int)matches.size(), ns = (int)a.n_desc.size();
    std::vector<int32_t> h_match;
    for (const auto& m : matches) h_match.insert(h_match.end(), m.begin(), m.end());
    const size_t nr = a.rows ? a.rows : 1;
    void* match = ps_dev_alloc(nr * 12);
    void* corr = ps_dev_alloc(nr * 16);
    void* src = ps_dev_alloc(nr * 4);
    void* mask = ps_dev_alloc(nr);
    void* models = ps_dev_alloc((size_t)np * 36);
    void* cnt = ps_dev_alloc((size_t)np * 4);
    size_t N = 0;
    std::vector<size_t> off(1, 0);
    for (int32_t n : a.n_feat) off.push_back(N += (size_t)n);
    void* of = ps_dev_alloc(N * 4);
    void* start = ps_dev_alloc((N / min_length + 1) * 4);
    void* mem = ps_dev_alloc(N * 4);
    std::vector<int32_t> n_corr(np), corr_start(np);
    for (int p = 0, r = 0; p < np; ++p) { corr_start[p] = r; r += a.n_desc[a.flat[2 * p]]; }
    ps_verify_params prm{PS_GEOM_HOMOGRAPHY, 1024, 4.0f, 1, 0};
    ps_track_counts c{};
    bool ok = ps_host_to_dev(match, h_match.data(), h_match.size() * 4) == PS_OK &&
              ps_match_correspondences(0, ns, a.feat.data(), a.rev.data(), a.n_desc.data(), np, a.flat.data(), (const int32_t*)match,
                                       (float*)corr, (int32_t*)src, n_corr.data()) == PS_OK &&
              (!verify || ps_verify_batch(0, np, (const float*)corr, corr_start.data(), n_corr.data(), &prm, (float*)models, (int32_t*)cnt,
                                          (uint8_t*)mask, nullptr) == PS_OK) &&
              ps_tracks_from_matches(0, ns, a.n_feat.data(), a.rev.data(), a.n_desc.data(), np, a.flat.data(), (const int32_t*)match,
                                     (const int32_t*)src, n_corr.data(), verify ? (const uint8_t*)mask : nullptr, min_length,
                                     (int32_t*)of, (int32_t*)start, (int32_t*)mem, &c) == PS_OK;
    if (ok) {
        std::vector<int32_t> m(c.n_members), o(N);
        t.start.resize(c.n_tracks + 1);
        ps_dev_to_host(t.start.data(), start, t.start.size() * 4);
        ps_dev_to_host(m.data(), mem, m.size() * 4);
        ps_dev_to_host(o.data(), of, o.size() * 4);
        for (int32_t g : m) {
            size_t s = 0;
            while (off[s + 1] <= (size_t)g) ++s;
            t.set.push_back((int)s);
            t.feature.push_back((int)(g - off[s]));
        }
        for (int i = 0; i < ns; ++i) t.track_of.emplace_back(o.begin() + off[i], o.begin() + off[i + 1]);
        t.n_components = c.n_components;
        t.n_conflicting = c.n_conflicting;
        t.n_short = c.n_short;
    }
    for (void* p : {match, corr, src, mask, models, cnt, of, start, mem}) ps_dev_free(p);
    return ok;
}

bool same(const popsift::Tracks& a, const popsift::Tracks& b)
{
    return a.start == b.start && a.set == b.set && a.feature == b.feature && a.track_of == b.track_of && a.n_components == b.n_components &&
           a.n_conflicting == b.n_conflicting && a.n_short == b.n_short;
}

} // namespace

int main(int argc, char** argv)
{
    if (argc < 5) { std::fprintf(stderr, "usage: tracks_check W H a.raw b.raw ...\n"); return 2; }
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
    const int n = (int)sets.size();
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j)
            if (i != j) pairs.push_back({i, j});
    Abi a;
    for (auto* s : sets) {
        a.feat.push_back(reinterpret_cast<const ps_feature*>(s->getFeatures()));
        a.rev.push_back(s->getReverseMap());
        a.n_desc.push_back(s->getDescriptorCount());
        a.n_feat.push_back(s->getFeatureCount());
    }
    for (const auto& p : pairs) { a.flat.push_back(p.first); a.flat.push_back(p.second); a.rows += (size_t)a.n_desc[p.first]; }

    popsift::VerifyParams prm;
    const auto matches = popsift::matchPairs(sets, pairs);
    const auto geom = popsift::verifyPairs(sets, pairs, matches, prm);
    const popsift::Tracks t1 = popsift::buildTracks(sets, pairs, matches, geom, 3);
    popsift::Tracks r1;
    if (!abi_tracks(a, matches, true, 3, r1)) { std::printf("FAIL C ABI: %s\n", ps_last_error(nullptr)); return 1; }
    if (!same(t1, r1)) { std::printf("FAIL verified tracks differ (%zu vs %zu)\n", t1.start.size(), r1.start.size()); return 1; }

    const auto guided = popsift::matchPairsGuided(sets, pairs, geom, prm);
    const popsift::Tracks t2 = popsift::buildTracks(sets, pairs, guided);
    popsift::Tracks r2;
    if (!abi_tracks(a, guided, false, 2, r2)) { std::printf("FAIL C ABI (guided): %s\n", ps_last_error(nullptr)); return 1; }
    if (!same(t2, r2)) { std::printf("FAIL guided tracks differ (%zu vs %zu)\n", t2.start.size(), r2.start.size()); return 1; }
    if (t1.start.size() < 2 || t2.start.size() < 2) { std::printf("FAIL no tracks\n"); return 1; }
    for (auto* s : sets) delete s;
    std::printf("OK %zu %zu\n", t1.start.size() - 1, t2.start.size() - 1);
    return 0;
}
