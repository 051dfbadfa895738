// popsift::twoViewGeometries through the C++ API against the C ABI on the same pairs: two frames extracted under
// Config::MatchingMode, both ordered pairs plus one self pair, matched with matchPairs, then classified.  The C path uploads
// the same match rows and runs ps_match_correspondences, ps_verify_batch (H, F), ps_relative_pose_batch and
// ps_two_view_config_batch itself; the configuration, counts, normal, tri_angle, E, F, R, t and the inlier and in-front rows
// must be identical.
// Usage: twoview_check W H a.raw b.raw fx0 fy0 cx0 cy0 fx1 fy1 cx1 cy1    prints "OK <pairs> <config per pair...>" or FAIL
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>
#include <popsift_b200_twoview.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 13) { std::fprintf(stderr, "usage: twoview_check W H a.raw b.raw fx0 fy0 cx0 cy0 fx1 fy1 cx1 cy1\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]);
    std::vector<popsift::Camera> cams(2);
    for (int k = 0; k < 2; ++k)
        cams[k] = popsift::Camera{(float)std::atof(argv[5 + 4 * k]), (float)std::atof(argv[6 + 4 * k]), (float)std::atof(argv[7 + 4 * k]),
                                  (float)std::atof(argv[8 + 4 * k])};
    popsift::Config config;
    PopSift sift(config, popsift::Config::MatchingMode, PopSift::ByteImages, 0);
    std::vector<popsift::FeaturesDev*> sets;
    for (int k = 0; k < 2; ++k) {
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
    const std::vector<std::pair<int, int>> pairs = {{0, 1}, {1, 0}, {0, 0}};
    const std::vector<std::vector<int>> matches = popsift::matchPairs(sets, pairs);
    popsift::PoseParams pp;
    pp.n_samples = 512;
    pp.threshold = 2.0f;
    pp.seed = 11;
    popsift::TwoViewConfigParams tc;
    tc.min_inliers = 20;
    const std::vector<popsift::TwoViewGeometry> got = popsift::twoViewGeometries(sets, pairs, matches, cams, pp, tc);
    // bad arguments throw
    try {
        popsift::twoViewGeometries(sets, pairs, matches, std::vector<popsift::Camera>(1), pp, tc);
        std::printf("FAIL no throw on a missing camera\n"); return 1;
    } catch (const std::runtime_error&) {}
    try {
        std::vector<popsift::Camera> bad = cams;
        bad[1].fx = 0.0f;
        popsift::twoViewGeometries(sets, pairs, matches, bad, pp, tc);
        std::printf("FAIL no throw on fx = 0\n"); return 1;
    } catch (const std::runtime_error&) {}
    try {
        popsift::TwoViewConfigParams bad = tc;
        bad.max_h_ratio = 2.0;
        popsift::twoViewGeometries(sets, pairs, matches, cams, pp, bad);
        std::printf("FAIL no throw on max_h_ratio = 2\n"); return 1;
    } catch (const std::runtime_error&) {}

    std::vector<const ps_feature*> feat(2);
    std::vector<const int32_t*> rev(2);
    std::vector<int32_t> n(2), flat, start;
    for (int k = 0; k < 2; ++k) {
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        rev[k] = sets[k]->getReverseMap();
        n[k] = sets[k]->getDescriptorCount();
    }
    size_t rows = 0;
    std::vector<ps_camera> c_cams;
    for (const auto& pq : pairs) {
        flat.push_back(pq.first); flat.push_back(pq.second); start.push_back((int32_t)rows); rows += n[pq.first];
        for (int s : {pq.first, pq.second}) c_cams.push_back(ps_camera{cams[s].fx, cams[s].fy, cams[s].cx, cams[s].cy});
    }
    int32_t* d_match = static_cast<int32_t*>(ps_dev_alloc(rows * 3 * sizeof(int32_t)));
    float* d_corr = static_cast<float*>(ps_dev_alloc(rows * 16));
    int32_t* d_src = static_cast<int32_t*>(ps_dev_alloc(rows * sizeof(int32_t)));
    uint8_t* d_mask = static_cast<uint8_t*>(ps_dev_alloc(rows));
    ps_two_view* d_ess = static_cast<ps_two_view*>(ps_dev_alloc(pairs.size() * sizeof(ps_two_view)));
    ps_two_view* d_out = static_cast<ps_two_view*>(ps_dev_alloc(pairs.size() * sizeof(ps_two_view)));
    uint8_t* d_emask = static_cast<uint8_t*>(ps_dev_alloc(rows));
    uint8_t* d_hmask = static_cast<uint8_t*>(ps_dev_alloc(rows));
    uint8_t* d_fmask = static_cast<uint8_t*>(ps_dev_alloc(rows));
    float* d_h = static_cast<float*>(ps_dev_alloc(pairs.size() * 36));
    float* d_f = static_cast<float*>(ps_dev_alloc(pairs.size() * 36));
    int32_t* d_hn = static_cast<int32_t*>(ps_dev_alloc(pairs.size() * 4));
    int32_t* d_fn = static_cast<int32_t*>(ps_dev_alloc(pairs.size() * 4));
    if (!d_match || !d_corr || !d_src || !d_mask || !d_out || !d_ess || !d_emask || !d_hmask || !d_fmask || !d_h || !d_f || !d_hn || !d_fn) {
        std::printf("FAIL alloc\n");
        return 1;
    }
    for (size_t p = 0; p < pairs.size(); ++p)
        ps_host_to_dev(d_match + 3 * (size_t)start[p], matches[p].data(), matches[p].size() * sizeof(int32_t));
    std::vector<int32_t> n_corr(pairs.size());
    if (ps_match_correspondences(0, 2, feat.data(), rev.data(), n.data(), (int)pairs.size(), flat.data(), d_match, d_corr, d_src,
                                 n_corr.data()) != PS_OK) { std::printf("FAIL ps_match_correspondences: %s\n", ps_last_error(nullptr)); return 1; }
    const int P = (int)pairs.size();
    ps_verify_params hp{PS_GEOM_HOMOGRAPHY, pp.n_samples, pp.threshold, 1, pp.seed}, fp{PS_GEOM_FUNDAMENTAL, pp.n_samples, pp.threshold, 1, pp.seed};
    ps_pose_params prm{pp.n_samples, pp.threshold, 1, 0, pp.seed};
    ps_two_view_config_params cp{tc.min_inliers, pp.threshold, tc.min_ef_ratio, tc.max_h_ratio, tc.min_rotation_ratio};
    std::vector<ps_two_view_info> info(pairs.size());
    if (ps_verify_batch(0, P, d_corr, start.data(), n_corr.data(), &hp, d_h, d_hn, d_hmask, nullptr) != PS_OK ||
        ps_verify_batch(0, P, d_corr, start.data(), n_corr.data(), &fp, d_f, d_fn, d_fmask, nullptr) != PS_OK ||
        ps_relative_pose_batch(0, P, d_corr, start.data(), n_corr.data(), c_cams.data(), &prm, d_ess, d_emask, nullptr, nullptr) != PS_OK ||
        ps_two_view_config_batch(0, P, d_corr, start.data(), n_corr.data(), c_cams.data(), d_ess, d_emask, d_fn, d_h, d_hmask, &cp, d_out,
                                 d_mask, nullptr, info.data()) != PS_OK) {
        std::printf("FAIL C ABI: %s\n", ps_last_error(nullptr));
        return 1;
    }
    std::vector<int32_t> src(rows);
    std::vector<uint8_t> mask(rows);
    std::vector<ps_two_view> two(pairs.size());
    ps_dev_to_host(src.data(), d_src, rows * sizeof(int32_t));
    ps_dev_to_host(mask.data(), d_mask, rows);
    ps_dev_to_host(two.data(), d_out, two.size() * sizeof(ps_two_view));
    if (got.size() != pairs.size()) { std::printf("FAIL %zu results\n", got.size()); return 1; }
    for (size_t p = 0; p < pairs.size(); ++p) {
        std::vector<int> want_in, want_front;
        for (int k = 0; k < n_corr[p]; ++k) {
            if (mask[start[p] + k] & 1) want_in.push_back(src[start[p] + k]);
            if (mask[start[p] + k] & 2) want_front.push_back(src[start[p] + k]);
        }
        const ps_two_view& v = two[p];
        const ps_two_view_info& in = info[p];
        const popsift::TwoViewPose& g = got[p].pose;
        const popsift::TwoViewGeometry& G = got[p];
        if (std::memcmp(g.E, v.E, 36) || std::memcmp(g.F, v.F, 36) || std::memcmp(g.R, v.R, 36) || std::memcmp(g.t, v.t, 12) ||
            g.n_inliers != v.n_inliers || g.n_front != v.n_front || g.inlier_rows != want_in || g.front_rows != want_front ||
            G.config != in.config || G.n_e != in.n_e || G.n_f != in.n_f || G.n_h != in.n_h || G.n_rotation != in.n_rotation ||
            std::memcmp(G.normal, in.normal, 12) || std::memcmp(&G.tri_angle, &in.tri_angle, 4)) {
            std::printf("FAIL pair (%d,%d): config %d vs %d, %d vs %d inliers\n", pairs[p].first, pairs[p].second, G.config, in.config,
                        g.n_inliers, v.n_inliers);
            return 1;
        }
    }
    std::printf("OK %zu", pairs.size());
    for (const auto& g : got) std::printf(" %d", g.config);
    std::printf("\n");
    for (void* p : {(void*)d_match, (void*)d_corr, (void*)d_src, (void*)d_mask, (void*)d_out, (void*)d_ess, (void*)d_emask, (void*)d_hmask,
                    (void*)d_fmask, (void*)d_h, (void*)d_f, (void*)d_hn, (void*)d_fn})
        ps_dev_free(p);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
