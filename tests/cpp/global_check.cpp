// popsift::rotationAveraging and popsift::globalPositioning through the C++ API against the C ABI on the same inputs: n
// frames extracted under Config::MatchingMode, every pair (i, j), i < j, matched with matchPairs, relative poses from
// relativePoses, rotation averaging (Cauchy, s = 2 degrees), tracks from buildTracks on verifyPairs' fundamental inliers,
// then global positioning under the averaged rotations.  The C path uploads the same arrays and runs
// ps_rotation_averaging and ps_global_positioning itself; rotations, flags, errors, poses, points and reports must be
// identical.
// Usage: global_check W H n f_0.raw .. f_{n-1}.raw then per view fx fy cx cy
//   prints "OK <registered> <used observations> <positioning cost>" or FAIL
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>
#include <popsift_b200_global.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <stdexcept>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 4) { std::fprintf(stderr, "usage: global_check W H n frames.. (fx fy cx cy) per view\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]), n = std::atoi(argv[3]);
    if (n < 2 || argc != 4 + n + 4 * n) { std::fprintf(stderr, "bad argument count\n"); return 2; }
    std::vector<popsift::Camera> cams(n);
    for (int k = 0; k < n; ++k) {
        const char* const* a = argv + 4 + n + 4 * k;
        cams[k] = popsift::Camera{(float)std::atof(a[0]), (float)std::atof(a[1]), (float)std::atof(a[2]), (float)std::atof(a[3])};
    }
    popsift::Config config;
    PopSift sift(config, popsift::Config::MatchingMode, PopSift::ByteImages, 0);
    std::vector<popsift::FeaturesDev*> sets;
    for (int k = 0; k < n; ++k) {
        std::vector<unsigned char> img((size_t)w * h);
        std::ifstream in(argv[4 + k], std::ios::binary);
        in.read(reinterpret_cast<char*>(img.data()), img.size());
        if (!in) { std::fprintf(stderr, "short read\n"); return 2; }
        SiftJob* job = sift.enqueue(w, h, img.data());
        popsift::FeaturesDev* fd = job->getDev();
        delete job;
        if (!fd || fd->getDescriptorCount() <= 0) { std::printf("FAIL no descriptors in frame %d\n", k); return 1; }
        sets.push_back(fd);
    }
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j) pairs.push_back({i, j});
    const std::vector<std::vector<int>> matches = popsift::matchPairs(sets, pairs);
    popsift::PoseParams pp;
    pp.threshold = 1.0f;
    pp.seed = 1;
    const std::vector<popsift::TwoViewPose> rel = popsift::relativePoses(sets, pairs, matches, cams, pp);
    popsift::RotationParams rp;
    rp.loss_scale = 2.0;
    const popsift::Rotations rot = popsift::rotationAveraging(n, pairs, rel, rp);
    try {
        popsift::RotationParams bad = rp;
        bad.cg_tol = 1.0;
        popsift::rotationAveraging(n, pairs, rel, bad);
        std::printf("FAIL no throw on a bad cg_tol\n"); return 1;
    } catch (const std::runtime_error&) {}
    popsift::VerifyParams vp;
    vp.model = popsift::VerifyParams::Fundamental;
    vp.threshold = 2.0f;
    const popsift::Tracks tracks = popsift::buildTracks(sets, pairs, matches, popsift::verifyPairs(sets, pairs, matches, vp), 2);
    popsift::PositionParams gp;
    gp.max_iters = 50;
    const popsift::Positions pos = popsift::globalPositioning(sets, tracks, cams, rot.R, rot.registered, gp);

    // the C ABI on the same inputs
    const size_t np = pairs.size(), nt = tracks.start.size() - 1, nm = tracks.set.size();
    std::vector<ps_two_view> rec(np);
    std::vector<int32_t> flat(2 * np);
    for (size_t p = 0; p < np; ++p) {
        rec[p] = ps_two_view{};
        std::memcpy(rec[p].R, rel[p].R, sizeof(rec[p].R));
        std::memcpy(rec[p].t, rel[p].t, sizeof(rec[p].t));
        rec[p].n_inliers = rel[p].n_inliers;
        rec[p].n_front = rel[p].n_front;
        flat[2 * p] = pairs[p].first;
        flat[2 * p + 1] = pairs[p].second;
    }
    ps_two_view* d_rec = static_cast<ps_two_view*>(ps_dev_alloc(np * sizeof(ps_two_view)));
    if (!d_rec) { std::printf("FAIL alloc\n"); return 1; }
    ps_host_to_dev(d_rec, rec.data(), np * sizeof(ps_two_view));
    ps_rotation_params rprm{};
    rprm.loss = PS_LOSS_CAUCHY;
    rprm.max_iters = rp.max_iters;
    rprm.cg_max_iters = rp.cg_max_iters;
    rprm.min_inliers = rp.min_inliers;
    rprm.loss_scale = rp.loss_scale;
    rprm.step_tol = rp.step_tol;
    rprm.cg_tol = rp.cg_tol;
    std::vector<double> R(9 * n);
    std::vector<uint8_t> reg(n);
    std::vector<float> perr(np);
    ps_rotation_report rrep;
    if (ps_rotation_averaging(0, n, (int)np, flat.data(), d_rec, &rprm, R.data(), reg.data(), perr.data(), &rrep) != PS_OK) {
        std::printf("FAIL ps_rotation_averaging: %s\n", ps_last_error(nullptr));
        return 1;
    }
    for (int k = 0; k < n; ++k)
        if (std::memcmp(rot.R[k].R, &R[9 * k], 72) || rot.registered[k] != (reg[k] != 0)) { std::printf("FAIL rotation %d differs\n", k); return 1; }
    if (std::memcmp(rot.pair_error.data(), perr.data(), np * 4) || std::memcmp(&rot.report.final_cost, &rrep.final_cost, 8) ||
        rot.report.iterations != rrep.iterations || rot.report.cg_iterations != rrep.cg_iterations || rot.report.n_pairs != rrep.n_pairs ||
        rot.report.n_registered != rrep.n_registered || rot.report.termination != rrep.termination) {
        std::printf("FAIL rotation reports differ\n");
        return 1;
    }
    std::vector<int32_t> n_feat(n), mem(nm), off(n + 1, 0);
    std::vector<const ps_feature*> feat(n);
    std::vector<ps_camera> c_cams(n);
    for (int k = 0; k < n; ++k) {
        n_feat[k] = sets[k]->getFeatureCount();
        off[k + 1] = off[k] + n_feat[k];
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        c_cams[k] = ps_camera{cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy};
    }
    for (size_t m = 0; m < nm; ++m) mem[m] = off[tracks.set[m]] + tracks.feature[m];
    int32_t* d_start = static_cast<int32_t*>(ps_dev_alloc((nt + 1) * sizeof(int32_t)));
    int32_t* d_mem = static_cast<int32_t*>(ps_dev_alloc(std::max<size_t>(nm, 1) * sizeof(int32_t)));
    double* d_X = static_cast<double*>(ps_dev_alloc(std::max<size_t>(nt, 1) * 24));
    if (!d_start || !d_mem || !d_X) { std::printf("FAIL alloc\n"); return 1; }
    ps_host_to_dev(d_start, tracks.start.data(), (nt + 1) * sizeof(int32_t));
    ps_host_to_dev(d_mem, mem.data(), nm * sizeof(int32_t));
    ps_position_params gprm{};
    gprm.loss = PS_LOSS_HUBER;
    gprm.max_iters = gp.max_iters;
    gprm.cg_max_iters = gp.cg_max_iters;
    gprm.loss_scale = gp.loss_scale;
    gprm.function_tol = gp.function_tol;
    gprm.cg_tol = gp.cg_tol;
    std::vector<ps_rigid> out(n);
    std::vector<uint8_t> positioned(n);
    ps_position_report grep;
    if (ps_global_positioning(0, n, n_feat.data(), feat.data(), c_cams.data(), R.data(), reg.data(), (int)nt, d_start, d_mem, (int)nm, &gprm,
                              out.data(), positioned.data(), d_X, &grep) != PS_OK) {
        std::printf("FAIL ps_global_positioning: %s\n", ps_last_error(nullptr));
        return 1;
    }
    std::vector<double> X(3 * nt);
    ps_dev_to_host(X.data(), d_X, nt * 24);
    if (std::memcmp(X.data(), pos.X.data(), nt * 24)) { std::printf("FAIL points differ\n"); return 1; }
    for (int k = 0; k < n; ++k)
        if (std::memcmp(pos.poses[k].R, out[k].R, 72) || std::memcmp(pos.poses[k].t, out[k].t, 24) || pos.positioned[k] != (positioned[k] != 0)) {
            std::printf("FAIL pose %d differs\n", k);
            return 1;
        }
    const popsift::PositionReport& r = pos.report;
    if (std::memcmp(&r.initial_cost, &grep.initial_cost, 8) || std::memcmp(&r.final_cost, &grep.final_cost, 8) || r.iterations != grep.iterations ||
        r.cg_iterations != grep.cg_iterations || r.n_obs != grep.n_obs || r.n_points != grep.n_points || r.n_cams != grep.n_cams ||
        r.termination != grep.termination) {
        std::printf("FAIL positioning reports differ\n");
        return 1;
    }
    std::printf("OK %d %d %.6g\n", rrep.n_registered, grep.n_obs, grep.final_cost);
    for (void* p : {(void*)d_rec, (void*)d_start, (void*)d_mem, (void*)d_X}) ps_dev_free(p);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
