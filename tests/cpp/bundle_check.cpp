// popsift::bundleAdjust through the C++ API against the C ABI on the same tracks and points: n frames extracted under
// Config::MatchingMode, every pair (i, j), i < j, matched with matchPairs, verified with verifyPairs (fundamental
// matrices), tracks from buildTracks, points from triangulateTracks at the given poses, then bundle adjustment with view 0
// fixed and component 0 of view 1's t held (Cauchy loss, s = 2 px).  The C path uploads the same arrays and runs
// ps_bundle_adjust itself; poses, points, pixel errors and reports must be identical.
// Usage: bundle_check W H n f_0.raw .. f_{n-1}.raw then per view fx fy cx cy R[9] t[3]
//   prints "OK <used observations> <accepted steps> <final cost>" or FAIL
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>
#include <popsift_b200_bundle.h>

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
    if (argc < 4) { std::fprintf(stderr, "usage: bundle_check W H n frames.. (fx fy cx cy R[9] t[3]) per view\n"); return 2; }
    const int w = std::atoi(argv[1]), h = std::atoi(argv[2]), n = std::atoi(argv[3]);
    if (n < 2 || argc != 4 + n + 16 * n) { std::fprintf(stderr, "bad argument count\n"); return 2; }
    std::vector<popsift::Camera> cams(n);
    std::vector<popsift::Rigid> poses(n);
    for (int k = 0; k < n; ++k) {
        const char* const* a = argv + 4 + n + 16 * k;
        cams[k] = popsift::Camera{(float)std::atof(a[0]), (float)std::atof(a[1]), (float)std::atof(a[2]), (float)std::atof(a[3])};
        for (int j = 0; j < 9; ++j) poses[k].R[j] = std::atof(a[4 + j]);
        for (int j = 0; j < 3; ++j) poses[k].t[j] = std::atof(a[13 + j]);
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
    popsift::VerifyParams vp;
    vp.model = popsift::VerifyParams::Fundamental;
    vp.threshold = 2.0f;
    const std::vector<popsift::PairGeometry> geo = popsift::verifyPairs(sets, pairs, matches, vp);
    const popsift::Tracks tracks = popsift::buildTracks(sets, pairs, matches, geo, 2);
    popsift::TriangulateParams tp;
    tp.max_error = 8.0f;
    const popsift::TrackPoints tri = popsift::triangulateTracks(sets, tracks, cams, poses, tp);
    std::vector<bool> fixed(n, false);
    fixed[0] = true;
    popsift::BundleParams bp;
    bp.loss = popsift::BundleParams::Cauchy;
    bp.loss_scale = 2.0;
    bp.max_iters = 20;
    bp.scale_set = 1;
    bp.scale_axis = 0;
    popsift::TrackPoints got = tri;
    const std::pair<std::vector<popsift::Rigid>, popsift::BundleReport> res = popsift::bundleAdjust(sets, tracks, cams, poses, fixed, got, bp);
    // bad arguments throw
    try {
        popsift::TrackPoints p = tri;
        popsift::bundleAdjust(sets, tracks, cams, poses, std::vector<bool>(n, false), p, bp);
        std::printf("FAIL no throw without a fixed set\n"); return 1;
    } catch (const std::runtime_error&) {}
    try {
        popsift::TrackPoints p = tri;
        popsift::BundleParams b2 = bp;
        b2.scale_axis = 3;
        popsift::bundleAdjust(sets, tracks, cams, poses, fixed, p, b2);
        std::printf("FAIL no throw on a bad scale axis\n"); return 1;
    } catch (const std::runtime_error&) {}

    const size_t nt = tracks.start.size() - 1, nm = tracks.set.size();
    std::vector<int32_t> n_feat(n), mem(nm);
    std::vector<const ps_feature*> feat(n);
    std::vector<ps_camera> c_cams(n);
    std::vector<ps_rigid> c_poses(n), c_out(n);
    std::vector<int32_t> off(n + 1, 0);
    std::vector<uint8_t> c_fixed(n, 0);
    c_fixed[0] = 1;
    for (int k = 0; k < n; ++k) {
        n_feat[k] = sets[k]->getFeatureCount();
        off[k + 1] = off[k] + n_feat[k];
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        c_cams[k] = ps_camera{cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy};
        std::memcpy(c_poses[k].R, poses[k].R, sizeof(c_poses[k].R));
        std::memcpy(c_poses[k].t, poses[k].t, sizeof(c_poses[k].t));
    }
    for (size_t m = 0; m < nm; ++m) mem[m] = off[tracks.set[m]] + tracks.feature[m];
    std::vector<ps_track_point> pts(nt);
    for (size_t t = 0; t < nt; ++t) {
        const popsift::TrackPoint& p = tri.points[t];
        std::memcpy(pts[t].X, p.X, sizeof(p.X));
        pts[t].error = p.error;
        pts[t].angle = p.angle;
        pts[t].n_inliers = p.n_inliers;
        pts[t].status = p.status;
    }
    int32_t* d_start = static_cast<int32_t*>(ps_dev_alloc((nt + 1) * sizeof(int32_t)));
    int32_t* d_mem = static_cast<int32_t*>(ps_dev_alloc(std::max<size_t>(nm, 1) * sizeof(int32_t)));
    ps_track_point* d_pts = static_cast<ps_track_point*>(ps_dev_alloc(std::max<size_t>(nt, 1) * sizeof(ps_track_point)));
    uint8_t* d_mask = static_cast<uint8_t*>(ps_dev_alloc(std::max<size_t>(nm, 1)));
    float* d_err = static_cast<float*>(ps_dev_alloc(std::max<size_t>(nm, 1) * sizeof(float)));
    if (!d_start || !d_mem || !d_pts || !d_mask || !d_err) { std::printf("FAIL alloc\n"); return 1; }
    ps_host_to_dev(d_start, tracks.start.data(), (nt + 1) * sizeof(int32_t));
    ps_host_to_dev(d_mem, mem.data(), nm * sizeof(int32_t));
    ps_host_to_dev(d_pts, pts.data(), nt * sizeof(ps_track_point));
    ps_host_to_dev(d_mask, tri.mask.data(), nm);
    ps_bundle_params prm{};
    prm.loss = PS_LOSS_CAUCHY;
    prm.max_iters = bp.max_iters;
    prm.cg_max_iters = bp.cg_max_iters;
    prm.scale_set = 1;
    prm.scale_axis = 0;
    prm.loss_scale = bp.loss_scale;
    prm.function_tol = bp.function_tol;
    prm.cg_tol = bp.cg_tol;
    prm.initial_lambda = bp.initial_lambda;
    ps_bundle_report rep;
    if (ps_bundle_adjust(0, n, n_feat.data(), feat.data(), c_cams.data(), c_poses.data(), (int)nt, d_start, d_mem, (int)nm, d_pts, d_mask,
                         c_fixed.data(), &prm, c_out.data(), d_err, &rep) != PS_OK) {
        std::printf("FAIL ps_bundle_adjust: %s\n", ps_last_error(nullptr));
        return 1;
    }
    std::vector<float> err(nm);
    ps_dev_to_host(pts.data(), d_pts, nt * sizeof(ps_track_point));
    ps_dev_to_host(err.data(), d_err, nm * sizeof(float));
    if (std::memcmp(got.obs_error.data(), err.data(), nm * sizeof(float))) { std::printf("FAIL pixel errors differ\n"); return 1; }
    for (int k = 0; k < n; ++k)
        if (std::memcmp(res.first[k].R, c_out[k].R, sizeof(c_out[k].R)) || std::memcmp(res.first[k].t, c_out[k].t, sizeof(c_out[k].t))) {
            std::printf("FAIL pose %d differs\n", k);
            return 1;
        }
    for (size_t t = 0; t < nt; ++t) {
        const popsift::TrackPoint& a = got.points[t];
        const ps_track_point& b = pts[t];
        if (std::memcmp(a.X, b.X, sizeof(a.X)) || std::memcmp(&a.error, &b.error, 4) || std::memcmp(&a.angle, &b.angle, 4) ||
            a.n_inliers != b.n_inliers || a.status != b.status) {
            std::printf("FAIL track %zu differs\n", t);
            return 1;
        }
    }
    const popsift::BundleReport& r = res.second;
    if (std::memcmp(&r.initial_cost, &rep.initial_cost, 8) || std::memcmp(&r.final_cost, &rep.final_cost, 8) || r.iterations != rep.iterations ||
        r.accepted != rep.accepted || r.cg_iterations != rep.cg_iterations || r.termination != rep.termination || r.n_obs != rep.n_obs ||
        r.n_points != rep.n_points || r.n_free_cams != rep.n_free_cams) {
        std::printf("FAIL reports differ\n");
        return 1;
    }
    std::printf("OK %d %d %.6g\n", rep.n_obs, rep.accepted, rep.final_cost);
    for (void* p : {(void*)d_start, (void*)d_mem, (void*)d_pts, (void*)d_mask, (void*)d_err}) ps_dev_free(p);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
