// popsift::triangulateTracks through the C++ API against the C ABI on the same tracks: n frames extracted under
// Config::MatchingMode, every pair (i, j), i < j, matched with matchPairs, verified with verifyPairs (fundamental
// matrices), tracks from buildTracks, then triangulated from the given cameras and poses.  The C path uploads the same
// track arrays and runs ps_triangulate_tracks itself; points, masks, errors and counts must be identical.
// Usage: triangulate_check W H n f_0.raw .. f_{n-1}.raw then per view fx fy cx cy R[9] t[3]
//   prints "OK <tracks> <OK points> <inlier observations>" or FAIL
#include <popsift/features.h>
#include <popsift/popsift.h>
#include <popsift/sift_conf.h>
#include <popsift_b200.h>
#include <popsift_b200_triangulate.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <utility>
#include <vector>

int main(int argc, char** argv)
{
    if (argc < 4) { std::fprintf(stderr, "usage: triangulate_check W H n frames.. (fx fy cx cy R[9] t[3]) per view\n"); return 2; }
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
    tp.max_error = 2.0f;
    tp.seed = 5;
    const popsift::TrackPoints got = popsift::triangulateTracks(sets, tracks, cams, poses, tp);
    // bad arguments throw
    try {
        popsift::triangulateTracks(sets, tracks, cams, std::vector<popsift::Rigid>(1), tp);
        std::printf("FAIL no throw on a missing pose\n"); return 1;
    } catch (const std::runtime_error&) {}
    try {
        std::vector<popsift::Rigid> bad = poses;
        bad[1].R[0] = 2.0;
        popsift::triangulateTracks(sets, tracks, cams, bad, tp);
        std::printf("FAIL no throw on a non-rotation\n"); return 1;
    } catch (const std::runtime_error&) {}

    const size_t nt = tracks.start.size() - 1, nm = tracks.set.size();
    std::vector<int32_t> n_feat(n), mem(nm);
    std::vector<const ps_feature*> feat(n);
    std::vector<ps_camera> c_cams(n);
    std::vector<ps_rigid> c_poses(n);
    std::vector<int32_t> off(n + 1, 0);
    for (int k = 0; k < n; ++k) {
        n_feat[k] = sets[k]->getFeatureCount();
        off[k + 1] = off[k] + n_feat[k];
        feat[k] = reinterpret_cast<const ps_feature*>(sets[k]->getFeatures());
        c_cams[k] = ps_camera{cams[k].fx, cams[k].fy, cams[k].cx, cams[k].cy};
        std::memcpy(c_poses[k].R, poses[k].R, sizeof(c_poses[k].R));
        std::memcpy(c_poses[k].t, poses[k].t, sizeof(c_poses[k].t));
    }
    for (size_t m = 0; m < nm; ++m) mem[m] = off[tracks.set[m]] + tracks.feature[m];
    int32_t* d_start = static_cast<int32_t*>(ps_dev_alloc((nt + 1) * sizeof(int32_t)));
    int32_t* d_mem = static_cast<int32_t*>(ps_dev_alloc(std::max<size_t>(nm, 1) * sizeof(int32_t)));
    ps_track_point* d_pts = static_cast<ps_track_point*>(ps_dev_alloc(std::max<size_t>(nt, 1) * sizeof(ps_track_point)));
    uint8_t* d_mask = static_cast<uint8_t*>(ps_dev_alloc(std::max<size_t>(nm, 1)));
    float* d_err = static_cast<float*>(ps_dev_alloc(std::max<size_t>(nm, 1) * sizeof(float)));
    if (!d_start || !d_mem || !d_pts || !d_mask || !d_err) { std::printf("FAIL alloc\n"); return 1; }
    ps_host_to_dev(d_start, tracks.start.data(), (nt + 1) * sizeof(int32_t));
    ps_host_to_dev(d_mem, mem.data(), nm * sizeof(int32_t));
    ps_triangulate_params prm{tp.max_error, tp.min_angle, tp.min_views, tp.n_samples, tp.refine_iters, 0, tp.seed};
    ps_triangulate_counts cnt;
    if (ps_triangulate_tracks(0, n, n_feat.data(), feat.data(), c_cams.data(), c_poses.data(), (int)nt, d_start, d_mem, (int)nm, &prm, d_pts,
                              d_mask, d_err, &cnt) != PS_OK) { std::printf("FAIL ps_triangulate_tracks: %s\n", ps_last_error(nullptr)); return 1; }
    std::vector<ps_track_point> pts(nt);
    std::vector<uint8_t> mask(nm);
    std::vector<float> err(nm);
    ps_dev_to_host(pts.data(), d_pts, nt * sizeof(ps_track_point));
    ps_dev_to_host(mask.data(), d_mask, nm);
    ps_dev_to_host(err.data(), d_err, nm * sizeof(float));
    if (got.points.size() != nt || got.mask != mask || std::memcmp(got.obs_error.data(), err.data(), nm * sizeof(float)) ||
        std::memcmp(got.n_status, cnt.n_status, sizeof(cnt.n_status)) || got.n_inlier_obs != cnt.n_inlier_obs) {
        std::printf("FAIL member outputs or counts differ\n");
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
    std::printf("OK %zu %d %d\n", nt, cnt.n_status[PS_TRI_OK], cnt.n_inlier_obs);
    for (void* p : {(void*)d_start, (void*)d_mem, (void*)d_pts, (void*)d_mask, (void*)d_err}) ps_dev_free(p);
    for (popsift::FeaturesDev* fd : sets) delete fd;
    sift.uninit();
    return 0;
}
