// popsift::depthMaps and popsift::filterDepthMaps against the C ABI (ps_depth_maps, ps_depth_filter) on the same device
// images: every set a reference with all the others as sources, 64 planes.  The maps, the consistency counts and the
// points must be identical bytes.
//   depth_check W H N img_0.raw .. img_{N-1}.raw  then per set: fx fy cx cy R(9) t(3) d_min d_max
// Prints "OK <pixels with a depth> <points>".
#include "popsift/features.h"
#include "popsift_b200.h"
#include "popsift_b200_depth.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

static int fail(const char* what)
{
    std::printf("FAIL %s: %s\n", what, ps_last_error(nullptr));
    return 1;
}

int main(int argc, char** argv)
{
    if (argc < 4) return fail("usage");
    const int W = std::atoi(argv[1]), H = std::atoi(argv[2]), N = std::atoi(argv[3]);
    if (argc != 4 + N + 18 * N) return fail("argument count");
    std::vector<popsift::DeviceImage> images(N);
    std::vector<ps_image> c_img(N);
    std::vector<popsift::Camera> cams(N);
    std::vector<ps_camera> c_cams(N);
    std::vector<popsift::Rigid> poses(N);
    std::vector<ps_rigid> c_poses(N);
    std::vector<std::pair<float, float>> ranges(N);
    std::vector<float> c_ranges;
    std::vector<void*> dev;
    for (int i = 0; i < N; ++i) {
        std::ifstream f(argv[4 + i], std::ios::binary);
        std::vector<char> px((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        if ((int)px.size() != W * H) return fail("image size");
        void* d = ps_dev_alloc(px.size());
        dev.push_back(d);
        if (ps_host_to_dev(d, px.data(), px.size()) != PS_OK) return fail("upload");
        images[i] = popsift::DeviceImage{static_cast<const std::uint8_t*>(d), W, W, H};
        c_img[i] = ps_image{static_cast<const uint8_t*>(d), W, W, H};
        const char* const* a = argv + 4 + N + 18 * i;
        cams[i] = popsift::Camera{(float)std::atof(a[0]), (float)std::atof(a[1]), (float)std::atof(a[2]), (float)std::atof(a[3])};
        c_cams[i] = ps_camera{cams[i].fx, cams[i].fy, cams[i].cx, cams[i].cy};
        for (int k = 0; k < 9; ++k) poses[i].R[k] = c_poses[i].R[k] = std::atof(a[4 + k]);
        for (int k = 0; k < 3; ++k) poses[i].t[k] = c_poses[i].t[k] = std::atof(a[13 + k]);
        ranges[i] = {(float)std::atof(a[16]), (float)std::atof(a[17])};
        c_ranges.insert(c_ranges.end(), {ranges[i].first, ranges[i].second});
    }
    std::vector<int> refs;
    std::vector<std::vector<int>> sources(N);
    std::vector<int32_t> c_refs, start{0}, src;
    for (int i = 0; i < N; ++i) {
        refs.push_back(i);
        c_refs.push_back(i);
        for (int j = 0; j < N; ++j)
            if (j != i) {
                sources[i].push_back(j);
                src.push_back(j);
            }
        start.push_back((int32_t)src.size());
    }
    popsift::DepthParams prm;
    prm.n_depths = 64;
    const popsift::DepthMaps maps = popsift::depthMaps(images, cams, poses, refs, sources, ranges, prm);
    popsift::DepthFilterParams fprm;
    const popsift::DensePoints pts = popsift::filterDepthMaps(images, cams, poses, refs, sources, maps, fprm);

    // the C ABI on device maps
    const size_t n = (size_t)W * H;
    std::vector<float*> d_depth(N), d_cost(N);
    std::vector<uint8_t*> d_nsrc(N), d_nc(N);
    for (int i = 0; i < N; ++i) {
        d_depth[i] = static_cast<float*>(ps_dev_alloc(n * 4));
        d_cost[i] = static_cast<float*>(ps_dev_alloc(n * 4));
        d_nsrc[i] = static_cast<uint8_t*>(ps_dev_alloc(n));
        d_nc[i] = static_cast<uint8_t*>(ps_dev_alloc(n));
        dev.insert(dev.end(), {(void*)d_depth[i], (void*)d_cost[i], (void*)d_nsrc[i], (void*)d_nc[i]});
    }
    const ps_depth_params cp{64, 3, 3, 1, 0.5f, 1.0f};
    ps_depth_report rep;
    if (ps_depth_maps(0, N, c_img.data(), c_cams.data(), c_poses.data(), N, c_refs.data(), c_ranges.data(), start.data(), src.data(), &cp,
                      d_depth.data(), d_cost.data(), d_nsrc.data(), &rep) != PS_OK)
        return fail("ps_depth_maps");
    if (rep.n_candidates != maps.n_candidates || rep.n_depths != maps.n_depths) return fail("depth report");
    std::vector<float> hf(n);
    std::vector<uint8_t> hb(n);
    for (int i = 0; i < N; ++i) {
        ps_dev_to_host(hf.data(), d_depth[i], n * 4);
        if (std::memcmp(hf.data(), maps.maps[i].depth.data(), n * 4)) return fail("depth bytes");
        ps_dev_to_host(hf.data(), d_cost[i], n * 4);
        if (std::memcmp(hf.data(), maps.maps[i].cost.data(), n * 4)) return fail("cost bytes");
        ps_dev_to_host(hb.data(), d_nsrc[i], n);
        if (std::memcmp(hb.data(), maps.maps[i].n_src.data(), n)) return fail("n_src bytes");
    }
    void* d_pts = ps_dev_alloc(N * n * sizeof(ps_dense_point));
    dev.push_back(d_pts);
    const ps_depth_filter_params cf{1.0f, 0.01f, 2, 0};
    ps_depth_filter_report frep;
    std::vector<const float*> cd(d_depth.begin(), d_depth.end());
    if (ps_depth_filter(0, N, c_img.data(), c_cams.data(), c_poses.data(), N, c_refs.data(), start.data(), src.data(), cd.data(), &cf,
                        d_nc.data(), static_cast<ps_dense_point*>(d_pts), &frep) != PS_OK)
        return fail("ps_depth_filter");
    if (frep.n_tested != pts.n_tested || frep.n_points != (long long)pts.points.size()) return fail("filter report");
    for (int i = 0; i < N; ++i) {
        ps_dev_to_host(hb.data(), d_nc[i], n);
        if (std::memcmp(hb.data(), pts.n_consistent[i].data(), n)) return fail("n_consistent bytes");
    }
    std::vector<ps_dense_point> cpts((size_t)frep.n_points);
    if (!cpts.empty()) ps_dev_to_host(cpts.data(), d_pts, cpts.size() * sizeof(ps_dense_point));
    for (size_t k = 0; k < cpts.size(); ++k) {
        const ps_dense_point& a = cpts[k];
        const popsift::DensePoint& b = pts.points[k];
        if (std::memcmp(a.X, b.X, sizeof(a.X)) || a.ref != b.ref || a.x != b.x || a.y != b.y || a.n_consistent != b.n_consistent ||
            a.grey != b.grey)
            return fail("point");
    }
    for (void* d : dev) ps_dev_free(d);
    std::printf("OK %lld %lld\n", (long long)rep.n_depths, (long long)frep.n_points);
    return 0;
}
