// popsift::clearVolume / integrateDepthMaps / extractMesh against the C ABI (ps_volume_clear, ps_tsdf_integrate,
// ps_tsdf_mesh) on the same device images and depth maps: the two volumes and the two meshes must be identical bytes.
//   mesh_check W H N trunc min_weight voxel nx ny nz ox oy oz  img_0.raw depth_0.raw .. img_{N-1}.raw depth_{N-1}.raw
//              then per view: fx fy cx cy R(9) t(3)
// Prints "OK <updates> <vertices> <triangles>".
#include "popsift/features.h"
#include "popsift_b200.h"
#include "popsift_b200_mesh.h"

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

static std::vector<char> read_file(const char* path)
{
    std::ifstream f(path, std::ios::binary);
    return std::vector<char>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv)
{
    if (argc < 13) return fail("usage");
    const int W = std::atoi(argv[1]), H = std::atoi(argv[2]), N = std::atoi(argv[3]);
    const float trunc = (float)std::atof(argv[4]), min_weight = (float)std::atof(argv[5]);
    const double voxel = std::atof(argv[6]);
    const int nx = std::atoi(argv[7]), ny = std::atoi(argv[8]), nz = std::atoi(argv[9]);
    const double origin[3] = {std::atof(argv[10]), std::atof(argv[11]), std::atof(argv[12])};
    if (argc != 13 + 2 * N + 16 * N) return fail("argument count");
    std::vector<popsift::DeviceImage> images(N);
    std::vector<ps_image> c_img(N);
    std::vector<popsift::Camera> cams(N);
    std::vector<ps_camera> c_cams(N);
    std::vector<popsift::Rigid> poses(N);
    std::vector<ps_rigid> c_poses(N);
    std::vector<popsift::DepthMap> maps(N);
    std::vector<const float*> d_depth(N);
    std::vector<void*> dev;
    for (int i = 0; i < N; ++i) {
        const std::vector<char> px = read_file(argv[13 + 2 * i]), dm = read_file(argv[14 + 2 * i]);
        if ((int)px.size() != W * H || (int)dm.size() != 4 * W * H) return fail("input size");
        void* d = ps_dev_alloc(px.size());
        void* dd = ps_dev_alloc(dm.size());
        dev.push_back(d);
        dev.push_back(dd);
        if (ps_host_to_dev(d, px.data(), px.size()) != PS_OK || ps_host_to_dev(dd, dm.data(), dm.size()) != PS_OK) return fail("upload");
        images[i] = popsift::DeviceImage{static_cast<const std::uint8_t*>(d), W, W, H};
        c_img[i] = ps_image{static_cast<const uint8_t*>(d), W, W, H};
        maps[i].width = W;
        maps[i].height = H;
        maps[i].depth.resize((size_t)W * H);
        std::memcpy(maps[i].depth.data(), dm.data(), dm.size());
        d_depth[i] = static_cast<const float*>(dd);
        const char* const* a = argv + 13 + 2 * N + 16 * i;
        cams[i] = popsift::Camera{(float)std::atof(a[0]), (float)std::atof(a[1]), (float)std::atof(a[2]), (float)std::atof(a[3])};
        c_cams[i] = ps_camera{cams[i].fx, cams[i].fy, cams[i].cx, cams[i].cy};
        for (int k = 0; k < 9; ++k) poses[i].R[k] = c_poses[i].R[k] = std::atof(a[4 + k]);
        for (int k = 0; k < 3; ++k) poses[i].t[k] = c_poses[i].t[k] = std::atof(a[13 + k]);
    }
    const size_t n = (size_t)nx * ny * nz;
    // the C ABI, on a volume of its own
    ps_volume c_vol;
    for (int k = 0; k < 3; ++k) c_vol.origin[k] = origin[k];
    c_vol.voxel = voxel;
    c_vol.nx = nx;
    c_vol.ny = ny;
    c_vol.nz = nz;
    c_vol.pad_ = 0;
    c_vol.tsdf = static_cast<float*>(ps_dev_alloc(n * 4));
    c_vol.weight = static_cast<float*>(ps_dev_alloc(n * 4));
    c_vol.grey = static_cast<float*>(ps_dev_alloc(n * 4));
    if (ps_volume_clear(0, &c_vol) != PS_OK) return fail("ps_volume_clear");
    const ps_tsdf_params prm{trunc, 0};
    ps_tsdf_report rep;
    if (ps_tsdf_integrate(0, N, c_img.data(), c_cams.data(), c_poses.data(), d_depth.data(), nullptr, &prm, &c_vol, &rep) != PS_OK)
        return fail("ps_tsdf_integrate");
    const ps_mesh_params mprm{min_weight, 0};
    ps_mesh_report mrep;
    if (ps_tsdf_mesh(0, &c_vol, &mprm, 0, 0, nullptr, nullptr, &mrep) != PS_ERR_OVERFLOW) return fail("count call");
    void* d_v = ps_dev_alloc((size_t)mrep.n_vertices * sizeof(ps_mesh_vertex));
    void* d_t = ps_dev_alloc((size_t)mrep.n_triangles * 12);
    if (ps_tsdf_mesh(0, &c_vol, &mprm, mrep.n_vertices, mrep.n_triangles, static_cast<ps_mesh_vertex*>(d_v), static_cast<int32_t*>(d_t),
                     &mrep) != PS_OK)
        return fail("fill call");
    std::vector<ps_mesh_vertex> c_verts((size_t)mrep.n_vertices);
    std::vector<int32_t> c_tris((size_t)mrep.n_triangles * 3);
    if (ps_dev_to_host(c_verts.data(), d_v, c_verts.size() * sizeof(ps_mesh_vertex)) != PS_OK ||
        ps_dev_to_host(c_tris.data(), d_t, c_tris.size() * 4) != PS_OK)
        return fail("download");
    std::vector<float> c_host(3 * n);
    for (int q = 0; q < 3; ++q)
        if (ps_dev_to_host(c_host.data() + q * n, q == 0 ? c_vol.tsdf : q == 1 ? c_vol.weight : c_vol.grey, n * 4) != PS_OK) return fail("download");
    // the C++ API: a volume integrated twice from a cleared start (the first pass checks that clearVolume resets it)
    try {
        popsift::DeviceVolume vol(origin, voxel, nx, ny, nz);
        popsift::integrateDepthMaps(vol, images, cams, poses, maps, {}, popsift::TsdfParams{trunc, 0});
        popsift::clearVolume(vol);
        const popsift::TsdfReport r = popsift::integrateDepthMaps(vol, images, cams, poses, maps, {}, popsift::TsdfParams{trunc, 0});
        if (r.n_updates != rep.n_updates || r.n_voxels_touched != rep.n_voxels_touched) return fail("integration report");
        std::vector<float> host(3 * n);
        for (int q = 0; q < 3; ++q)
            if (ps_dev_to_host(host.data() + q * n, q == 0 ? vol.tsdf() : q == 1 ? vol.weight() : vol.grey(), n * 4) != PS_OK) return fail("download");
        if (std::memcmp(host.data(), c_host.data(), host.size() * 4) != 0) return fail("volumes differ");
        popsift::MeshParams mp;
        mp.min_weight = min_weight;
        const popsift::Mesh m = popsift::extractMesh(vol, mp);
        if (m.n_cells != mrep.n_cells || m.vertices.size() != c_verts.size() || m.triangles.size() != c_tris.size()) return fail("mesh sizes");
        if (!m.vertices.empty() && std::memcmp(m.vertices.data(), c_verts.data(), c_verts.size() * sizeof(ps_mesh_vertex)) != 0)
            return fail("vertices differ");
        if (!m.triangles.empty() && std::memcmp(m.triangles.data(), c_tris.data(), c_tris.size() * 4) != 0) return fail("triangles differ");
    } catch (const std::exception& e) {
        std::printf("FAIL %s\n", e.what());
        return 1;
    }
    for (void* p : {(void*)c_vol.tsdf, (void*)c_vol.weight, (void*)c_vol.grey, d_v, d_t}) ps_dev_free(p);
    for (void* p : dev) ps_dev_free(p);
    std::printf("OK %lld %lld %lld\n", (long long)rep.n_updates, (long long)mrep.n_vertices, (long long)mrep.n_triangles);
    return 0;
}
