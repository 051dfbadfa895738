// popsift::renderMesh / textureMesh against the C ABI (ps_mesh_render, ps_mesh_texture) on the same mesh and device
// images: the maps, the atlas and the views must be identical bytes.
//   render_check W H N n_vertices n_triangles vertices.raw triangles.raw img_0.raw .. img_{N-1}.raw
//                then per view: fx fy cx cy R(9) t(3)
// Prints "OK <drawn> <covered> <viewed>".
#include "popsift/features.h"
#include "popsift_b200.h"
#include "popsift_b200_render.h"

#include <cmath>
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
    if (argc < 8) return fail("usage");
    const int W = std::atoi(argv[1]), H = std::atoi(argv[2]), N = std::atoi(argv[3]);
    const long long nv = std::atoll(argv[4]), nt = std::atoll(argv[5]);
    if (argc != 8 + N + 16 * N) return fail("argument count");
    popsift::Mesh mesh;
    const std::vector<char> vb = read_file(argv[6]), tb = read_file(argv[7]);
    if ((long long)vb.size() != nv * 16 || (long long)tb.size() != nt * 12) return fail("mesh files");
    mesh.vertices.resize(nv);
    mesh.triangles.resize(3 * nt);
    std::memcpy(mesh.vertices.data(), vb.data(), vb.size());
    std::memcpy(mesh.triangles.data(), tb.data(), tb.size());
    std::vector<popsift::DeviceImage> images(N);
    std::vector<ps_image> c_img(N);
    std::vector<void*> dev;
    for (int v = 0; v < N; ++v) {
        const std::vector<char> px = read_file(argv[8 + v]);
        if ((int)px.size() != W * H) return fail("image size");
        void* d = ps_dev_alloc(px.size());
        dev.push_back(d);
        if (ps_host_to_dev(d, px.data(), px.size()) != PS_OK) return fail("upload");
        images[v].data = static_cast<const uint8_t*>(d);
        images[v].pitch = W;
        images[v].width = W;
        images[v].height = H;
        c_img[v] = ps_image{images[v].data, W, W, H};
    }
    std::vector<popsift::Camera> cams(N);
    std::vector<popsift::Rigid> poses(N);
    std::vector<ps_camera> c_cam(N);
    std::vector<ps_rigid> c_pose(N);
    int a = 8 + N;
    for (int v = 0; v < N; ++v) {
        cams[v] = popsift::Camera{(float)std::atof(argv[a]), (float)std::atof(argv[a + 1]), (float)std::atof(argv[a + 2]), (float)std::atof(argv[a + 3])};
        a += 4;
        for (int k = 0; k < 9; ++k) poses[v].R[k] = c_pose[v].R[k] = std::atof(argv[a++]);
        for (int k = 0; k < 3; ++k) poses[v].t[k] = c_pose[v].t[k] = std::atof(argv[a++]);
        c_cam[v] = ps_camera{cams[v].fx, cams[v].fy, cams[v].cx, cams[v].cy};
    }
    std::vector<std::pair<int, int>> sizes(N, std::make_pair(W, H));
    popsift::RenderedMesh r;
    popsift::TexturedMesh t;
    try {
        r = popsift::renderMesh(mesh, cams, poses, sizes);
        t = popsift::textureMesh(mesh, images, cams, poses);
    } catch (const std::exception& e) {
        std::printf("FAIL C++ API: %s\n", e.what());
        return 1;
    }
    // the same through the C ABI
    void* d_v = ps_dev_alloc(vb.size() + 16);
    void* d_t = ps_dev_alloc(tb.size() + 16);
    ps_host_to_dev(d_v, vb.data(), vb.size());
    ps_host_to_dev(d_t, tb.data(), tb.size());
    std::vector<float*> d_depth(N);
    std::vector<int32_t*> d_tri(N);
    std::vector<int32_t> sz;
    for (int v = 0; v < N; ++v) {
        d_depth[v] = static_cast<float*>(ps_dev_alloc((size_t)W * H * 4));
        d_tri[v] = static_cast<int32_t*>(ps_dev_alloc((size_t)W * H * 4));
        sz.insert(sz.end(), {W, H});
    }
    const ps_render_params rp{1e-3f, 0};
    ps_render_report rrep;
    if (ps_mesh_render(0, N, sz.data(), c_cam.data(), c_pose.data(), static_cast<const ps_mesh_vertex*>(d_v), nv, static_cast<const int32_t*>(d_t), nt,
                       &rp, d_depth.data(), d_tri.data(), &rrep) != PS_OK)
        return fail("ps_mesh_render");
    if (rrep.n_drawn != r.n_drawn || rrep.n_big != r.n_big || rrep.n_covered != r.n_covered) return fail("render report");
    std::vector<float> D((size_t)W * H);
    std::vector<int> T((size_t)W * H);
    for (int v = 0; v < N; ++v) {
        ps_dev_to_host(D.data(), d_depth[v], D.size() * 4);
        ps_dev_to_host(T.data(), d_tri[v], T.size() * 4);
        if (std::memcmp(D.data(), r.maps[v].depth.data(), D.size() * 4) || std::memcmp(T.data(), r.maps[v].triangle.data(), T.size() * 4))
            return fail("maps");
    }
    const int cpr = std::max(1, std::min((int)std::ceil(std::sqrt((double)std::max(nt, 1LL))), 65535 / 8));
    if (t.cells_per_row != cpr || t.width != cpr * 8 || t.height != (int)((nt + cpr - 1) / cpr) * 8) return fail("atlas size");
    void* d_atlas = ps_dev_alloc((size_t)t.width * t.height + 16);
    void* d_view = ps_dev_alloc((size_t)nt * 4 + 16);
    const ps_texture_params tp{8, cpr, 0.01f, 0.1f, 1e-3f, 0};
    ps_texture_report trep;
    std::vector<const float*> c_depth(d_depth.begin(), d_depth.end());
    if (ps_mesh_texture(0, N, c_img.data(), c_cam.data(), c_pose.data(), c_depth.data(), static_cast<const ps_mesh_vertex*>(d_v), nv,
                        static_cast<const int32_t*>(d_t), nt, &tp, static_cast<uint8_t*>(d_atlas), static_cast<int32_t*>(d_view), &trep) != PS_OK)
        return fail("ps_mesh_texture");
    std::vector<uint8_t> atlas(t.atlas.size());
    std::vector<int> view((size_t)nt);
    ps_dev_to_host(atlas.data(), d_atlas, atlas.size());
    ps_dev_to_host(view.data(), d_view, view.size() * 4);
    if (atlas != t.atlas || view != t.view || trep.n_viewed != t.n_viewed || trep.n_fallback != t.n_fallback) return fail("texture");
    for (void* p : dev) ps_dev_free(p);
    for (int v = 0; v < N; ++v) {
        ps_dev_free(d_depth[v]);
        ps_dev_free(d_tri[v]);
    }
    ps_dev_free(d_v);
    ps_dev_free(d_t);
    ps_dev_free(d_atlas);
    ps_dev_free(d_view);
    std::printf("OK %lld %lld %lld\n", (long long)r.n_drawn, (long long)r.n_covered, (long long)t.n_viewed);
    return 0;
}
