// Host build of k_triangulate.h, the per-observation math of ps_triangulate_tracks, for tests/test_triangulate_cpu.py.
// Reads one case per line from stdin and prints one result line with every double as %.17g (exact round trip):
//   c R[9] t[3]                              -> c C[3]                       (camera centre)
//   d fx fy cx cy R[9] t[3] x y              -> d ok d[3]                    (unit ray direction)
//   h Ca[3] da[3] Cb[3] db[3] cos_min        -> h ok X[3]                    (two-ray hypothesis)
//   r fx fy cx cy R[9] t[3] X[3] x y         -> r ok ex ey Jx[3] Jy[3]       (pixel residual and Jacobian)
//   s S[10]                                  -> s ok dX[3]                   (Gauss-Newton step)
#include "k_triangulate.h"

#include <cstdio>
#include <cstring>

using namespace psb;

static bool read_n(double* v, int n)
{
    for (int i = 0; i < n; ++i)
        if (std::scanf("%lf", v + i) != 1) return false;
    return true;
}

static void print_n(const double* v, int n)
{
    for (int i = 0; i < n; ++i) std::printf(" %.17g", v[i]);
}

static bool read_cam(TriCam& K)
{
    double v[16];
    if (!read_n(v, 16)) return false;
    K.fx = v[0]; K.fy = v[1]; K.cx = v[2]; K.cy = v[3];
    std::memcpy(K.R, v + 4, sizeof(K.R));
    std::memcpy(K.t, v + 13, sizeof(K.t));
    tri_centre(K.R, K.t, K.C);
    return true;
}

int main()
{
    char tag[4];
    while (std::scanf("%3s", tag) == 1) {
        if (tag[0] == 'c') {
            double v[12], C[3];
            if (!read_n(v, 12)) return 2;
            tri_centre(v, v + 9, C);
            std::printf("c");
            print_n(C, 3);
        } else if (tag[0] == 'd') {
            TriCam K;
            double xy[2], d[3] = {0, 0, 0};
            if (!read_cam(K) || !read_n(xy, 2)) return 2;
            const bool ok = tri_direction(K, xy[0], xy[1], d);
            std::printf("d %d", ok ? 1 : 0);
            print_n(d, 3);
        } else if (tag[0] == 'h') {
            double v[13], X[3] = {0, 0, 0};
            if (!read_n(v, 13)) return 2;
            const bool ok = tri_hypothesis(v, v + 3, v + 6, v + 9, v[12], X);
            std::printf("h %d", ok ? 1 : 0);
            print_n(X, 3);
        } else if (tag[0] == 'r') {
            TriCam K;
            double v[5], e[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (!read_cam(K) || !read_n(v, 5)) return 2;
            const bool ok = tri_residual(K, v, v[3], v[4], e[0], e[1], e + 2, e + 5);
            std::printf("r %d", ok ? 1 : 0);
            print_n(e, 8);
        } else if (tag[0] == 's') {
            double S[10], dX[3] = {0, 0, 0};
            if (!read_n(S, 10)) return 2;
            const bool ok = tri_step(S, dX);
            std::printf("s %d", ok ? 1 : 0);
            print_n(dX, 3);
        } else {
            return 2;
        }
        std::printf("\n");
    }
    return 0;
}
