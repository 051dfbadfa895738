// Host build of k_depth.h, the per-pixel math of the depth kernels, for tests/test_depth_cpu.py.  Reads one request per
// line from stdin and prints one result line each ("= v ...", %.17g):
//   h Kr(4) Rr(9) tr(3) Ks(4) Rs(9) ts(3)               dp_homography: H(9) b(3)
//   w H(9) b(3) x y iota w_s h_s                          dp_warp<double>: valid u v
//   n m A AA B BB AB floor_m2                             dp_ncc: valid c
//   a nv top_k min_sources c_1 .. c_n                     dp_insert<32> of the float costs, then dp_mean<float, 32>
//   p cm c0 cp k n                                        dp_parabola<double> (inf spelled "inf")
//   c Kr(4) Rr(9) tr(3) wr hr Ks(4) Rs(9) ts(3) ws hs x y D Dq max_reproj max_diff
//                                                         dp_lookup then dp_consistent at Dq: found qx qy zs consistent
#include "k_depth.h"

#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

using namespace psb;

static DpCam cam_of(const double* a)
{
    DpCam c;
    for (int k = 0; k < 4; ++k) c.K[k] = a[k];
    for (int k = 0; k < 9; ++k) c.R[k] = a[4 + k];
    for (int k = 0; k < 3; ++k) c.t[k] = a[13 + k];
    c.w = (int32_t)a[16];
    c.h = (int32_t)a[17];
    return c;
}

int main()
{
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op, tok;
        in >> op;
        std::vector<double> a;
        while (in >> tok) a.push_back(std::strtod(tok.c_str(), nullptr));
        if (op == "h" && a.size() == 32) {
            double H[9], b[3];
            dp_homography(a.data(), a.data() + 4, a.data() + 13, a.data() + 16, a.data() + 20, a.data() + 29, H, b);
            std::printf("=");
            for (double v : H) std::printf(" %.17g", v);
            for (double v : b) std::printf(" %.17g", v);
            std::printf("\n");
        } else if (op == "w" && a.size() == 17) {
            double u = 0.0, v = 0.0;
            const bool ok = dp_warp<double>(a.data(), a.data() + 9, a[12], a[13], a[14], a[15], a[16], u, v);
            std::printf("= %d %.17g %.17g\n", ok ? 1 : 0, u, v);
        } else if (op == "n" && a.size() == 7) {
            double c = 0.0;
            const bool ok = dp_ncc(a[0], a[1], a[2], a[3], a[4], a[5], a[6], c);
            std::printf("= %d %.17g\n", ok ? 1 : 0, c);
        } else if (op == "a" && a.size() >= 3) {
            float top[32];
            for (float& t : top) t = INFINITY;
            for (size_t k = 3; k < a.size(); ++k) dp_insert<32>(top, (float)a[k]);
            const float C = dp_mean<float, 32>(top, (int)(a.size() - 3), (int)a[1], (int)a[2]);
            (void)a[0];
            std::printf("= %.17g\n", (double)C);
        } else if (op == "p" && a.size() == 5) {
            std::printf("= %.17g\n", dp_parabola<double>(a[0], a[1], a[2], (int)a[3], (int)a[4]));
        } else if (op == "c" && a.size() == 42) {
            const DpCam r = cam_of(a.data()), s = cam_of(a.data() + 18);
            int qx = 0, qy = 0;
            double zs = 0.0;
            const bool found = dp_lookup(r, s, a[36], a[37], a[38], qx, qy, zs);
            const bool cons = found && a[39] > 0.0 && dp_consistent(r, s, a[36], a[37], qx, qy, zs, a[39], a[40], a[41]);
            std::printf("= %d %d %d %.17g %d\n", found ? 1 : 0, qx, qy, zs, cons ? 1 : 0);
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
    }
    return 0;
}
