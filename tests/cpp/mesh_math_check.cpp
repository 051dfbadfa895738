// Host build of k_mesh.h, the per-voxel math of the mesh kernels, for tests/test_mesh_cpu.py.  Reads one request per line
// from stdin and prints one result line each ("= v ..."; doubles as %.17g, floats as %.9g, both exact round trips):
//   p origin(3) voxel i j k R(9) t(3) K(4) w h     ts_point, ts_to_camera, ts_pixel: X(3) Xc(3) found qx qy
//   t D z trunc                                    ts_tau: ok tau
//   u T W G tau grey                               ts_update: T W G
//   v o(3) h ax ay az d Ta Tb Ga Gb                ts_vertex: X(3) grey
//   c mask                                         ts_cell_counts: n_edges n_tris
//   k                                              the tables: kKuhnTet (24), kTetTriCount (16), kTetTri (576), kCellEdge (19)
#include "k_mesh.h"

#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

using namespace psb;

int main()
{
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op, tok;
        in >> op;
        std::vector<double> a;
        while (in >> tok) a.push_back(std::strtod(tok.c_str(), nullptr));
        if (op == "p" && a.size() == 25) {
            double X[3], Xc[3];
            ts_point(a.data(), a[3], (int)a[4], (int)a[5], (int)a[6], X);
            ts_to_camera(a.data() + 7, a.data() + 16, X, Xc);
            int qx = -1, qy = -1;
            const bool ok = ts_pixel(a.data() + 19, (int)a[23], (int)a[24], Xc, qx, qy);
            std::printf("= %.17g %.17g %.17g %.17g %.17g %.17g %d %d %d\n", X[0], X[1], X[2], Xc[0], Xc[1], Xc[2], ok ? 1 : 0, qx, qy);
        } else if (op == "t" && a.size() == 3) {
            float tau = 0.0f;
            const bool ok = ts_tau((float)a[0], a[1], (float)a[2], tau);
            std::printf("= %d %.9g\n", ok ? 1 : 0, (double)tau);
        } else if (op == "u" && a.size() == 5) {
            float T = (float)a[0], W = (float)a[1], G = (float)a[2];
            ts_update(T, W, G, (float)a[3], (float)a[4]);
            std::printf("= %.9g %.9g %.9g\n", (double)T, (double)W, (double)G);
        } else if (op == "v" && a.size() == 12) {
            const float o[3] = {(float)a[0], (float)a[1], (float)a[2]};
            float X[3], grey;
            ts_vertex(o, (float)a[3], (int)a[4], (int)a[5], (int)a[6], (int)a[7], (float)a[8], (float)a[9], (float)a[10], (float)a[11], X, grey);
            std::printf("= %.9g %.9g %.9g %.9g\n", (double)X[0], (double)X[1], (double)X[2], (double)grey);
        } else if (op == "c" && a.size() == 1) {
            int ne, nt;
            ts_cell_counts((unsigned)a[0], ne, nt);
            std::printf("= %d %d\n", ne, nt);
        } else if (op == "k") {
            std::printf("=");
            for (const auto& t : kKuhnTet)
                for (int c : t) std::printf(" %d", c);
            for (int c : kTetTriCount) std::printf(" %d", c);
            for (const auto& t : kTetTri)
                for (const auto& cs : t)
                    for (const auto& tr : cs)
                        for (int e : tr) std::printf(" %d", e);
            for (int e : kCellEdge) std::printf(" %d", e);
            std::printf("\n");
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
    }
    return 0;
}
