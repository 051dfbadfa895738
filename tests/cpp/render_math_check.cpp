// Host build of k_render.h, the per-element math of the render and texture kernels, for tests/test_render_cpu.py.  Reads
// one request per line from stdin and prints one result line each ("= v ..."; doubles as %.17g, floats as %.9g):
//   r K(4) R(9) t(3) w h z_near X0(3) X1(3) X2(3) x y    rd_project x 3, rd_setup, rd_cover at (x, y): drawn A box(4)
//                                                        covered z (float) key
//   f K(4) R(9) t(3) c(3) w h z_near tol1 min_cos V0(3) V1(3) V2(3) D(w h)
//                                                        tx_frame, tx_facing, tx_probe x 4, the score: facing visible score
//   u i j cell                                           tx_uv: u v
//   b w h x y I(w h)                                     tx_bilinear, tx_round: S texel
#include "k_render.h"

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
        if (op == "r" && a.size() == 30) {
            const int w = (int)a[16], h = (int)a[17];
            double p[3][2], z[3], A = 0.0;
            int box[4] = {0, 0, 0, 0};
            bool drawn = true;
            for (int k = 0; k < 3; ++k) drawn = rd_project(a.data(), a.data() + 4, a.data() + 13, a.data() + 19 + 3 * k, a[18], p[k], z[k]) && drawn;
            drawn = drawn && rd_setup(p, w, h, A, box);
            float zf = 0.0f;
            const bool cov = drawn && rd_cover(p, z, A, (int)a[28], (int)a[29], zf);
            std::printf("= %d %.17g %d %d %d %d %d %.9g %llu\n", drawn ? 1 : 0, drawn ? A : 0.0, box[0], box[1], box[2], box[3], cov ? 1 : 0,
                        (double)zf, cov ? rd_key(zf, 7) : 0ull);
        } else if (op == "f" && a.size() >= 33) {
            TxView V;
            for (int k = 0; k < 4; ++k) V.K[k] = a[k];
            for (int k = 0; k < 9; ++k) V.R[k] = a[4 + k];
            for (int k = 0; k < 3; ++k) V.t[k] = a[13 + k];
            for (int k = 0; k < 3; ++k) V.c[k] = a[16 + k];
            V.w = (int)a[19];
            V.h = (int)a[20];
            std::vector<float> D((size_t)V.w * V.h);
            if (a.size() != 33 + D.size()) { std::fprintf(stderr, "bad request: %s\n", line.c_str()); return 1; }
            for (size_t q = 0; q < D.size(); ++q) D[q] = (float)a[33 + q];
            V.depth = D.data();
            V.img = nullptr;
            V.pitch = 0;
            double P[4][3], n[3], p[4][2];
            for (int k = 0; k < 3; ++k)
                for (int c = 0; c < 3; ++c) P[k][c] = a[24 + 3 * k + c];
            tx_frame(P[0], P[1], P[2], P[3], n);
            const bool facing = tx_facing(n, P[3], V.c, (float)a[23]);
            bool vis = true;
            for (int k = 0; k < 4 && vis; ++k) vis = tx_probe(V, P[k], a[21], a[22], p[k]);
            const double score = vis ? fabs(rd_edge(p[0], p[1], p[2][0], p[2][1])) / 2.0 : 0.0;
            std::printf("= %d %d %.17g\n", facing ? 1 : 0, vis ? 1 : 0, score);
        } else if (op == "u" && a.size() == 3) {
            double u, v;
            tx_uv((int)a[0], (int)a[1], (int)a[2], u, v);
            std::printf("= %.17g %.17g\n", u, v);
        } else if (op == "b" && a.size() >= 4) {
            const int w = (int)a[0], h = (int)a[1];
            if (a.size() != 4 + (size_t)w * h) { std::fprintf(stderr, "bad request: %s\n", line.c_str()); return 1; }
            std::vector<uint8_t> I((size_t)w * h);
            for (size_t q = 0; q < I.size(); ++q) I[q] = (uint8_t)a[4 + q];
            const double S = tx_bilinear(I.data(), w, w, h, a[2], a[3]);
            std::printf("= %.17g %d\n", S, (int)tx_round(S));
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
    }
    return 0;
}
