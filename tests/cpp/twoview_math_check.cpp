// Host build of k_twoview.h, the math the two-view configuration kernel runs, for tests/test_twoview_cpu.py.  Reads one
// request per line from stdin and prints one result line each ("=" and the values, %.17g):
//   k B(9)                     tv_kabsch: ok R0(9)
//   d H(9)                     tv_h_normalise, then tv_h_decompose of the normalised H: nd, then R(9) t(3) n(3) of each
//                              candidate (nd = 4), then the pruned indices (up to 4, -1 padded)
//   c H(9) xl yl xr yr ...     tv_h_normalise and tv_h_side: the number of rows with x_r^T H x_l > 0
//   f R(9) t(3) xl yl xr yr    pose_front: ok X(3), and tv_angle of X under (R, t)
#include "k_twoview.h"

#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

using namespace psb;

static void put(const double* v, int n)
{
    for (int i = 0; i < n; ++i) std::printf(" %.17g", v[i]);
}

int main()
{
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string op;
        in >> op;
        std::vector<double> a;
        double x;
        while (in >> x) a.push_back(x);
        if (op == "k" && a.size() == 9) {
            double B[9], R[9] = {0};
            for (int j = 0; j < 9; ++j) B[j] = a[j];
            const bool ok = tv_kabsch(B, R);
            std::printf("= %d", ok ? 1 : 0);
            put(R, 9);
        } else if (op == "d" && a.size() == 9) {
            double Hn[9], R[4][9], t[4][3], n[4][3];
            int nd = -2;
            if (tv_h_normalise(a.data(), Hn)) nd = tv_h_decompose(Hn, R, t, n);
            std::printf("= %d", nd);
            if (nd == 4) {
                for (int k = 0; k < 4; ++k) { put(R[k], 9); put(t[k], 3); put(n[k], 3); }
                int keep[4] = {-1, -1, -1, -1};
                tv_prune(n, keep);
                for (int k = 0; k < 4; ++k) std::printf(" %d", keep[k]);
            }
        } else if (op == "c" && a.size() >= 9 && (a.size() - 9) % 4 == 0) {
            double Hn[9];
            int c = -1;
            if (tv_h_normalise(a.data(), Hn)) {
                c = 0;
                for (size_t i = 9; i < a.size(); i += 4) c += tv_h_side(Hn, a[i], a[i + 1], a[i + 2], a[i + 3]) > 0.0 ? 1 : 0;
            }
            std::printf("= %d", c);
        } else if (op == "f" && a.size() == 16) {
            double X[3] = {0, 0, 0};
            const bool ok = pose_front(a.data(), a.data() + 9, a[12], a[13], a[14], a[15], X);
            std::printf("= %d", ok ? 1 : 0);
            put(X, 3);
            const double ang = ok ? tv_angle(X, a.data(), a.data() + 9) : 0.0;
            put(&ang, 1);
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
        std::printf("\n");
    }
    return 0;
}
