// Host build of k_global.h, the math the global-pose kernels run, for tests/test_global_cpu.py.  Reads one request per
// line from stdin and prints one result line each ("= v0 v1 ...", %.17g):
//   g R(9)                 gl_log(R)
//   q M(9)                 gl_orthonormal of M rounded to float
//   r Rl(9) Rr(9) Rp(9)    gl_pair_residual
//   u R(9) x(3)            gl_rot_update: R Exp(x)
//   o v(3) X(3) c(3)       gl_obs: d, e(3), |e|^2
#include "k_global.h"

#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

using namespace psb;

static void put(const double* v, int n)
{
    std::printf("=");
    for (int k = 0; k < n; ++k) std::printf(" %.17g", v[k]);
    std::printf("\n");
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
        if (op == "g" && a.size() == 9) {
            double w[3];
            gl_log(a.data(), w);
            put(w, 3);
        } else if (op == "q" && a.size() == 9) {
            float m[9];
            for (int k = 0; k < 9; ++k) m[k] = (float)a[k];
            double R[9];
            gl_orthonormal(m, R);
            put(R, 9);
        } else if (op == "r" && a.size() == 27) {
            double r[3];
            gl_pair_residual(a.data(), a.data() + 9, a.data() + 18, r);
            put(r, 3);
        } else if (op == "u" && a.size() == 12) {
            double R[9];
            gl_rot_update(a.data(), a.data() + 9, R);
            put(R, 9);
        } else if (op == "o" && a.size() == 9) {
            double d, e[3];
            const double e2 = gl_obs(a.data(), a.data() + 3, a.data() + 6, d, e);
            const double out[5] = {d, e[0], e[1], e[2], e2};
            put(out, 5);
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
    }
    return 0;
}
