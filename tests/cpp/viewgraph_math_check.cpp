// Host build of k_viewgraph.h, the cycle error the view-graph kernel computes, for tests/test_viewgraph_cpu.py.  Reads one
// request per line from stdin and prints one result line each ("= e", %.17g):
//   c Rab(9) t_ab Rbc(9) t_bc Rca(9) t_ca     vg_cycle_error (t_* 0 or 1: the pair is stored the other way round)
#include "k_viewgraph.h"

#include <cstdio>
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
        std::string op;
        in >> op;
        std::vector<double> a;
        double x;
        while (in >> x) a.push_back(x);
        if (op == "c" && a.size() == 30) {
            const double e = vg_cycle_error(a.data(), a[9] != 0.0, a.data() + 10, a[19] != 0.0, a.data() + 20, a[29] != 0.0);
            std::printf("= %.17g\n", e);
        } else {
            std::fprintf(stderr, "bad request: %s\n", line.c_str());
            return 1;
        }
    }
    return 0;
}
