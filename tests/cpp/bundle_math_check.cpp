// Host build of k_bundle.h, the per-observation math of ps_bundle_adjust, for tests/test_bundle_cpu.py.  Reads one case
// per line from stdin and prints one result line with every double as %.17g (exact round trip):
//   j fx fy cx cy R[9] t[3] X[3] x y   -> j ok e[2] Jc[12] Jp[6]      (residual and Jacobians)
//   l kind z                           -> l rho w                     (loss and IRLS weight)
//   u R[9] t[3] d[6]                   -> u Rn[9] tn[3]               (Rodrigues pose update)
//   c A[36]                            -> c ok L[36] x[6]             (6 x 6 Cholesky, and the solve of A x = (1..6))
//   i S[6]                             -> i ok I[6]                   (symmetric 3 x 3 inverse)
#include "k_bundle.h"

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

int main()
{
    char tag[4];
    while (std::scanf("%3s", tag) == 1) {
        if (tag[0] == 'j') {
            double v[21], out[20] = {0};
            if (!read_n(v, 21)) return 2;
            TriCam K;
            K.fx = v[0]; K.fy = v[1]; K.cx = v[2]; K.cy = v[3];
            std::memcpy(K.R, v + 4, sizeof(K.R));
            std::memcpy(K.t, v + 13, sizeof(K.t));
            tri_centre(K.R, K.t, K.C);
            const bool ok = ba_jacobian(K, v + 16, v[19], v[20], out, out + 2, out + 14);
            std::printf("j %d", ok ? 1 : 0);
            print_n(out, 20);
        } else if (tag[0] == 'l') {
            double v[2], rho = 0, w = 0;
            if (!read_n(v, 2)) return 2;
            ba_loss((int)v[0], v[1], rho, w);
            std::printf("l %.17g %.17g", rho, w);
        } else if (tag[0] == 'u') {
            double v[18], R[9], t[3];
            if (!read_n(v, 18)) return 2;
            ba_pose_update(v, v + 9, v + 12, R, t);
            std::printf("u");
            print_n(R, 9);
            print_n(t, 3);
        } else if (tag[0] == 'c') {
            double A[36], L[36], x[6] = {0, 0, 0, 0, 0, 0};
            const double b[6] = {1, 2, 3, 4, 5, 6};
            if (!read_n(A, 36)) return 2;
            const bool ok = ba_chol6(A, L);
            if (ok) ba_chol6_solve(L, b, x);
            std::printf("c %d", ok ? 1 : 0);
            print_n(L, 36);
            print_n(x, 6);
        } else if (tag[0] == 'i') {
            double S[6], I[6] = {0, 0, 0, 0, 0, 0};
            if (!read_n(S, 6)) return 2;
            const bool ok = ba_inv3(S, I);
            std::printf("i %d", ok ? 1 : 0);
            print_n(I, 6);
        } else {
            return 2;
        }
        std::printf("\n");
    }
    return 0;
}
