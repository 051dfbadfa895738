// Host-side runs of ps_relative_pose_batch's math: the same __host__ __device__ functions the kernels use
// (k_pose_solve.h, k_verify_sample.h), compiled with a plain host compiler.  tests/test_pose_cpu.py writes the inputs
// and compares the outputs with tests/pose_oracle.py.
//   pose_solver_check solve  in out   in: int64 N, N x 20 doubles (five calibrated rows); out: N int32 counts, then
//                                     N x 10 x 9 doubles (the solutions in slot order, zero beyond the count)
//   pose_solver_check pose   in out   in: int64 N, int64 M, per scene 9 doubles E then M x 4 doubles (calibrated rows);
//                                     out: per scene int32 winner and 4 int32 counts, then per scene R (9) and t (3)
//   pose_solver_check sample in out   in: uint64 seed, int64 N, N x (int32 p, int32 s, uint32 n); out: N x (int32 valid,
//                                     5 uint32 indices)
#include "k_pose_solve.h"
#include "k_verify_sample.h"

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

using namespace psb;

template <class T>
static bool rd(FILE* f, T* p, size_t n) { return fread(p, sizeof(T), n, f) == n; }

int main(int argc, char** argv)
{
    if (argc != 4) { fprintf(stderr, "usage: pose_solver_check solve|pose|sample in out\n"); return 2; }
    FILE* in = fopen(argv[2], "rb");
    FILE* out = fopen(argv[3], "wb");
    if (!in || !out) { fprintf(stderr, "cannot open files\n"); return 2; }
    const std::string mode = argv[1];
    if (mode == "solve") {
        int64_t N = 0;
        if (!rd(in, &N, 1)) return 3;
        std::vector<double> p(N * 20);
        if (!rd(in, p.data(), p.size())) return 3;
        std::vector<int32_t> cnt(N);
        std::vector<double> sol(N * kPoseSlots * 9, 0.0);
        for (int64_t i = 0; i < N; ++i) {
            double q[5][4], Es[kPoseSlots][9];
            for (int j = 0; j < 5; ++j)
                for (int k = 0; k < 4; ++k) q[j][k] = p[i * 20 + 4 * j + k];
            cnt[i] = pose_five_point(q, Es);
            for (int j = 0; j < cnt[i]; ++j) {
                double e[9];
                if (!pose_scale(Es[j], e)) continue;
                for (int k = 0; k < 9; ++k) sol[(i * kPoseSlots + j) * 9 + k] = e[k];
            }
        }
        fwrite(cnt.data(), 4, N, out);
        fwrite(sol.data(), 8, sol.size(), out);
    } else if (mode == "pose") {
        int64_t N = 0, M = 0;
        if (!rd(in, &N, 1) || !rd(in, &M, 1)) return 3;
        std::vector<int32_t> head(N * 5);
        std::vector<double> rt(N * 12, 0.0);
        std::vector<double> buf(9 + 4 * M);
        for (int64_t i = 0; i < N; ++i) {
            if (!rd(in, buf.data(), buf.size())) return 3;
            double E[9], U[3][3], V[3][3], R[4][9], t[4][3];
            for (int k = 0; k < 9; ++k) E[k] = buf[k];
            int c[4] = {0, 0, 0, 0};
            if (pose_svd(E, U, V)) {
                pose_candidates(U, V, R, t);
                for (int64_t r = 0; r < M; ++r) {
                    const double* q = &buf[9 + 4 * r];
                    for (int k = 0; k < 4; ++k) c[k] += pose_front(R[k], t[k], q[0], q[1], q[2], q[3]) ? 1 : 0;
                }
            }
            int best = 0;
            for (int k = 1; k < 4; ++k) if (c[k] > c[best]) best = k;
            head[i * 5] = best;
            for (int k = 0; k < 4; ++k) head[i * 5 + 1 + k] = c[k];
            for (int k = 0; k < 9; ++k) rt[i * 12 + k] = R[best][k];
            for (int k = 0; k < 3; ++k) rt[i * 12 + 9 + k] = t[best][k];
        }
        fwrite(head.data(), 4, head.size(), out);
        fwrite(rt.data(), 8, rt.size(), out);
    } else if (mode == "sample") {
        uint64_t seed = 0;
        int64_t N = 0;
        if (!rd(in, &seed, 1) || !rd(in, &N, 1)) return 3;
        std::vector<int32_t> rec(N * 3);
        if (!rd(in, rec.data(), rec.size())) return 3;
        std::vector<uint32_t> res(N * 6);
        for (int64_t i = 0; i < N; ++i) {
            uint32_t idx[5];
            const bool ok = verify_sample<5>(seed, rec[3 * i], rec[3 * i + 1], (uint32_t)rec[3 * i + 2], idx);
            res[6 * i] = ok ? 1u : 0u;
            for (int k = 0; k < 5; ++k) res[6 * i + 1 + k] = idx[k];
        }
        fwrite(res.data(), 4, res.size(), out);
    } else {
        return 2;
    }
    fclose(out);
    fclose(in);
    return 0;
}
