// popsift::filterViewGraph through the C++ API against the C ABI on the same input: a seeded planted view graph of 60
// sets (noisy relative rotations, 10 % random ones, some pairs below min_inliers, a self pair).  The C path uploads the
// same records and runs ps_view_graph_filter itself, with d_kept; keep, statistics and report must be identical, and
// d_kept must be the kept records.  A duplicate pair (reversed) must throw.
// Usage: viewgraph_check      prints "OK <triangles> <kept>" or FAIL
#include <popsift/features.h>
#include <popsift_b200.h>
#include <popsift_b200_viewgraph.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <stdexcept>
#include <utility>
#include <vector>

namespace {

void quat_rotation(double w, double x, double y, double z, double* R)
{
    const double n = std::sqrt(w * w + x * x + y * y + z * z);
    w /= n; x /= n; y /= n; z /= n;
    const double M[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    std::memcpy(R, M, sizeof(M));
}

} // namespace

int main()
{
    const int n = 60;
    std::mt19937 gen(7);
    std::normal_distribution<double> nd;
    std::uniform_real_distribution<double> ud(0.0, 1.0);
    std::vector<double> Rt(9 * n);
    for (int i = 0; i < n; ++i) quat_rotation(nd(gen), nd(gen), nd(gen), nd(gen), &Rt[9 * i]);
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j)
            if (j == i + 1 || ud(gen) < 0.25) pairs.push_back(ud(gen) < 0.5 ? std::make_pair(i, j) : std::make_pair(j, i));
    pairs.push_back({5, 5});
    std::vector<popsift::TwoViewPose> rel(pairs.size(), popsift::TwoViewPose{});
    for (size_t p = 0; p < pairs.size(); ++p) {
        const int l = pairs[p].first, r = pairs[p].second;
        double Rp[9];
        if (ud(gen) < 0.1) {
            quat_rotation(nd(gen), nd(gen), nd(gen), nd(gen), Rp);
        } else {
            double E[9];    // about 0.5 degree of noise: a quaternion (1, small)
            quat_rotation(1.0, 0.004 * nd(gen), 0.004 * nd(gen), 0.004 * nd(gen), E);
            double A[9];    // R_r R_l^T
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    A[3 * a + b] = Rt[9 * r + 3 * a] * Rt[9 * l + 3 * b] + Rt[9 * r + 3 * a + 1] * Rt[9 * l + 3 * b + 1] +
                                   Rt[9 * r + 3 * a + 2] * Rt[9 * l + 3 * b + 2];
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) Rp[3 * a + b] = E[3 * a] * A[b] + E[3 * a + 1] * A[3 + b] + E[3 * a + 2] * A[6 + b];
        }
        popsift::TwoViewPose& t = rel[p];
        for (int k = 0; k < 9; ++k) t.R[k] = (float)Rp[k];
        t.n_front = ud(gen) < 0.05 ? 5 : 30 + (int)(ud(gen) * 470);
        t.n_inliers = t.n_front;
    }
    popsift::ViewGraphParams vp;
    vp.min_fraction = 0.3;
    vp.keep_untested = true;
    const popsift::ViewGraph vg = popsift::filterViewGraph(n, pairs, rel, vp);
    try {
        std::vector<std::pair<int, int>> dup = pairs;
        dup.push_back({pairs[0].second, pairs[0].first});
        std::vector<popsift::TwoViewPose> rd = rel;
        rd.push_back(rel[0]);
        popsift::filterViewGraph(n, dup, rd, vp);
        std::printf("FAIL no throw on a duplicate pair\n");
        return 1;
    } catch (const std::runtime_error&) {}

    // the C ABI on the same input
    const size_t np = pairs.size();
    std::vector<ps_two_view> rec(np);
    std::vector<int32_t> flat(2 * np);
    for (size_t p = 0; p < np; ++p) {
        rec[p] = ps_two_view{};
        std::memcpy(rec[p].R, rel[p].R, sizeof(rec[p].R));
        std::memcpy(rec[p].t, rel[p].t, sizeof(rec[p].t));
        rec[p].n_inliers = rel[p].n_inliers;
        rec[p].n_front = rel[p].n_front;
        flat[2 * p] = pairs[p].first;
        flat[2 * p + 1] = pairs[p].second;
    }
    ps_two_view* d_rec = static_cast<ps_two_view*>(ps_dev_alloc(np * sizeof(ps_two_view)));
    ps_two_view* d_kept = static_cast<ps_two_view*>(ps_dev_alloc(np * sizeof(ps_two_view)));
    if (!d_rec || !d_kept) { std::printf("FAIL alloc\n"); return 1; }
    ps_host_to_dev(d_rec, rec.data(), np * sizeof(ps_two_view));
    ps_view_graph_params prm{};
    prm.min_inliers = vp.min_inliers;
    prm.min_consistent = vp.min_consistent;
    prm.keep_untested = 1;
    prm.max_cycle_error = vp.max_cycle_error;
    prm.min_fraction = vp.min_fraction;
    std::vector<uint8_t> keep(np);
    std::vector<ps_cycle_stats> cs(np);
    ps_view_graph_report rep;
    if (ps_view_graph_filter(0, n, (int)np, flat.data(), d_rec, &prm, keep.data(), cs.data(), d_kept, &rep) != PS_OK) {
        std::printf("FAIL ps_view_graph_filter: %s\n", ps_last_error(nullptr));
        return 1;
    }
    std::vector<ps_two_view> kept(rep.n_kept);
    ps_dev_to_host(kept.data(), d_kept, kept.size() * sizeof(ps_two_view));
    size_t k = 0;
    for (size_t p = 0; p < np; ++p) {
        const popsift::CycleStats& s = vg.stats[p];
        if (vg.keep[p] != (keep[p] != 0) || s.n_triangles != cs[p].n_triangles || s.n_consistent != cs[p].n_consistent ||
            std::memcmp(&s.min_error, &cs[p].min_error, 4)) {
            std::printf("FAIL pair %zu differs\n", p);
            return 1;
        }
        if (keep[p] && (k >= kept.size() || std::memcmp(&kept[k++], &rec[p], sizeof(ps_two_view)))) {
            std::printf("FAIL kept record %zu differs\n", p);
            return 1;
        }
    }
    const popsift::ViewGraphReport& r = vg.report;
    if (k != kept.size() || r.n_triangles != rep.n_triangles || r.n_consistent_triangles != rep.n_consistent_triangles ||
        r.n_used != rep.n_used || r.n_kept != rep.n_kept || r.n_untested != rep.n_untested || rep.n_used >= (int)np || rep.n_triangles == 0) {
        std::printf("FAIL reports differ\n");
        return 1;
    }
    std::printf("OK %lld %d\n", (long long)rep.n_triangles, rep.n_kept);
    ps_dev_free(d_rec);
    ps_dev_free(d_kept);
    return 0;
}
