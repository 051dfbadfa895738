// Host check of the batched matcher's planner (popsift_b200/csrc/k_match_plan.h) at the 8-bit matcher's pooled row size
// (kMatchU8RowBytes = 132 bytes: a u8 descriptor and its norm key).  Random set sizes (0, 1 and 129 among them), random pair
// lists with repeats and self pairs, 132 and 148 SMs, workspace caps from 300 KB to 1 GB.  For every plan: every group
// counts 132-byte rows, and every group of more than one pair fits the cap at that size; each (pair, left tile, right tile)
// is covered by exactly one item; a row's chunks are contiguous, start at the right set's first tile and number at most
// kMatchMaxChunks; the output offsets are the prefix sums of the left sizes; S = 1 whenever a group's left tiles alone fill
// the SMs; every pair with rows is in exactly one group; items address the pooled rows of their own pair's sets; the
// makespan model equals the items built.  Also: a plan asked for at the float row size is the default plan, item for item.
// Usage: match_plan_u8_check                                       the sweep, prints "OK ..." or a FAIL line
//        match_plan_u8_check plan SMS CAP N0,N1,... L0,R0,... ROW_BYTES   the group count and each group's S of one plan
#include "k_match_plan.h"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

using namespace psb;

#define FAIL(...) do { std::printf("FAIL case %d: ", cs); std::printf(__VA_ARGS__); std::printf("\n"); return 1; } while (0)

static bool same_plan(const MatchPlan& a, const MatchPlan& b)
{
    if (a.out_row != b.out_row || a.groups.size() != b.groups.size()) return false;
    for (size_t g = 0; g < a.groups.size(); ++g) {
        const MatchGroup &x = a.groups[g], &y = b.groups[g];
        if (x.rows != y.rows || x.cand_slots != y.cand_slots || x.left_rows != y.left_rows || x.chunks != y.chunks ||
            x.row_bytes != y.row_bytes || x.sets.size() != y.sets.size() || x.pairs.size() != y.pairs.size() ||
            x.items.size() != y.items.size())
            return false;
        if (!x.items.empty() && std::memcmp(x.items.data(), y.items.data(), x.items.size() * sizeof(MatchItem)) != 0) return false;
    }
    return true;
}

int main(int argc, char** argv)
{
    if (argc == 7 && std::string(argv[1]) == "plan") {
        auto ints = [](const char* s) { std::vector<int32_t> v; for (const char* p = s; *p; ) { v.push_back((int32_t)std::strtol(p, const_cast<char**>(&p), 10)); if (*p == ',') ++p; } return v; };
        const std::vector<int32_t> n = ints(argv[4]), pr = ints(argv[5]);
        const MatchPlan plan = plan_match((int)n.size(), n.data(), (int)pr.size() / 2, pr.data(), std::atoi(argv[2]),
                                          (size_t)std::strtoull(argv[3], nullptr, 10), (size_t)std::strtoull(argv[6], nullptr, 10));
        std::printf("groups=%zu S=", plan.groups.size());
        for (const MatchGroup& g : plan.groups) std::printf("%d,", g.chunks);
        std::printf("\n");
        return 0;
    }
    std::mt19937 rng(24680);
    const int special[] = {0, 1, 2, 127, 128, 129, 255, 257, 1000, 4097};
    long items_checked = 0, groups_seen = 0, split_groups = 0, multi_group_plans = 0;
    for (int cs = 0; cs < 1500; ++cs) {
        const int n_sets = 1 + (int)(rng() % 12);
        std::vector<int32_t> n_desc(n_sets);
        for (int i = 0; i < n_sets; ++i) {
            const int kind = (int)(rng() % 4);
            n_desc[i] = kind == 0 ? special[rng() % 10] : kind == 1 ? (int)(rng() % 300) : kind == 2 ? (int)(rng() % 9000) : (int)(rng() % 70000);
        }
        const int n_pairs = (int)(rng() % 40);
        std::vector<int32_t> pairs(2 * (size_t)n_pairs);
        for (int p = 0; p < n_pairs; ++p) {
            pairs[2 * p] = (int)(rng() % n_sets);
            pairs[2 * p + 1] = rng() % 5 == 0 ? pairs[2 * p] : (int)(rng() % n_sets);                     // self pairs
            if (p > 0 && rng() % 6 == 0) { pairs[2 * p] = pairs[2 * p - 2]; pairs[2 * p + 1] = pairs[2 * p - 1]; }   // repeats
        }
        const int sms = cs % 2 ? 148 : 132;
        const size_t caps[] = {(size_t)300 << 10, (size_t)1 << 20, (size_t)5 << 20, (size_t)1 << 30};
        const size_t cap = caps[rng() % 4];
        if (!same_plan(plan_match(n_sets, n_desc.data(), n_pairs, pairs.data(), sms, cap),
                       plan_match(n_sets, n_desc.data(), n_pairs, pairs.data(), sms, cap, kMatchRowBytes)))
            FAIL("the plan at the float row size differs from the default plan");
        const MatchPlan plan = plan_match(n_sets, n_desc.data(), n_pairs, pairs.data(), sms, cap, kMatchU8RowBytes);

        int64_t pre = 0;
        if ((int)plan.out_row.size() != n_pairs) FAIL("out_row size");
        for (int p = 0; p < n_pairs; ++p) {
            if (plan.out_row[p] != pre) FAIL("out_row[%d]", p);
            pre += n_desc[pairs[2 * p]];
        }
        std::vector<int> seen(n_pairs, 0);
        if (plan.groups.size() > 1) ++multi_group_plans;
        for (const MatchGroup& g : plan.groups) {
            ++groups_seen;
            if (g.pairs.empty()) FAIL("empty group");
            if (g.row_bytes != kMatchU8RowBytes) FAIL("group row bytes %zu", g.row_bytes);
            const size_t bytes = (size_t)g.rows * kMatchU8RowBytes + (size_t)g.cand_slots * kMatchCand * 4;
            if (g.bytes() != bytes) FAIL("group bytes %zu, want %zu", g.bytes(), bytes);
            if (g.pairs.size() > 1 && bytes > cap) FAIL("group of %zu pairs needs %zu bytes > cap %zu", g.pairs.size(), bytes, cap);
            if (g.chunks < 1 || g.chunks > kMatchMaxChunks) FAIL("S = %d", g.chunks);
            int64_t left_tiles = 0, rows = 0, slots = 0;
            for (const MatchGroupPair& gp : g.pairs) {
                const int nl = n_desc[pairs[2 * gp.pair]], nr = n_desc[pairs[2 * gp.pair + 1]];
                ++seen[gp.pair];
                if (gp.row != rows) FAIL("group row offsets");
                rows += nl;
                if (nr > 0) left_tiles += match_tiles(nl);
                if (gp.cand != slots) FAIL("candidate offsets");
                slots += (int64_t)nl * gp.chunks;
                if (nr == 0 ? gp.chunks != 0 : (gp.chunks < 1 || gp.chunks > g.chunks || gp.chunks > match_tiles(nr))) FAIL("pair chunks %d", gp.chunks);
            }
            if (rows != g.left_rows || slots != g.cand_slots) FAIL("group totals");
            if (left_tiles >= sms && g.chunks != 1) FAIL("S = %d although %lld left tiles fill %d SMs", g.chunks, (long long)left_tiles, sms);
            if (g.chunks > 1) ++split_groups;
            {
                const size_t G = std::min<size_t>((size_t)sms, g.items.size());
                int64_t worst = 0;
                for (size_t b = 0; b < G; ++b) {
                    int64_t t = 0;
                    for (size_t i = b; i < g.items.size(); i += G) t += 2 * (int64_t)g.items[i].b_tiles + 1;
                    worst = std::max(worst, t);
                }
                if (worst != plan_detail::makespan(g, n_desc.data(), pairs.data(), g.chunks, sms)) FAIL("makespan model");
            }
            int64_t prow = 0;
            std::vector<int64_t> set_row(n_sets, -1);
            for (const MatchGroupSet& s : g.sets) {
                if (s.row != prow || set_row[s.set] != -1) FAIL("pooled set rows");
                set_row[s.set] = s.row;
                prow += match_tiles(n_desc[s.set]) * kMatchTile;
            }
            if (prow != g.rows) FAIL("pooled row total");
            std::vector<std::vector<int>> cover(g.pairs.size());
            std::vector<std::vector<std::vector<std::pair<int, int>>>> chunks(g.pairs.size());
            for (size_t k = 0; k < g.pairs.size(); ++k) {
                const int nl = n_desc[pairs[2 * g.pairs[k].pair]], nr = n_desc[pairs[2 * g.pairs[k].pair + 1]];
                cover[k].assign((size_t)match_tiles(nl) * match_tiles(nr), 0);
                chunks[k].resize((size_t)match_tiles(nl));
            }
            int last = 1 << 30;
            for (const MatchItem& it : g.items) {
                ++items_checked;
                if (it.b_tiles > last) FAIL("items not sorted largest first");
                last = it.b_tiles;
                if (it.pair < 0 || it.pair >= (int)g.pairs.size()) FAIL("item pair");
                const MatchGroupPair& gp = g.pairs[it.pair];
                const int l = pairs[2 * gp.pair], r = pairs[2 * gp.pair + 1];
                const int nl = n_desc[l], nr = n_desc[r];
                const int lt = it.l_row0 / kMatchTile, rt0 = it.b_col0 / kMatchTile;
                if (it.l_row0 % kMatchTile || it.b_col0 % kMatchTile || it.b_tiles < 1) FAIL("item alignment");
                if (it.nl != nl || it.stride != gp.chunks) FAIL("item nl / stride");
                if (set_row[l] < 0 || set_row[r] < 0) FAIL("item set not in group");
                if (it.a_row != set_row[l] + it.l_row0 || it.b_row != set_row[r] + it.b_col0) FAIL("item pooled rows");
                if (lt >= match_tiles(nl) || rt0 + it.b_tiles > match_tiles(nr)) FAIL("item out of range");
                const int64_t c = it.cand - gp.cand - (int64_t)it.l_row0 * gp.chunks;
                if (c < 0 || c >= gp.chunks) FAIL("item candidate slot");
                for (int t = rt0; t < rt0 + it.b_tiles; ++t) ++cover[it.pair][(size_t)lt * match_tiles(nr) + t];
                chunks[it.pair][lt].push_back({(int)c, rt0});
            }
            for (size_t k = 0; k < g.pairs.size(); ++k) {
                for (int v : cover[k]) if (v != 1) FAIL("pair %d: a (left tile, right tile) covered %d times", g.pairs[k].pair, v);
                const int nr = n_desc[pairs[2 * g.pairs[k].pair + 1]];
                for (auto& ch : chunks[k]) {
                    if (nr == 0) { if (!ch.empty()) FAIL("items for an empty right set"); continue; }
                    if ((int)ch.size() != g.pairs[k].chunks) FAIL("row has %zu chunks, want %d", ch.size(), g.pairs[k].chunks);
                    std::vector<int> start(ch.size(), -1);
                    for (auto& e : ch) start[e.first] = e.second;
                    if (start[0] != 0) FAIL("first chunk does not start at tile 0");
                    for (size_t c = 1; c < start.size(); ++c) if (start[c] <= start[c - 1]) FAIL("chunks not in order");
                }
            }
        }
        for (int p = 0; p < n_pairs; ++p) {
            const int want = n_desc[pairs[2 * p]] > 0 ? 1 : 0;
            if (seen[p] != want) FAIL("pair %d in %d groups", p, seen[p]);
        }
    }
    if (split_groups == 0 || multi_group_plans == 0) { std::printf("FAIL the sweep never split a right set or never made two groups\n"); return 1; }
    std::printf("OK u8 groups=%ld split_groups=%ld multi_group_plans=%ld items=%ld\n", groups_seen, split_groups, multi_group_plans, items_checked);
    return 0;
}
