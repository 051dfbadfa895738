// Work plan of the batched matcher (host only, no CUDA): which pairs share one set of launches, where each set's
// split planes sit in the pooled hi / lo planes, and the (pair, 128-row left tile, contiguous chunk of right tiles)
// work items of match_tc_kernel.  Checked on the host by tests/cpp/match_plan_check.cpp.
//
//   * Groups.  Pairs are taken in order and a pair joins the current group while the split planes of the group's
//     distinct sets plus its candidate buffer stay within `cap` bytes; a set used by several groups is split again
//     in each.  A pair larger than the cap on its own forms a group of one.  Pairs with an empty left set have no rows
//     and no work; pairs with an empty right set have rows (the re-rank writes (0, 0, 0)) but no sets and no items.
//   * Chunks.  Every pair of a group cuts its right set into the same number S of chunks (fewer when the right set
//     has fewer tiles).  S = 1 whenever the group's left tiles alone fill the SMs; otherwise S (<= kMatchMaxChunks) is
//     the one with the shortest modelled makespan, ties to the smaller S, and only as large as the cap allows.
//   * Order.  Items are sorted by size, largest first (stable), and CTA b of the persistent grid runs items b, b + G,
//     b + 2G, ...; the makespan model is exactly that assignment.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace psb {

constexpr int kMatchTile = 128;                 // rows of a left tile and of a right tile
constexpr int kMatchMaxChunks = 8;              // bound of S
constexpr int kMatchCand = 4;                   // candidates one item keeps per left row
constexpr size_t kMatchRowBytes = 2 * 512 + 4;  // pooled hi + lo row and its norm (float32 descriptors)
constexpr size_t kMatchU8RowBytes = 128 + 4;    // pooled 8-bit row and its norm key (k_match_u8.cu)
// guided matching adds the row's pixel position (float2) to either
constexpr size_t kMatchGuidedRowBytes = kMatchRowBytes + 8;
constexpr size_t kMatchU8GuidedRowBytes = kMatchU8RowBytes + 8;
// freed workspace the library's memory pool (workspace.cu) keeps mapped, and the default cap of one group's workspace
// (POPSIFT_B200_MATCH_WS=bytes overrides the cap)
constexpr size_t kMatchPoolKeep = (size_t)1 << 30;

// One unit of work of match_tc_kernel.  Candidate slot of left row l_row0 + i: cand + i * stride (units of kMatchCand ints).
struct MatchItem {
    int64_t cand;
    int32_t a_row;     // first pooled row of the left tile
    int32_t b_row;     // first pooled row of the chunk (rows of the hi / lo planes and of the norms)
    int32_t b_tiles;   // right tiles in the chunk (>= 1)
    int32_t b_col0;    // index within the right set of the chunk's first row
    int32_t l_row0;    // index within the left set of the tile's first row
    int32_t nl;        // rows of the left set
    int32_t stride;    // the pair's chunk count
    int32_t pair;      // index into MatchGroup::pairs
};

struct MatchGroupPair {
    int     pair;      // index into the caller's pair list
    int     chunks;    // S of this pair (0 when its right set is empty)
    int64_t cand;      // first candidate slot of the pair (its row i, chunk c: cand + i * chunks + c)
    int64_t row;       // first row of the pair among the group's left rows
};

struct MatchGroupSet {
    int     set;       // index into the caller's set list
    int64_t row;       // first pooled row (the set's rows padded to a multiple of kMatchTile follow)
};

struct MatchGroup {
    std::vector<MatchGroupSet>  sets;
    std::vector<MatchGroupPair> pairs;
    std::vector<MatchItem>      items;
    int64_t rows = 0;          // pooled rows
    int64_t cand_slots = 0;
    int64_t left_rows = 0;     // rows the re-rank writes
    int     chunks = 1;        // S of the group
    size_t  row_bytes = kMatchRowBytes;   // workspace bytes of one pooled row
    size_t  bytes() const { return (size_t)rows * row_bytes + (size_t)cand_slots * kMatchCand * 4; }
};

struct MatchPlan {
    std::vector<int64_t>    out_row;   // per pair: first output row (prefix sum of the left sizes)
    std::vector<MatchGroup> groups;
};

inline int64_t match_tiles(int64_t n) { return (n + kMatchTile - 1) / kMatchTile; }

namespace plan_detail {

// items of a group for S chunks per pair; fills cand / chunks of the group's pairs
inline void make_items(MatchGroup& g, const int32_t* n_desc, const int32_t* pairs, int S)
{
    g.items.clear();
    g.cand_slots = 0;
    g.chunks = S;
    int64_t set_row_l = 0, set_row_r = 0;
    for (size_t k = 0; k < g.pairs.size(); ++k) {
        MatchGroupPair& gp = g.pairs[k];
        const int l = pairs[2 * gp.pair], r = pairs[2 * gp.pair + 1];
        const int nl = n_desc[l], nr = n_desc[r];
        gp.cand = g.cand_slots;
        gp.chunks = 0;
        if (nr <= 0) continue;
        for (const MatchGroupSet& s : g.sets) {
            if (s.set == l) set_row_l = s.row;
            if (s.set == r) set_row_r = s.row;
        }
        const int nt = (int)match_tiles(nr), lt = (int)match_tiles(nl);
        const int sp = std::min(S, nt);
        gp.chunks = sp;
        for (int t = 0; t < lt; ++t) {
            int c0 = 0;
            for (int c = 0; c < sp; ++c) {
                const int len = nt / sp + (c < nt % sp ? 1 : 0);
                MatchItem it;
                it.cand = gp.cand + (int64_t)t * kMatchTile * sp + c;
                it.a_row = (int32_t)(set_row_l + (int64_t)t * kMatchTile);
                it.b_row = (int32_t)(set_row_r + (int64_t)c0 * kMatchTile);
                it.b_tiles = len;
                it.b_col0 = c0 * kMatchTile;
                it.l_row0 = t * kMatchTile;
                it.nl = nl;
                it.stride = sp;
                it.pair = (int32_t)k;
                g.items.push_back(it);
                c0 += len;
            }
        }
        g.cand_slots += (int64_t)nl * sp;
    }
    std::stable_sort(g.items.begin(), g.items.end(), [](const MatchItem& a, const MatchItem& b) { return a.b_tiles > b.b_tiles; });
}

// Modelled run time of the group's items for S chunks per pair on `sms` persistent CTAs, in half tiles: a right tile
// costs 2, an item 1 more (A tile load, pipeline fill, candidate merge).  The items, largest first, go round-robin to
// the CTAs (CTA b runs items b, b + G, ...); computed from the runs of equal chunk lengths without building the items,
// since the planner runs on every call.
inline int64_t makespan(const MatchGroup& g, const int32_t* n_desc, const int32_t* pairs, int S, int sms)
{
    std::vector<std::pair<int64_t, int64_t>> runs;          // (chunk length in tiles, number of items)
    for (const MatchGroupPair& gp : g.pairs) {
        const int nr = n_desc[pairs[2 * gp.pair + 1]];
        if (nr <= 0) continue;
        const int64_t nt = match_tiles(nr), lt = match_tiles(n_desc[pairs[2 * gp.pair]]);
        const int64_t sp = std::min<int64_t>(S, nt), q = nt / sp, rem = nt % sp;
        if (rem) runs.push_back({q + 1, lt * rem});
        runs.push_back({q, lt * (sp - rem)});
    }
    std::sort(runs.begin(), runs.end(), [](const std::pair<int64_t, int64_t>& a, const std::pair<int64_t, int64_t>& b) { return a.first > b.first; });
    int64_t n_items = 0;
    for (const auto& r : runs) n_items += r.second;
    const int64_t G = std::min<int64_t>(sms, n_items);
    if (G <= 0) return 0;
    // every CTA gets `all`; diff[] adds the partial rounds (cyclic ranges of CTAs)
    std::vector<int64_t> diff((size_t)G + 1, 0);
    int64_t all = 0, pos = 0;
    for (const auto& r : runs) {
        const int64_t cost = 2 * r.first + 1, full = r.second / G, part = r.second % G;
        all += full * cost;
        const int64_t end = pos + part;
        if (end <= G) { diff[pos] += cost; diff[end] -= cost; }
        else { diff[pos] += cost; diff[G] -= cost; diff[0] += cost; diff[end - G] -= cost; }
        pos = (pos + r.second) % G;
    }
    int64_t worst = 0, run = 0;
    for (int64_t b = 0; b < G; ++b) { run += diff[b]; worst = std::max(worst, run); }
    return all + worst;
}

// candidate slots of the group for S chunks per pair
inline int64_t cand_slots(const MatchGroup& g, const int32_t* n_desc, const int32_t* pairs, int S)
{
    int64_t slots = 0;
    for (const MatchGroupPair& gp : g.pairs) {
        const int nr = n_desc[pairs[2 * gp.pair + 1]];
        if (nr > 0) slots += (int64_t)n_desc[pairs[2 * gp.pair]] * std::min<int64_t>(S, match_tiles(nr));
    }
    return slots;
}

} // namespace plan_detail

// n_desc: n_sets sizes; pairs: n_pairs x {left, right} (indices already validated); sms: persistent CTAs; cap: bytes;
// row_bytes: workspace bytes of one pooled row (kMatchRowBytes for float32 descriptors, kMatchU8RowBytes for 8-bit ones)
inline MatchPlan plan_match(int n_sets, const int32_t* n_desc, int n_pairs, const int32_t* pairs, int sms, size_t cap,
                            size_t row_bytes = kMatchRowBytes)
{
    MatchPlan plan;
    plan.out_row.resize((size_t)n_pairs);
    int64_t out = 0;
    for (int p = 0; p < n_pairs; ++p) { plan.out_row[p] = out; out += n_desc[pairs[2 * p]]; }
    sms = std::max(sms, 1);

    // groups, sized with one chunk per pair
    std::vector<int> member((size_t)std::max(n_sets, 0), -1);     // set -> group that holds it
    MatchGroup cur;
    cur.row_bytes = row_bytes;
    auto close = [&]() {
        if (!cur.pairs.empty()) plan.groups.push_back(std::move(cur));
        cur = MatchGroup();
        cur.row_bytes = row_bytes;
    };
    for (int p = 0; p < n_pairs; ++p) {
        const int l = pairs[2 * p], r = pairs[2 * p + 1];
        const int nl = n_desc[l], nr = n_desc[r];
        if (nl <= 0) continue;
        const int gi = (int)plan.groups.size();
        int64_t rows = cur.rows, slots = cur.cand_slots;
        if (nr > 0) {
            if (member[l] != gi) rows += match_tiles(nl) * kMatchTile;
            if (member[r] != gi && r != l) rows += match_tiles(nr) * kMatchTile;
            slots += nl;
        }
        if (!cur.pairs.empty() && (size_t)rows * row_bytes + (size_t)slots * kMatchCand * 4 > cap) {
            close();
            p -= 1;                                     // the pair opens the next group
            continue;
        }
        if (nr > 0) {
            for (int s : {l, r})
                if (member[s] != gi) {
                    member[s] = gi;
                    cur.sets.push_back({s, cur.rows});
                    cur.rows += match_tiles(n_desc[s]) * kMatchTile;
                }
            cur.cand_slots = slots;
        }
        cur.pairs.push_back({p, 0, 0, cur.left_rows});
        cur.left_rows += nl;
    }
    close();

    for (MatchGroup& g : plan.groups) {
        int64_t left_tiles = 0;
        for (const MatchGroupPair& gp : g.pairs)
            if (n_desc[pairs[2 * gp.pair + 1]] > 0) left_tiles += match_tiles(n_desc[pairs[2 * gp.pair]]);
        int best_s = 1;
        if (left_tiles > 0 && left_tiles < sms) {
            int64_t best_t = plan_detail::makespan(g, n_desc, pairs, 1, sms);
            for (int S = 2; S <= kMatchMaxChunks; ++S) {
                // more chunks only cost more candidate slots
                if (g.pairs.size() > 1 && (size_t)g.rows * row_bytes + (size_t)plan_detail::cand_slots(g, n_desc, pairs, S) * kMatchCand * 4 > cap) break;
                const int64_t t = plan_detail::makespan(g, n_desc, pairs, S, sms);
                if (t < best_t) { best_t = t; best_s = S; }
            }
        }
        plan_detail::make_items(g, n_desc, pairs, best_s);
    }
    return plan;
}

} // namespace psb
