"""The shapes at which ps_bundle_adjust, ps_global_positioning and ps_rotation_averaging change how they split their work,
one scene per row, for tests/test_bundle_global_scale.py (on the GPU) and tests/test_bundle_cpu.py (which checks that every
row still sits on the boundary it names, with the constants read from the kernel sources).

The constants (k_bundle.cu, k_global.cu, k_scan.h):
- kCamT / kNodeT threads stride over one set's observations or one camera node's edges;
- kCgT / kRedT threads of the single-CTA loops stride over the sets, the nodes or the partials;
- kT threads per per-track / per-member / per-pair CTA, one partial each;
- the exclusive scan goes to more than one block past kScanChunk entries; the radix sort runs one pass per 8 bits of the
  largest key, over tiles of kRadixTile entries, and scans 256 histogram entries per tile.

Each row gives its scene and the quantities it claims; QUANTITIES says how each follows from the scene and the constants."""
from __future__ import annotations

import numpy as np

import bundle_oracle as bo
import global_oracle as go
import triangulate_oracle as tro


def blocks(n, per):
    return -(-int(n) // int(per))


def passes(max_key):
    """8-bit radix passes over keys 0 .. max_key"""
    return blocks(int(max_key).bit_length(), 8)


# ---- scenes ----------------------------------------------------------------------------------------------------------

def bundle_scene(seed, n_sets, lengths=None, sets=None, empty=(), fixed=(0,), noise=0.5):
    """bo.planted with the cameras of every track given (or drawn), then `empty` sets without features inserted (their
    indices in the result).  Returns the scene with 'fixed' (uint8) added."""
    rng = np.random.default_rng(seed)
    n = n_sets - len(empty)
    if sets is None:
        sets = [rng.choice(n, size=int(L), replace=False) for L in lengths]
    sc = bo.planted(rng, n, [len(s) for s in sets], noise=noise, sets=sets)
    keep = [i for i in range(n_sets) if i not in set(empty)]
    feats, cams, poses, truth = [np.zeros((0, 2), np.float32)] * n_sets, np.zeros((n_sets, 4), np.float32), [None] * n_sets, [None] * n_sets
    for k, i in enumerate(keep):
        feats[i], cams[i], poses[i], truth[i] = sc["feats"][k], sc["cams"][k], sc["poses"][k], sc["poses_true"][k]
    for i in empty:
        cams[i], poses[i], truth[i] = sc["cams"][0], sc["poses"][0], sc["poses_true"][0]
    # members index the concatenated features, so the empty sets change nothing there
    sc.update(feats=feats, cams=cams, poses=poses, poses_true=truth)
    f = np.zeros(n_sets, np.uint8)
    f[list(fixed)] = 1
    sc["fixed"] = f
    sc["R"] = np.stack([np.asarray(R) for R, _ in truth])
    return sc


def counts_sets(rng, counts, n_other):
    """track camera lists giving set i (i < len(counts)) exactly counts[i] observations: each track has one such set and
    one or two of the n_other sets after them"""
    out = []
    for i, c in enumerate(counts):
        for _ in range(c):
            k = int(rng.integers(1, 3))
            out.append(np.r_[i, len(counts) + rng.choice(n_other, size=k, replace=False)])
    return out


def lengths_summing(rng, total, lo=2, hi=4):
    L = []
    while total - sum(L) > hi + lo:
        L.append(int(rng.integers(lo, hi + 1)))
    rest = total - sum(L)
    L += [rest] if rest <= hi else [lo, rest - lo]
    return L


def _rng_lengths(seed, T, lo=2, hi=4):
    return list(np.random.default_rng(1000 + seed).integers(lo, hi + 1, size=T))


COUNTS = (127, 128, 129, 256, 257)
FIXED_COUNT = 200


def _counts_scene():
    """sets 0 .. 4 with 127, 128, 129, 256 and 257 observations, set 5 fixed with 200; empty sets at 8 and at the end"""
    rng = np.random.default_rng(31)
    sets = counts_sets(rng, COUNTS + (FIXED_COUNT,), 14)
    return bundle_scene(31, 22, sets=sets, empty=(8, 21), fixed=(5,))


def _members_scene(M):
    rng = np.random.default_rng(40 + M)
    return bundle_scene(40 + M, 30, lengths=lengths_summing(rng, M))


SCENES = {
    "sets_256": lambda: bundle_scene(11, 256, lengths=_rng_lengths(11, 700)),
    "sets_257": lambda: bundle_scene(12, 257, lengths=_rng_lengths(12, 700)),
    "sets_255": lambda: bundle_scene(13, 255, lengths=_rng_lengths(13, 700)),
    "counts": _counts_scene,
    "tracks_256": lambda: bundle_scene(14, 20, lengths=_rng_lengths(14, 256)),
    "tracks_257": lambda: bundle_scene(15, 20, lengths=_rng_lengths(15, 257)),
    "members_4095": lambda: _members_scene(4095),
    "members_4096": lambda: _members_scene(4096),
    "members_4097": lambda: _members_scene(4097),
    "large": lambda: bundle_scene(16, 300, lengths=_rng_lengths(16, 66000)),
}


def graph(seed, n, p, hub=None):
    return go.view_graph(np.random.default_rng(seed), n, p, noise_deg=0.5, outliers=0.1, hub=hub)


GRAPHS = {
    "pairs_256": lambda: graph(21, 40, 256),
    "pairs_257": lambda: graph(22, 40, 257),
    "sets_257_hub": lambda: graph(23, 257, 700, hub=(5, 200)),
    "large": lambda: graph(24, 600, 66000),
}


# ---- what each scene's numbers are -----------------------------------------------------------------------------------

def bundle_stats(sc):
    """the numbers the bundle kernels split on (every member used: all tracks OK, mask all 1)"""
    S, T, M = len(sc["feats"]), len(sc["start"]) - 1, len(sc["members"])
    off = np.cumsum([0] + [len(f) for f in sc["feats"]])
    cnt = np.bincount(np.searchsorted(off, sc["members"], side="right") - 1, minlength=S)
    return dict(S=S, T=T, M=M, U=M, counts=cnt)


def graph_stats(g):
    _, pairs, _, _, _ = g
    pairs = np.asarray(pairs)
    S = int(pairs.max()) + 1
    return dict(S=S, P=len(pairs), degree=np.bincount(pairs.reshape(-1), minlength=S))


def quantities(kind, st, k):
    """kind 'bundle', 'position' or 'rotation'; st from bundle_stats / graph_stats; k the constants"""
    if kind == "bundle":
        nb = blocks(st["U"], k["kRadixTile"])
        return dict(radix_passes=passes(st["S"] - 1), set_trips=blocks(st["S"], k["kCgT"]),
                    cam_trips=[blocks(c, k["kCamT"]) for c in st["counts"]], track_partials=blocks(st["T"], k["kT"]),
                    reduce_trips=blocks(blocks(st["T"], k["kT"]), k["kCgT"]), member_scan_blocks=blocks(st["M"] + 1, k["kScanChunk"]),
                    radix_tiles=nb, hist_scan_blocks=blocks(256 * nb, k["kScanChunk"]))
    if kind == "position":
        nbP = blocks(st["T"], k["kT"])
        nb = blocks(st["M"], k["kRadixTile"])
        return dict(radix_passes=passes(st["S"]), node_trips=[blocks(c, k["kNodeT"]) for c in st["counts"]],
                    sum_parts_trips=blocks(nbP + st["S"], k["kRedT"]), nbN=blocks(st["S"] + st["T"], k["kT"]),
                    cost_trips=blocks(blocks(st["M"], k["kT"]), k["kRedT"]), radix_tiles=nb, hist_scan_blocks=blocks(256 * nb, k["kScanChunk"]))
    return dict(set_trips=blocks(st["S"], k["kRedT"]), pair_partials=blocks(st["P"], k["kT"]),
                cost_trips=blocks(blocks(st["P"], k["kT"]), k["kRedT"]), hub_trips=blocks(int(st["degree"].max()), k["kNodeT"]))


# ---- the rows: (kind, scene, doc, claims).  A claim on cam_trips / node_trips is checked on sets 0 .. len - 1. ---------

ROWS = {
    "ba_sets_256": ("bundle", "sets_256", "S = 256: one radix pass (keys 0 .. 255), one trip of the 256-thread set loops",
                    dict(radix_passes=1, set_trips=1)),
    "ba_sets_257": ("bundle", "sets_257", "S = 257: two radix passes, two trips of the set loops",
                    dict(radix_passes=2, set_trips=2)),
    "ba_counts": ("bundle", "counts", "set observation counts 127 / 128 / 129 / 256 / 257 and a fixed set of 200 over the "
                  "128-thread per-set CTAs; empty sets in the middle and at the end", dict(cam_trips=[1, 1, 2, 2, 3, 2])),
    "ba_tracks_256": ("bundle", "tracks_256", "T = 256: one per-track partial", dict(track_partials=1)),
    "ba_tracks_257": ("bundle", "tracks_257", "T = 257: two per-track partials", dict(track_partials=2)),
    "ba_members_4095": ("bundle", "members_4095", "M = 4095: the member scan of M + 1 = 4096 entries in one block",
                        dict(member_scan_blocks=1, radix_tiles=1)),
    "ba_members_4096": ("bundle", "members_4096", "M = 4096: the member scan in two blocks, one radix tile",
                        dict(member_scan_blocks=2, radix_tiles=1)),
    "ba_members_4097": ("bundle", "members_4097", "M = U = 4097: two radix tiles", dict(member_scan_blocks=2, radix_tiles=2)),
    "ba_large": ("bundle", "large", "S = 300, T = 66 000 (lengths 2-4): more than 256 cost partials in the reduce, a "
                 "multi-block histogram scan", dict(radix_passes=2, set_trips=2, reduce_trips=2, hist_scan_blocks=4)),
    "gp_sets_255": ("position", "sets_255", "S = 255: keys 0 .. 255, one radix pass", dict(radix_passes=1)),
    "gp_sets_256": ("position", "sets_256", "S = 256: keys 0 .. 256, two radix passes", dict(radix_passes=2)),
    "gp_counts": ("position", "counts", "camera-node edge counts 127 / 128 / 129 / 256 / 257 / 200 over the 128-thread CTAs",
                  dict(node_trips=[1, 1, 2, 2, 3, 2])),
    "gp_members_4096": ("position", "members_4096", "M = 4096: one radix tile", dict(radix_tiles=1)),
    "gp_members_4097": ("position", "members_4097", "M = 4097: two radix tiles", dict(radix_tiles=2)),
    "gp_large": ("position", "large", "S = 300, T = 66 000: nbP + nC and nbN above 256, more than 256 cost partials, a "
                 "multi-block histogram scan", dict(radix_passes=2, sum_parts_trips=3, cost_trips=4, hist_scan_blocks=4)),
    "ra_pairs_256": ("rotation", "pairs_256", "P = 256: one per-pair partial", dict(pair_partials=1, set_trips=1)),
    "ra_pairs_257": ("rotation", "pairs_257", "P = 257: two per-pair partials", dict(pair_partials=2)),
    "ra_sets_257_hub": ("rotation", "sets_257_hub", "S = 257 (two trips of the node loops) and a node of degree 200 (two "
                        "trips of its 128-thread CTA)", dict(set_trips=2, hub_trips=2)),
    "ra_large": ("rotation", "large", "S = 600, P = 66 000 > 65 536: more than 256 cost partials",
                 dict(set_trips=3, cost_trips=2)),
}


def stats(row, scene):
    kind = ROWS[row][0]
    return graph_stats(scene) if kind == "rotation" else bundle_stats(scene)
