#!/usr/bin/env python
"""Times feature tracks on the GPU (ps_tracks_from_matches / ps_tracks_from_edges):

  verify     the verify_bench.py workload: 16 seeded affine views of one 1920x1080 frame, all 240 ordered pairs matched,
             gathered and verified with a homography (1 024 samples); ps_tracks_from_matches on the inliers, against
             ps_verify_batch's time in the same run;
  sfm        a seeded synthetic SfM-scale graph: 2 000 sets x 3 000 features, 40 000 pairs x 400 edges, with planted forks;
  path       the same node count as one path with its edges in random order.

Reports the median ms per call after a warm-up (host clock around calls that end in a device synchronise), edges/s, and
the achieved bytes/s over the algorithmic byte count below; as context, scipy's connected_components on the same graph
(single-threaded host work, components only).  Also the geometry of the verify workload's tracks: the share whose
members all lie within 3 t of their mean in the first view (through the views' known maps).  Card name and power limit
are read in the same run.

    python tools/tracks_bench.py [--reps N] [out.json]

Algorithmic bytes (int32 ids, N nodes, E edges, A active nodes, P radix passes): the edges read once (8 E, plus 12 E for
the chain's src / match / reverse-map reads and 1 E of mask), parent written and read by init / compress / size / flags /
gather (5 x 4 N), the gids moved by every radix pass (2 x 4 A read and written, plus 4 A key gathers, per pass), the
classify / heads / start / members passes (about 6 x 4 A), the outputs (4 N track_of + 4 M members)."""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from popsift_b200 import api  # noqa: E402
from verify_bench import card, median_ms, views  # noqa: E402


def algo_bytes(N, E, A, M, per_edge=8):
    passes = max(1, (int(N - 1).bit_length() + 7) // 8)
    return per_edge * E + 20 * N + passes * 12 * A + 24 * A + 4 * N + 4 * M


def edges_case(lib, name, n_feat, e, reps):
    n_feat = np.ascontiguousarray(n_feat, np.int32)
    N = int(n_feat.sum())
    e = np.ascontiguousarray(e, np.int32)
    bufs = api._DevBuffers(lib)
    try:
        d_e = bufs.upload(e)
        d_of, d_st, d_mem = bufs.alloc(N * 4), bufs.alloc((N // 2 + 1) * 4), bufs.alloc(N * 4)
        cnt = api.PsTrackCounts()

        def run():
            assert lib.ps_tracks_from_edges(0, len(n_feat), n_feat.ctypes.data, len(e), d_e, 2, d_of, d_st, d_mem, C.byref(cnt)) == 0
        ms, all_ms = median_ms(run, reps)
        of = bufs.download(d_of, N, np.int32)
    finally:
        bufs.free()
    A = int((of >= 0).sum())    # kept members (a lower bound of the active nodes)
    r = {"nodes": N, "edges": len(e), "ms": ms, "ms_all": all_ms, "tracks": cnt.n_tracks, "members": cnt.n_members,
         "conflicting": cnt.n_conflicting, "short": cnt.n_short, "edges_per_s": len(e) / (ms * 1e-3)}
    r["algo_bytes"] = algo_bytes(N, len(e), max(A, cnt.n_members), cnt.n_members)
    r["achieved_GBps"] = r["algo_bytes"] / (ms * 1e-3) / 1e9
    try:
        from scipy.sparse import coo_matrix
        from scipy.sparse.csgraph import connected_components
        t0 = time.perf_counter()
        g = coo_matrix((np.ones(len(e), np.int8), (e[:, 0], e[:, 1])), shape=(N, N))
        connected_components(g, directed=True, connection="weak")
        r["scipy_components_ms_single_thread_host"] = (time.perf_counter() - t0) * 1e3
    except ImportError:
        r["scipy_components_ms_single_thread_host"] = None
    return r


def sfm_graph(seed=11, n_sets=2000, n_feat=3000, n_pairs=40000, per_pair=400, fork_share=0.02):
    rng = np.random.default_rng(seed)
    l = rng.integers(0, n_sets, n_pairs)
    r = (l + rng.integers(1, n_sets, n_pairs)) % n_sets
    fl = rng.integers(0, n_feat, (n_pairs, per_pair))
    fr = rng.integers(0, n_feat, (n_pairs, per_pair))
    u = l[:, None] * n_feat + fl
    v = r[:, None] * n_feat + fr
    fork = rng.random((n_pairs, per_pair)) < fork_share
    v = np.where(fork, l[:, None] * n_feat + (fl + 1) % n_feat, v)      # planted forks: an edge inside the left set
    return [n_feat] * n_sets, np.stack([u.ravel(), v.ravel()], 1)


def verify_case(lib, reps):
    w, h = 1920, 1080
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    sets = [ps.enqueue(w, h, im).getDev() for im in views()]
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    prm = api._verify_params("homography", 4.0, 1024, 0, True)
    bufs = api._DevBuffers(lib)
    r = {}
    try:
        ch = api._verify_chain(lib, bufs, sets, pairs, None, 0, False, None, False, prm)
        d_corr = api._correspondences_dev(lib, bufs, sets, pairs, ch.d_match, ch.device)[0]
        d_models, d_n = bufs.alloc(len(pairs) * 36), bufs.alloc(len(pairs) * 4)
        c_start, c_corr = np.ascontiguousarray(ch.start, np.int32), np.ascontiguousarray(ch.n_corr, np.int32)

        def verify():
            assert lib.ps_verify_batch(0, len(pairs), d_corr, c_start.ctypes.data, c_corr.ctypes.data, C.byref(prm), d_models, d_n,
                                       ch.d_mask, None) == 0
        r["verify_ms"], r["verify_ms_all"] = median_ms(verify, reps)
        n = len(sets)
        n_feat = [s.getFeatureCount() for s in sets]
        N = sum(n_feat)
        c_nf = (C.c_int32 * n)(*n_feat)
        c_rev = (C.c_void_p * n)(*[s.getReverseMap() for s in sets])
        c_nd = (C.c_int32 * n)(*[s.getDescriptorCount() for s in sets])
        d_of, d_st, d_mem = bufs.alloc(N * 4), bufs.alloc((N // 2 + 1) * 4), bufs.alloc(N * 4)
        cnt = api.PsTrackCounts()
        c_pairs = api._c_pairs(pairs)

        def tracks():
            assert lib.ps_tracks_from_matches(0, n, c_nf, c_rev, c_nd, len(pairs), c_pairs, ch.d_match, ch.d_src, c_corr.ctypes.data,
                                              ch.d_mask, 2, d_of, d_st, d_mem, C.byref(cnt)) == 0
        r["tracks_ms"], r["tracks_ms_all"] = median_ms(tracks, reps)
        E = int(ch.mask.sum())
        r.update(frames=n, pairs=len(pairs), features=N, correspondences=int(c_corr.sum()), inlier_edges=E,
                 tracks=cnt.n_tracks, members=cnt.n_members, conflicting=cnt.n_conflicting,
                 tracks_over_verify=r["tracks_ms"] / r["verify_ms"], edges_per_s=E / (r["tracks_ms"] * 1e-3))
        r["algo_bytes"] = algo_bytes(N, int(c_corr.sum()), cnt.n_members, cnt.n_members, per_edge=21)
        r["achieved_GBps"] = r["algo_bytes"] / (r["tracks_ms"] * 1e-3) / 1e9
        t = api.tracks(sets, pairs, model="homography", threshold=4.0)
        r["track_lengths"] = np.bincount(np.diff(t.start)).tolist()
    finally:
        bufs.free()
    ps.uninit()
    return r


def geometry_case():
    """the share of affine_set tracks within 3 t of their mean in image 1 (the floor test_tracks.py asserts)"""
    from popsift_b200.synth import affine_set
    vs = affine_set()
    h, w = vs[0][0].shape
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    sets = [ps.enqueue(w, h, im).getDev() for im, _ in vs]
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    t = api.tracks(sets, pairs, model="homography", threshold=4.0)
    feats = [s.to_host()[0] for s in sets]
    inv = [np.linalg.inv(np.vstack([A, [0, 0, 1]])) for _, A in vs]
    lens = np.diff(t.start)
    spread = []
    for k in range(len(lens)):
        a, b = t.start[k], t.start[k + 1]
        pts = np.array([(inv[s] @ [feats[s]["x"][f], feats[s]["y"][f], 1.0])[:2] for s, f in zip(t.set[a:b], t.feature[a:b])])
        spread.append(np.linalg.norm(pts - pts.mean(0), axis=1).max())
    spread = np.array(spread)
    ps.uninit()
    return {"tracks": len(lens), "share_within_12px": float((spread < 12.0).mean()), "len_ge3": int((lens >= 3).sum()),
            "len6": int((lens == 6).sum()), "lengths": np.bincount(lens).tolist(), "conflicting": t.n_conflicting}


def main():
    args = sys.argv[1:]
    reps = 10
    if "--reps" in args:
        i = args.index("--reps")
        reps = int(args[i + 1])
        del args[i:i + 2]
    out_path = args[0] if args else None
    lib = api.load_library()
    info = {"card": card()}
    info["geometry"] = geometry_case()
    info["verify"] = verify_case(lib, reps)
    n_feat, e = sfm_graph()
    info["sfm"] = edges_case(lib, "sfm", n_feat, e, reps)
    N = int(np.sum(n_feat))
    p = np.random.default_rng(12).permutation(N - 1)
    info["path"] = edges_case(lib, "path", np.ones(N, np.int32), np.stack([p, p + 1], 1), reps)
    info["card_after"] = card()
    line = json.dumps(info)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
