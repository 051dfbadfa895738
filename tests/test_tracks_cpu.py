"""Feature tracks without a GPU: the oracle against a brute-force breadth-first search on small random graphs, the new
header's exports and the counts struct's layout."""
import ctypes as C
import os
import re
from collections import deque

import numpy as np
import pytest

import tracks_oracle as to
from popsift_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def brute(n_feat, edges, min_length):
    """the contract by breadth-first search, one component at a time, in increasing order of the smallest unvisited id"""
    off = to.offsets(n_feat)
    N = int(off[-1])
    adj = [[] for _ in range(N)]
    for u, v in edges:
        if u != v:
            adj[u].append(v)
            adj[v].append(u)
    seen = [False] * N
    tracks, comps, conf, short = [], 0, 0, 0
    for s in range(N):
        if seen[s] or not adj[s]:
            continue
        comp, q = [], deque([s])
        seen[s] = True
        while q:
            x = q.popleft()
            comp.append(x)
            for y in adj[x]:
                if not seen[y]:
                    seen[y] = True
                    q.append(y)
        comps += 1
        comp.sort()
        sets = [int(np.searchsorted(off, g, side="right") - 1) for g in comp]
        if len(set(sets)) < len(sets):
            conf += 1
        elif len(comp) < min_length:
            short += 1
        else:
            tracks.append(comp)
    track_of = np.full(N, -1, np.int32)
    for t, m in enumerate(tracks):
        track_of[m] = t
    start = np.concatenate([[0], np.cumsum([len(m) for m in tracks])]).astype(np.int32)
    members = np.array([g for m in tracks for g in m], np.int32)
    return track_of, start, members, dict(n_tracks=len(tracks), n_members=int(start[-1]), n_components=comps,
                                          n_conflicting=conf, n_short=short)


def random_graph(rng):
    n_sets = int(rng.integers(1, 7))
    n_feat = rng.integers(0, 9, n_sets)
    n_feat[rng.random(n_sets) < 0.2] = 0
    N = int(n_feat.sum())
    if N == 0:
        return n_feat.tolist(), np.zeros((0, 2), np.int64)
    E = int(rng.integers(0, 2 * N + 1))
    e = rng.integers(0, N, size=(E, 2))
    if E:
        # self-loops, reversed and repeated edges
        loops = rng.random(E) < 0.1
        e[loops, 1] = e[loops, 0]
        e = np.concatenate([e, e[: E // 4, ::-1], e[: E // 5]])
    return n_feat.tolist(), e


@pytest.mark.parametrize("min_length", [2, 3, 4, 5])
def test_oracle_equals_bfs(min_length):
    rng = np.random.default_rng(min_length)
    for _ in range(80):
        n_feat, e = random_graph(rng)
        got, want = to.tracks(n_feat, e, min_length), brute(n_feat, e, min_length)
        for a, b in zip(got[:3], want[:3]):
            assert np.array_equal(a, b)
        assert got[3] == want[3]


def test_oracle_planted():
    # sets of 3 features; a track across all four sets, a fork (two features of set 1), a short pair and a self-loop
    n_feat = [3, 3, 3, 3]
    e = [(0, 3), (3, 6), (6, 9), (1, 4), (4, 5), (2, 7), (11, 11)]
    track_of, start, members, c = to.tracks(n_feat, e, 3)
    assert members.tolist() == [0, 3, 6, 9] and start.tolist() == [0, 4]
    assert c == dict(n_tracks=1, n_members=4, n_components=3, n_conflicting=1, n_short=1)
    assert track_of.tolist() == [0, -1, -1, 0, -1, -1, 0, -1, -1, 0, -1, -1]
    # a single set: any edge between two features is a fork
    assert to.tracks([5], [(0, 1)], 2)[3]["n_conflicting"] == 1


def test_chain_edges_rule():
    # pair (0, 1) with 3 left rows of which 2 correspond, the second masked out; pair (1, 1) with one row
    match = np.array([[1, 0, 1], [0, 1, 1], [1, 0, 1], [1, 0, 1], [0, 1, 1]], np.int32)
    src = np.array([0, 2, 0, 1, 0], np.int32)
    rev = [np.array([0, 0, 1]), np.array([1, 0])]
    e = to.chain_edges([(0, 1), (1, 1)], [3, 2], [2, 2], match, src, [2, 1], np.array([1, 0, 0, 1, 0]), rev)
    assert e.tolist() == [[0, 2 + 0], [2 + 0, 2 + 1]]
    e = to.chain_edges([(0, 1)], [3, 2], [2, 2], match, src, [2], None, rev)
    assert e.tolist() == [[0, 2], [1, 2]]


def test_header_exports():
    """every ps_*( of popsift_b200_tracks.h is exported and listed in api.TRACKS_EXPORTS, apart from the other lists"""
    hdr = open(os.path.join(ROOT, "include", "popsift_b200_tracks.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    decl = sorted(set(re.findall(r"\b(ps_\w+)\(", hdr)))
    assert decl == sorted(api.TRACKS_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS):
        assert not set(api.TRACKS_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.TRACKS_EXPORTS:
        assert hasattr(lib, name)


def test_counts_layout():
    assert C.sizeof(api.PsTrackCounts) == 20
    assert [f[0] for f in api.PsTrackCounts._fields_] == ["n_tracks", "n_members", "n_components", "n_conflicting", "n_short"]
