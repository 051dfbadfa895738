"""Feature tracks on the GPU (ps_tracks_from_edges / ps_tracks_from_matches): the edge entry against the oracle byte for
byte on seeded graphs and union-find worst cases, invariance to edge order, direction and duplicates, argument errors with
the outputs untouched, the chain entry on real extractions against the edge entry and the oracle, the geometry of tracks
through known affine maps, and the C++ API."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import tracks_oracle as to
from popsift_b200 import api
from popsift_b200.synth import affine_set

pytestmark = pytest.mark.gpu
PS_ERR_ARG = -1
SENTINEL = 0x5A5A5A5A


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


def run_edges(lib, n_feat, edges, min_length=2, rc_only=False):
    """ps_tracks_from_edges on global-id edges: (rc, track_of, track_start, members, counts); outputs prefilled with a
    sentinel so that an untouched output can be recognised"""
    n_feat = np.ascontiguousarray(n_feat, np.int32)
    e = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
    N = int(n_feat.astype(np.int64).sum())
    cap = N // max(min_length, 2) + 1
    bufs = api._DevBuffers(lib)
    try:
        fill = np.full(max(N, cap), SENTINEL, np.int32)
        d_of, d_st, d_mem = bufs.upload(fill[:N]), bufs.upload(fill[:cap]), bufs.upload(fill[:N])
        cnt = api.PsTrackCounts()
        rc = lib.ps_tracks_from_edges(0, len(n_feat), n_feat.ctypes.data, len(e), bufs.upload(e), min_length, d_of, d_st, d_mem,
                                      C.byref(cnt))
        if rc_only:
            return rc, bufs.download(d_of, N, np.int32), bufs.download(d_st, cap, np.int32)
        assert rc == 0, api._last_error(lib)
        counts = dict(n_tracks=cnt.n_tracks, n_members=cnt.n_members, n_components=cnt.n_components,
                      n_conflicting=cnt.n_conflicting, n_short=cnt.n_short)
        return (bufs.download(d_of, N, np.int32), bufs.download(d_st, cnt.n_tracks + 1, np.int32),
                bufs.download(d_mem, cnt.n_members, np.int32), counts)
    finally:
        bufs.free()


def check(lib, n_feat, edges, min_length=2):
    got = run_edges(lib, n_feat, edges, min_length)
    want = to.tracks(n_feat, edges, min_length)
    for g, w in zip(got[:3], want[:3]):
        assert np.array_equal(g, w)
    assert got[3] == want[3]
    return got


def planted(rng, n_sets=40, n_feat=500, n_tracks=3000, fork_share=0.2):
    """tracks of 2 .. n_sets features in distinct sets joined by random spanning edges; a share of them gets a second
    feature of one of its sets (a fork)"""
    off = np.arange(n_sets + 1) * n_feat
    used = np.zeros(n_sets * n_feat, bool)
    edges = []
    for _ in range(n_tracks):
        L = int(rng.integers(2, n_sets + 1))
        sets = rng.choice(n_sets, L, replace=False)
        nodes = off[sets] + rng.integers(0, n_feat, L)
        if rng.random() < fork_share:
            nodes = np.r_[nodes, off[sets[0]] + rng.integers(0, n_feat)]
        nodes = nodes[~used[nodes]]
        used[nodes] = True
        for k in range(1, len(nodes)):
            edges.append((nodes[k], nodes[int(rng.integers(0, k))]))
    return [n_feat] * n_sets, np.array(edges, np.int64).reshape(-1, 2)


def case_graph(name):
    rng = np.random.default_rng(len(name))
    if name == "sparse":
        n_feat = rng.integers(0, 3000, 30)
        N = int(n_feat.sum())
        return n_feat, rng.integers(0, N, (N // 2, 2)), 2
    if name == "planted":
        n_feat, e = planted(rng)
        return n_feat, e, 3
    if name == "giant":
        n_feat = [1000] * 8
        p = rng.permutation(8000)
        return n_feat, np.stack([p[:-1], p[1:]], 1), 2
    if name == "empty_sets":
        n_feat = [0, 50, 0, 0, 70, 0, 30, 0]
        return n_feat, rng.integers(0, 150, (120, 2)), 2
    if name == "no_edges":
        return [10, 20], np.zeros((0, 2), np.int64), 2
    if name == "n3":
        return [1, 1, 1], np.array([[0, 1], [2, 1], [1, 1]]), 3
    if name == "big":
        N = (1 << 24) + 4099
        n_feat = [N // 4, N // 4, N // 4, N - 3 * (N // 4)]
        return n_feat, rng.integers(0, N, (1 << 21, 2)), 2
    raise KeyError(name)


@pytest.mark.parametrize("name", ["sparse", "planted", "giant", "empty_sets", "no_edges", "n3", "big"])
def test_edges_against_oracle(lib, name):
    n_feat, e, m = case_graph(name)
    got = check(lib, n_feat, e, m)
    if name == "planted":
        assert got[3]["n_conflicting"] > 100 and got[3]["n_tracks"] > 1000
    if name == "giant":
        assert got[3]["n_conflicting"] == 1 and got[3]["n_tracks"] == 0
    for mlen in (2, 4, 7):
        if name in ("planted", "empty_sets"):
            check(lib, n_feat, e, mlen)


@pytest.mark.parametrize("order", ["ascending", "descending", "random"])
def test_long_path(lib, order):
    """a path over 2^22 nodes, one feature per set: one track of all of them, whatever the edge order"""
    N = 1 << 22
    e = np.stack([np.arange(N - 1), np.arange(1, N)], 1)
    if order == "descending":
        e = e[::-1]
    elif order == "random":
        e = e[np.random.default_rng(3).permutation(N - 1)]
    of, st, mem, c = check(lib, np.ones(N, np.int32), e)
    assert c["n_tracks"] == 1 and st.tolist() == [0, N]
    # the same path over 64 sets: one conflicting component
    assert check(lib, [N // 64] * 64, e)[3]["n_conflicting"] == 1


@pytest.mark.parametrize("centre", ["smallest", "largest"])
def test_star(lib, centre):
    """2^20 leaves on one centre: every edge's CAS meets the same root"""
    n = (1 << 20) + 1
    c = 0 if centre == "smallest" else n - 1
    leaves = np.setdiff1d(np.arange(n), [c])
    e = np.stack([np.full(len(leaves), c), leaves], 1)
    e[::2] = e[::2, ::-1]
    e = e[np.random.default_rng(4).permutation(len(e))]
    assert check(lib, np.ones(n, np.int32), e)[3]["n_members"] == n


def test_disjoint_cliques(lib):
    """2 000 disjoint K_32 in shuffled node order over sets of 16 and of 1: forks and tracks"""
    rng = np.random.default_rng(5)
    k, s = 2000, 32
    perm = rng.permutation(k * s)
    iu = np.triu_indices(s, 1)
    e = np.concatenate([np.stack([perm[q * s + iu[0]], perm[q * s + iu[1]]], 1) for q in range(k)])
    e = e[rng.permutation(len(e))]
    check(lib, [16] * (k * s // 16), e)
    c = check(lib, np.ones(k * s, np.int32), e, 32)[3]
    assert c["n_tracks"] == k
    assert check(lib, np.ones(k * s, np.int32), e, 33)[3]["n_short"] == k


def test_invariance(lib):
    rng = np.random.default_rng(6)
    n_feat, e = planted(rng, n_tracks=2000)
    base = run_edges(lib, n_feat, e, 2)
    for variant in range(3):
        f = e[rng.permutation(len(e))]
        flip = rng.random(len(f)) < 0.5
        f[flip] = f[flip, ::-1]
        f = np.concatenate([f, f[rng.integers(0, len(f), len(f) // 3)]])
        f = f[rng.permutation(len(f))]
        got = run_edges(lib, n_feat, f, 2)
        for a, b in zip(got[:3], base[:3]):
            assert a.tobytes() == b.tobytes()
        assert got[3] == base[3]
    again = run_edges(lib, n_feat, e, 2)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(again[:3], base[:3]))


def test_errors(lib):
    n_feat = [5, 5]
    for bad in ([[0, 10]], [[-1, 3]], [[3, 2 ** 31 - 1]]):
        rc, of, st = run_edges(lib, n_feat, bad, 2, rc_only=True)
        assert rc == PS_ERR_ARG
        assert (of == SENTINEL).all() and (st == SENTINEL).all()
    # an endpoint out of range among good edges: still refused, outputs untouched
    rc, of, st = run_edges(lib, n_feat, [[0, 1], [1, 2], [9, 10]], 2, rc_only=True)
    assert rc == PS_ERR_ARG and (of == SENTINEL).all()
    for m in (1, 0, -3):
        assert run_edges(lib, n_feat, [[0, 1]], m, rc_only=True)[0] == PS_ERR_ARG
    assert run_edges(lib, [5, -1], [[0, 1]], 2, rc_only=True)[0] == PS_ERR_ARG
    cnt = api.PsTrackCounts()
    huge = np.array([2 ** 30, 2 ** 30], np.int32)
    assert lib.ps_tracks_from_edges(0, 2, huge.ctypes.data, 0, None, 2, None, None, None, C.byref(cnt)) == PS_ERR_ARG
    assert lib.ps_tracks_from_edges(0, -1, None, 0, None, 2, None, None, None, C.byref(cnt)) == PS_ERR_ARG
    assert lib.ps_tracks_from_edges(0, 2, np.array([5, 5], np.int32).ctypes.data, -1, None, 2, None, None, None, C.byref(cnt)) == PS_ERR_ARG
    # host memory where device memory is required
    host = np.zeros(16, np.int32)
    bufs = api._DevBuffers(lib)
    try:
        d = bufs.alloc(64)
        nf = np.array([5, 5], np.int32)
        assert lib.ps_tracks_from_edges(0, 2, nf.ctypes.data, 0, None, 2, host.ctypes.data, d, d, C.byref(cnt)) == PS_ERR_ARG
        assert lib.ps_tracks_from_edges(0, 2, nf.ctypes.data, 0, None, 2, d, host.ctypes.data, d, C.byref(cnt)) == PS_ERR_ARG
        assert lib.ps_tracks_from_edges(0, 2, nf.ctypes.data, 1, host.ctypes.data, 2, d, d, d, C.byref(cnt)) == PS_ERR_ARG
        assert lib.ps_tracks_from_edges(0, 2, nf.ctypes.data, 0, None, 2, d, d, d, None) == PS_ERR_ARG
        assert lib.ps_tracks_from_edges(0, 2, nf.ctypes.data, 0, None, 2, d, d, d, C.byref(cnt)) == 0 and cnt.n_tracks == 0
    finally:
        bufs.free()
    with pytest.raises(api.PopSiftError):
        api.build_tracks([3, 3], [[0, 3, 1, 0]])


# ---- the chain entry on real extractions

def _extract(norm_multi=None):
    views = affine_set()
    h, w = views[0][0].shape
    cfg = api.Config()
    if norm_multi is not None:
        cfg.setNormalizationMultiplier(norm_multi)
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    return ps, [ps.enqueue(w, h, im).getDev() for im, _ in views], [A for _, A in views]


@pytest.fixture(scope="module")
def affine_sets():
    """the 6 views of synth.affine_set under MatchingMode, with their maps A_k (image 1 -> image k)"""
    ps, sets, maps = _extract()
    yield sets, maps
    ps.uninit()


@pytest.fixture(scope="module")
def affine_sets_u8():
    """the same views extracted with norm_multi = 9, the scale at which 8-bit descriptors keep their information"""
    ps, sets, maps = _extract(9)
    yield sets, maps
    ps.uninit()


def _chain_vs_edges(lib, sets, pairs, min_length, **kw):
    """ps_tracks_from_matches on the chain's device arrays, ps_tracks_from_edges on edges built on the host from their
    downloads, the oracle, and api.tracks: all equal"""
    guided, u8 = kw.pop("guided", False), kw.pop("u8", False)
    prm = api._verify_params(**kw)
    bufs = api._DevBuffers(lib)
    try:
        ch = api._verify_chain(lib, bufs, sets, pairs, None, 0, u8, None, guided, prm)
        n_desc = [s.getDescriptorCount() for s in sets]
        n_feat = [s.getFeatureCount() for s in sets]
        match = bufs.download(ch.d_match, (ch.rows, 3), np.int32)
        src = bufs.download(ch.d_src, ch.rows, np.int32)
        mask = None if ch.d_mask is None else bufs.download(ch.d_mask, ch.rows, np.uint8)
        rev = [s.to_host()[2] for s in sets]
        n = len(sets)
        c_corr = np.ascontiguousarray(ch.n_corr, np.int32)
        got = api._tracks_dev(lib, bufs, n_feat, min_length, lambda of, st, mem, cnt: lib.ps_tracks_from_matches(
            ch.device, n, (C.c_int32 * n)(*n_feat), (C.c_void_p * n)(*[s.getReverseMap() for s in sets]), (C.c_int32 * n)(*n_desc),
            len(pairs), api._c_pairs(pairs), ch.d_match, ch.d_src, c_corr.ctypes.data, ch.d_mask, min_length, of, st, mem, C.byref(cnt)))
    finally:
        bufs.free()
    e = to.chain_edges(pairs, n_desc, n_feat, match, src, ch.n_corr, mask, rev)
    assert len(e) > 100
    off = to.offsets(n_feat)
    se = np.searchsorted(off, e, side="right") - 1
    via_edges = api.build_tracks(n_feat, np.stack([se[:, 0], e[:, 0] - off[se[:, 0]], se[:, 1], e[:, 1] - off[se[:, 1]]], 1), min_length)
    want = to.tracks(n_feat, e, min_length)
    via_api = api.tracks(sets, pairs, min_length=min_length, guided=guided, u8=u8, **kw)
    for t in (via_edges, via_api):
        for f in t._fields:
            a, b = getattr(got, f), getattr(t, f)
            if f == "track_of":
                assert all(np.array_equal(x, y) for x, y in zip(a, b))
            else:
                assert np.array_equal(a, b), f
    assert np.array_equal(got.start, want[1])
    assert np.array_equal(np.concatenate(got.track_of), want[0])
    assert (got.n_components, got.n_conflicting, got.n_short) == (want[3]["n_components"], want[3]["n_conflicting"], want[3]["n_short"])
    return got


@pytest.mark.parametrize("kw", [dict(model="homography"), dict(model="fundamental", n_samples=2048),
                                dict(model="homography", guided=True, u8=True)], ids=["H", "F", "guided-u8"])
def test_chain_against_edges_and_oracle(lib, request, kw):
    sets, _ = request.getfixturevalue("affine_sets_u8" if kw.get("u8") else "affine_sets")
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    for m in (2, 4):
        t = _chain_vs_edges(lib, sets, pairs, m, **kw)
        assert len(t.start) > 50


def test_chain_self_pairs_conflict(lib, affine_sets):
    """a self pair joins features of one set: its edges make their components conflicting"""
    sets, _ = affine_sets
    t = _chain_vs_edges(lib, sets[:3], [(0, 1), (1, 2), (0, 0)], 2)
    assert t.n_conflicting > 0


def test_geometry_end_to_end(affine_sets):
    """all ordered pairs of the 6 affine views, verified with homographies: most tracks map to one point of image 1
    through the views' known maps, and long tracks exist"""
    sets, maps = affine_sets
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    t = api.tracks(sets, pairs, model="homography", threshold=4.0)
    feats = [s.to_host()[0] for s in sets]
    inv = [np.linalg.inv(np.vstack([A, [0, 0, 1]])) for A in maps]
    lens = np.diff(t.start)
    good = 0
    for k in range(len(lens)):
        a, b = t.start[k], t.start[k + 1]
        pts = np.array([(inv[s] @ [feats[s]["x"][f], feats[s]["y"][f], 1.0])[:2] for s, f in zip(t.set[a:b], t.feature[a:b])])
        good += np.linalg.norm(pts - pts.mean(0), axis=1).max() < 3 * 4.0
    share = good / max(len(lens), 1)
    assert len(lens) > 200 and share > 0.9, (len(lens), share)
    assert (lens >= 3).sum() > 100 and (lens == 6).sum() > 20, np.bincount(lens)


def test_cpp_tracks(tmp_path):
    """popsift::buildTracks (both overloads) equal the C ABI (tests/cpp/tracks_check.cpp)"""
    from popsift_b200 import build as B
    B.build()
    files = []
    for k, (im, _) in enumerate(affine_set()[:4]):
        f = tmp_path / ("f%d.raw" % k)
        im.tofile(f)
        files.append(str(f))
    h, w = affine_set()[0][0].shape
    out = subprocess.run([B.TRACKS_CHECK, str(w), str(h)] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
