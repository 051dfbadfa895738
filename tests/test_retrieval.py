"""Image retrieval on the GPU (ps_vlad_train / ps_vlad_encode / ps_retrieve_pairs): assignment, k-means steps and VLAD
vectors against the float64 oracle, scores against the host program on the kernels' own header, neighbour lists against
the oracle's top-m rule, grouping and determinism, argument errors, an end-to-end retrieval of synthetic scenes and the
C++ API."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import retrieval_oracle as ro
from popsift_b200 import api
from popsift_b200.synth import affine_warp, make_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTO, EXACT, TENSOR = 0, 1, 2
PS_ERR_ARG = -1

pytestmark = pytest.mark.gpu


def _unit(rng, n):
    d = np.abs(rng.normal(size=(n, 128))).astype(np.float32)
    return d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12).astype(np.float32)


def _c_sets(bufs, sets):
    ptrs = [bufs.upload(np.ascontiguousarray(s, np.float32).reshape(-1, 128)) for s in sets]
    n = max(len(sets), 1)
    return (C.c_void_p * n)(*ptrs), (C.c_int32 * n)(*[len(s) for s in sets])


def _train(lib, sets, k, iters, seed=0, flags=EXACT):
    bufs = api._DevBuffers(lib)
    try:
        cs, cn = _c_sets(bufs, sets)
        d = bufs.alloc(k * 512)
        assert lib.ps_vlad_train(0, len(sets), cs, cn, k, iters, seed, d, flags) == 0, lib.ps_last_error(None)
        return bufs.download(d, (k, 128), np.float32)
    finally:
        bufs.free()


def _encode(lib, sets, cb, flags=EXACT):
    bufs = api._DevBuffers(lib)
    try:
        cs, cn = _c_sets(bufs, sets)
        N = sum(len(s) for s in sets)
        d_v, d_a = bufs.alloc(len(sets) * cb.size * 4), bufs.alloc(N * 4)
        assert lib.ps_vlad_encode(0, len(sets), cs, cn, len(cb), bufs.upload(cb), d_v, d_a, flags) == 0, lib.ps_last_error(None)
        return bufs.download(d_v, (len(sets), cb.size), np.float32), bufs.download(d_a, N, np.int32)
    finally:
        bufs.free()


def _host_scores(v, rows=None):
    from popsift_b200 import build as B
    B.build()
    v = np.ascontiguousarray(v, np.float32)
    rows = len(v) if rows is None else rows
    with tempfile.TemporaryDirectory() as d:
        inp, out = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(inp, "wb") as f:
            f.write(np.int32(v.shape[0]).tobytes() + np.int32(v.shape[1]).tobytes() + v.tobytes())
        r = subprocess.run([B.RETRIEVAL_HOST, "score", inp, out, "0", str(rows)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr
        return np.fromfile(out, np.float32).reshape(rows, len(v))


def _scenes(n_scenes, views, w, h, seed0=100):
    """n_scenes synthetic frames, each seen in `views` affine views (rotation +-20 deg, scale 0.8-1.25, shear +-0.15,
    shift +-40 px about the centre); the first view is the frame itself"""
    rng = np.random.default_rng(7)
    out = []
    for s in range(n_scenes):
        base = make_frame(w, h, seed0 + s)
        for v in range(views):
            if v == 0:
                out.append(base)
                continue
            a = np.deg2rad(rng.uniform(-20, 20))
            sc = rng.uniform(0.8, 1.25)
            sh = rng.uniform(-0.15, 0.15)
            L = sc * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]) @ np.array([[1, sh], [0, 1]])
            c = np.array([w / 2, h / 2])
            t = c - L @ c + rng.uniform(-40, 40, 2)
            out.append(affine_warp(base, np.c_[L, t]))
    return out


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


@pytest.fixture(scope="module")
def frames():
    """descriptors of 6 extracted 640x480 frames (3 scenes x 2 views), as host arrays"""
    imgs = _scenes(3, 2, 640, 480)
    ps = api.PopSift(api.Config(), max_width=640, max_height=480, slots=1)
    out = [ps.enqueue(640, 480, im).get().desc.reshape(-1, 128).astype(np.float32) for im in imgs]
    ps.uninit()
    return out


def test_assignment_random_and_planted(lib):
    rng = np.random.default_rng(1)
    sets = [_unit(rng, n) for n in (0, 5, 3000, 2049)]
    pool = np.concatenate(sets)
    for k in (1, 16, 300):
        cb = pool[rng.choice(len(pool), k, replace=False)] + rng.normal(scale=0.01, size=(k, 128)).astype(np.float32)
        _, a = _encode(lib, sets, cb.astype(np.float32))
        assert np.array_equal(a, ro.assign(pool, cb)), k
    # equidistant centroids: each descriptor is planted midway between centroids 2c and 2c + 1; the lower index wins
    base = np.zeros((8, 128), np.float32)
    for c in range(4):
        base[2 * c, c] = 1.0
        base[2 * c + 1, c + 4] = 1.0
    x = np.zeros((4, 128), np.float32)
    for c in range(4):
        x[c, c] = x[c, c + 4] = 0.5
    _, a = _encode(lib, [x], base)
    assert a.tolist() == [0, 2, 4, 6] == ro.assign(x, base).tolist()


def test_assignment_extracted_auto_equals_exact(lib, frames):
    cb = _train(lib, frames, 32, 0)
    _, a_exact = _encode(lib, frames, cb, EXACT)
    _, a_auto = _encode(lib, frames, cb, AUTO)
    assert np.array_equal(a_exact, ro.assign(np.concatenate(frames), cb))
    assert np.array_equal(a_auto, a_exact)


def test_training_steps(lib, frames):
    pool = np.concatenate(frames)
    k = 48
    c0 = _train(lib, frames, k, 0, seed=3)
    assert np.array_equal(c0, pool[ro.draw(3, len(pool), k)])
    prev = c0
    for it in range(1, 4):
        got = _train(lib, frames, k, it, seed=3)
        a = ro.assign(pool, prev)
        want = ro.kmeans_step(pool, prev, a)
        ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert ulp.max() <= 1, it
        empty = np.setdiff1d(np.arange(k), a)
        assert np.array_equal(got[empty], prev[empty])
        prev = got
    # centroids without members keep their values: rows 40..49 repeat rows 0..9, so a codebook of all 50 rows holds ten
    # duplicate centroids, and (ties to the lower index) the later of each duplicate never wins a descriptor; the others
    # are the mean of identical rows
    x = _unit(np.random.default_rng(8), 50)
    x[40:] = x[:10]
    c0 = _train(lib, [x], 50, 0)
    assert np.array_equal(c0, x[ro.draw(0, 50, 50)])
    assert len(np.setdiff1d(np.arange(50), ro.assign(x, c0))) == 10
    assert np.array_equal(_train(lib, [x], 50, 1), c0)


def test_encoding_against_oracle(lib, frames):
    sets = frames[:3] + [np.zeros((0, 128), np.float32)] + frames[3:]
    for k in (1, 8, 64):
        cb = _train(lib, frames, k, 2)
        v, a = _encode(lib, sets, cb)
        starts = np.cumsum([0] + [len(s) for s in sets])
        for i, s in enumerate(sets):
            want = ro.vlad(s, cb, a[starts[i]:starts[i + 1]])
            assert np.abs(v[i].astype(np.float64) - want).max() <= 1e-6, (k, i)
        assert not v[3].any()
        assert np.array_equal(a, ro.assign(np.concatenate(sets), cb))


_GROUP_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from popsift_b200 import api
d = np.load(sys.argv[2])
sets = [d["s%d" % i] for i in range(int(d["n"]))]
v, a = api.vlad_encode(sets, d["cb"], flags=1, assign=True)
cb = api.vlad_codebook(sets, k=64, iters=3, seed=5, flags=1)
nbr, sc = api.retrieve(d["vec"], 5)
np.savez(sys.argv[3], v=v, a=a, cb=cb, nbr=nbr, sc=sc)
"""

GROUP_SIZES = (700, 0, 2500, 1, 900, 4100, 300)
GROUP_K = 64
GROUP_WS = 250000


def _vlad_groups(sizes, k, cap, encode):
    """the number of set groups of k_retrieval.cu (set_groups with its per-set workspace estimates)"""
    per = [n * 12 + -(-n // 2048) * k * (128 * 8 + 4) + 256 + (k * 128 * 8 if encode else 0) for n in sizes]
    groups, used, first = 1, 0, True
    for b in per:
        if not first and used + b > cap:
            groups, used = groups + 1, 0
        used += b
        first = False
    return groups


def test_small_workspace_gives_identical_bytes(lib, tmp_path):
    """POPSIFT_B200_MATCH_WS small enough that training and encoding run in several groups of sets (their offsets, plan
    uploads and the training sums carried across groups) and that the score matrix goes in row blocks (no mirror): the same
    bytes as with the default workspace"""
    assert _vlad_groups(GROUP_SIZES, GROUP_K, GROUP_WS, encode=False) >= 3
    assert _vlad_groups(GROUP_SIZES, GROUP_K, GROUP_WS, encode=True) >= 5
    assert _vlad_groups(GROUP_SIZES, GROUP_K, 1 << 30, encode=True) == 1
    assert 700 * 700 * 4 > GROUP_WS
    rng = np.random.default_rng(5)
    sets = [_unit(rng, n) for n in GROUP_SIZES]
    cb = _unit(rng, GROUP_K)
    vec = rng.normal(size=(700, 132)).astype(np.float32)
    inp = str(tmp_path / "in.npz")
    np.savez(inp, n=len(sets), cb=cb, vec=vec, **{"s%d" % i: s for i, s in enumerate(sets)})
    res = []
    for ws in (None, GROUP_WS):
        out = str(tmp_path / ("out_%s.npz" % ws))
        env = dict(os.environ)
        if ws:
            env["POPSIFT_B200_MATCH_WS"] = str(ws)
        subprocess.run([sys.executable, "-c", _GROUP_SCRIPT, ROOT, inp, out], env=env, check=True, timeout=600)
        res.append(np.load(out))
    for key in ("v", "a", "cb", "nbr", "sc"):
        assert res[0][key].tobytes() == res[1][key].tobytes(), key
    # and the grouped run is right, not merely equal: assignments and encodings against the oracle
    pool = np.concatenate(sets)
    assert np.array_equal(res[1]["a"], ro.assign(pool, cb))
    starts = np.cumsum([0] + [len(s) for s in sets])
    for i, s in enumerate(sets):
        assert np.abs(res[1]["v"][i].astype(np.float64) - ro.vlad(s, cb, res[1]["a"][starts[i]:starts[i + 1]])).max() <= 1e-6


_ORDER_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from popsift_b200 import api
d = np.load(sys.argv[2])
cb = api.vlad_codebook([d["s0"], d["s1"], d["s2"]], k=1, iters=1, seed=0, flags=1)
np.save(sys.argv[3], cb)
"""


def test_training_sum_is_one_chain_across_groups(lib, tmp_path):
    """The k-means sums run as one double chain over the pool's chunks whatever the grouping.  Sets [2^54, 2^30], [1.5],
    [1.5] (dimension 0) with k = 1: in pool order each 1.5 is lost against 2^54 + 2^30 (double ulp 4), and the mean lands
    exactly halfway between two floats (rounded to even); summing the second group on its own first (1.5 + 1.5 = 3) would
    carry 4 more and round the other way.  A cap of 2 600 bytes puts the first set alone and the other two together."""
    assert _vlad_groups((2, 1, 1), 1, 2600, encode=False) == 2
    assert _vlad_groups((2, 1), 1, 2600, encode=False) == 2 and _vlad_groups((1, 1), 1, 2600, encode=False) == 1
    s0 = np.zeros((2, 128), np.float32)
    s0[0, 0], s0[1, 0] = 2.0 ** 54, 2.0 ** 30
    s1 = np.zeros((1, 128), np.float32)
    s1[0, 0] = 1.5
    chunk0 = (0.0 + 2.0 ** 54) + 2.0 ** 30
    want = np.float32((((0.0 + chunk0) + 1.5) + 1.5) / 4)
    grouped_first = np.float32((chunk0 + ((0.0 + 1.5) + 1.5)) / 4)
    assert want != grouped_first                     # the data tells the two orders apart
    inp = str(tmp_path / "order.npz")
    np.savez(inp, s0=s0, s1=s1, s2=s1)
    for ws in (None, 2600):
        out = str(tmp_path / ("order_%s.npy" % ws))
        env = dict(os.environ)
        if ws:
            env["POPSIFT_B200_MATCH_WS"] = str(ws)
        subprocess.run([sys.executable, "-c", _ORDER_SCRIPT, ROOT, inp, out], env=env, check=True, timeout=300)
        cb = np.load(out)
        assert cb[0, 0] == want, (ws, cb[0, 0], want)
        assert not cb[0, 1:].any()


@pytest.mark.parametrize("n,dim,m", [(300, 260, 7), (129, 4, 128), (1, 8, 3), (5, 64, 9), (257, 8192, 20)])
def test_retrieval_against_host_scores(lib, n, dim, m):
    rng = np.random.default_rng(n + dim)
    v = rng.normal(size=(n, dim)).astype(np.float32)
    if n > 10:
        v[10] = v[3]                     # planted duplicates: equal scores, the lower index first
        v[11] = v[3]
        v[7] = 0.0                       # all-zero row: every score +0
    nbr, sc = api.retrieve(v, m)
    S = _host_scores(v)
    want_n, want_s = ro.topm(S, m)
    assert np.array_equal(nbr, want_n)
    assert np.array_equal(sc.view(np.uint32), want_s.view(np.uint32))
    # every returned score is the host chain bit for bit, and the chain is symmetric
    assert np.array_equal(S.view(np.uint32), S.T.view(np.uint32))
    if n == 1:
        assert (nbr == -1).all() and (sc == -np.inf).all()
    if m >= n:
        assert (nbr[:, n - 1:] == -1).all()


def test_retrieval_large_rows(lib):
    """n = 1 000, dim = 8 192: the first 40 rows' neighbour lists against the host chain"""
    rng = np.random.default_rng(9)
    v = rng.normal(size=(1000, 8192)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    v[500] = v[2]
    nbr, sc = api.retrieve(v, 16)
    S = _host_scores(v, rows=40)
    want_n, want_s = ro.topm(S, 16)
    assert np.array_equal(nbr[:40], want_n)
    assert np.array_equal(sc[:40].view(np.uint32), want_s.view(np.uint32))
    assert nbr[2, 0] == 500 and nbr[500, 0] == 2


def test_retrieval_nan_rows(lib):
    v = np.random.default_rng(2).normal(size=(40, 16)).astype(np.float32)
    v[5, 3] = np.nan
    nbr, sc = api.retrieve(v, 39)
    want_n, _ = ro.topm(_host_scores(v), 39)
    assert np.array_equal(nbr, want_n)
    assert nbr[0, -1] == 5 and np.isnan(sc[0, -1])


def test_determinism(lib, frames):
    rng = np.random.default_rng(3)
    vec = rng.normal(size=(400, 256)).astype(np.float32)
    a = [api.retrieve(vec, 10) for _ in range(2)]
    assert a[0][0].tobytes() == a[1][0].tobytes() and a[0][1].tobytes() == a[1][1].tobytes()
    for flags in (EXACT, AUTO):
        cbs = [_train(lib, frames, 32, 3, flags=flags) for _ in range(2)]
        assert cbs[0].tobytes() == cbs[1].tobytes()
        enc = [_encode(lib, frames, cbs[0], flags) for _ in range(2)]
        assert enc[0][0].tobytes() == enc[1][0].tobytes() and enc[0][1].tobytes() == enc[1][1].tobytes()


def test_argument_errors(lib):
    rng = np.random.default_rng(0)
    bufs = api._DevBuffers(lib)
    try:
        x = _unit(rng, 20)
        cs, cn = _c_sets(bufs, [x])
        d_c, d_v, d_a = bufs.alloc(64 * 512), bufs.alloc(64 * 512), bufs.alloc(80)
        host = np.zeros(64 * 128, np.float32)
        T, E = lib.ps_vlad_train, lib.ps_vlad_encode
        assert T(0, 1, cs, cn, 21, 1, 0, d_c, 0) == PS_ERR_ARG                  # k > N
        assert T(0, 1, cs, cn, 0, 1, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, cs, cn, 1025, 1, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, cs, cn, 4, -1, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, cs, cn, 4, 1001, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, cs, cn, 4, 1, 0, host.ctypes.data, 0) == PS_ERR_ARG     # host centroids
        assert T(0, -1, cs, cn, 4, 1, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, None, cn, 4, 1, 0, d_c, 0) == PS_ERR_ARG
        hs = (C.c_void_p * 1)(x.ctypes.data)                                   # a host set
        assert T(0, 1, hs, cn, 4, 1, 0, d_c, 0) == PS_ERR_ARG
        neg = (C.c_int32 * 1)(-1)
        assert T(0, 1, cs, neg, 4, 1, 0, d_c, 0) == PS_ERR_ARG
        assert T(0, 1, cs, cn, 20, 0, 0, d_c, 0) == 0                           # N == k is fine
        assert E(0, 1, cs, cn, 0, d_c, d_v, None, 0) == PS_ERR_ARG
        assert E(0, 1, cs, cn, 1025, d_c, d_v, None, 0) == PS_ERR_ARG
        assert E(0, 1, hs, cn, 4, d_c, d_v, None, 0) == PS_ERR_ARG
        assert E(0, 1, cs, neg, 4, d_c, d_v, None, 0) == PS_ERR_ARG
        assert E(0, 1, cs, cn, 4, host.ctypes.data, d_v, None, 0) == PS_ERR_ARG
        assert E(0, 1, cs, cn, 4, d_c, host.ctypes.data, None, 0) == PS_ERR_ARG
        assert E(0, 1, cs, cn, 4, d_c, d_v, host.ctypes.data, 0) == PS_ERR_ARG
        assert E(0, 0, None, None, 4, None, None, None, 0) == 0                 # nothing to do
        assert E(0, 1, cs, cn, 4, d_c, d_v, d_a, 0) == 0
        R = lib.ps_retrieve_pairs
        d_n, d_s = bufs.alloc(20 * 128 * 4), bufs.alloc(20 * 128 * 4)
        assert R(0, 20, d_v, 64, 5, d_n, d_s) == 0
        assert R(0, 20, d_v, 62, 5, d_n, d_s) == PS_ERR_ARG                     # dim % 4
        assert R(0, 20, d_v, 0, 5, d_n, d_s) == PS_ERR_ARG
        assert R(0, 20, d_v, 64, 0, d_n, d_s) == PS_ERR_ARG
        assert R(0, 20, d_v, 64, 129, d_n, d_s) == PS_ERR_ARG
        assert R(0, -1, d_v, 64, 5, d_n, d_s) == PS_ERR_ARG
        assert R(0, 20, d_v + 4, 64, 5, d_n, d_s) == PS_ERR_ARG                 # not 16-byte aligned
        assert R(0, 20, host.ctypes.data, 64, 5, d_n, d_s) == PS_ERR_ARG
        assert R(0, 20, d_v, 64, 5, host.ctypes.data, d_s) == PS_ERR_ARG
        assert R(0, 20, d_v, 64, 5, d_n, host.ctypes.data) == PS_ERR_ARG
        assert R(0, 0, None, 64, 5, None, None) == 0
    finally:
        bufs.free()


def test_end_to_end_scenes(lib):
    """12 scenes x 4 views at 640x480, extracted on the GPU: k = 64, 10 iterations, seed 0, m = 3 retrieves exactly the
    other views of each scene, and every selected pair verifies with a homography of at least 60 inliers"""
    n_sc, views, w, h = 12, 4, 640, 480
    imgs = _scenes(n_sc, views, w, h)
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    sets = [ps.enqueue(w, h, im).getDev() for im in imgs]
    cb = api.vlad_codebook(sets, k=64, iters=10, seed=0)
    v = api.vlad_encode(sets, cb)
    nbr, sc = api.retrieve(v, 3)
    scene = np.arange(len(sets)) // views
    prec = (scene[nbr] == scene[:, None]).mean()
    assert prec == 1.0, (prec, sc)
    pairs = api.select_pairs(nbr)
    want = sorted((i, j) for i in range(len(sets)) for j in range(i + 1, len(sets)) if scene[i] == scene[j])
    assert pairs == want and len(pairs) == 72
    res = api.verify_pairs(sets, pairs, model="homography", threshold=4.0)
    n_in = [r[1] for r in res]
    print("retrieval e2e: same-scene cos min %.3f, inliers min %d median %d" % (sc.min(), min(n_in), int(np.median(n_in))))
    # the first run on an H100 gave at least 140 inliers per pair (median 205); the floor leaves room for extraction order
    assert min(n_in) >= 60, n_in
    ps.uninit()


def test_cpp_retrieval(tmp_path):
    """popsift::vladCodebook / vladEncode / retrievePairs equal the C ABI (tests/cpp/retrieval_check.cpp)"""
    from popsift_b200 import build as B
    B.build()
    files = []
    for k, im in enumerate(_scenes(2, 2, 640, 480)):
        f = tmp_path / ("f%d.raw" % k)
        im.tofile(f)
        files.append(str(f))
    out = subprocess.run([B.RETRIEVAL_CHECK, "640", "480"] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
