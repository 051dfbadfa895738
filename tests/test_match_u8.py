"""Exact 8-bit descriptor matching (ps_descriptors_to_u8 / ps_match_u8_batch, popsift::matchPairsU8, api.descriptors_to_u8 /
api.match_pairs_u8).  The oracle is numpy: squared distances by a float64 matmul (exact for these integers), the
lexicographically smallest (distance, index) pair and the next one, and the ratio in float32.  Every comparison is exact."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from popsift_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EXACT, TENSOR, AUTO = api.FeaturesDev.MATCH_EXACT, api.FeaturesDev.MATCH_TENSOR, api.FeaturesDev.MATCH_AUTO
U8_ROW_BYTES = 132          # k_match_plan.h kMatchU8RowBytes: a pooled 8-bit row and its norm key


def _plan_check():
    from popsift_b200 import build as B
    B.build()
    return B.MATCH_PLAN_U8_CHECK


def _plan(sms, cap, sizes, pairs, row_bytes=U8_ROW_BYTES):
    out = subprocess.run([_plan_check(), "plan", str(sms), str(cap), ",".join(map(str, sizes)),
                          ",".join(str(v) for p in pairs for v in p), str(row_bytes)],
                         capture_output=True, text=True, check=True).stdout.strip()
    g, s = out.split()
    return int(g.split("=")[1]), [int(v) for v in s.split("=")[1].split(",") if v]


def test_u8_planner_sweep_at_132_byte_rows():
    """The planner sweep of test_match_planner_covers_every_tile_pair_once at the 8-bit matcher's 132-byte rows
    (tests/cpp/match_plan_u8_check.cpp), and plans asked for at the float row size equal the default plans."""
    out = subprocess.run([_plan_check()], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("OK u8 "), out.stdout


def test_u8_planner_row_size():
    """8-bit rows change only how many sets fit a group: the same work split for one pair, about 8x more rows per group."""
    assert _plan(132, 1 << 30, [64, 60000], [(0, 1)]) == (1, [8])
    assert _plan(132, 1 << 30, [200, 50000], [(0, 1)]) == (1, [8])
    assert _plan(132, 1 << 30, [16330, 16330], [(0, 1)]) == (1, [1])
    assert _plan(132, 1 << 30, [1, 50000], [(0, 1)]) == (1, [8])         # the chunk boundaries of the tie tests
    # 40 sets of 100 000 descriptors, each matched with the next: ~4 GB of float rows but ~0.5 GB of 8-bit rows
    pairs = [(i, (i + 1) % 40) for i in range(40)]
    assert _plan(132, 1 << 30, [100000] * 40, pairs, 1028)[0] > 1
    assert _plan(132, 1 << 30, [100000] * 40, pairs)[0] == 1


def test_shipped_sass_u8_matcher_uses_tma_and_igmma():
    """match_u8_kernel streams its operands with TMA and issues integer warpgroup MMAs (IGMMA), no float ones (HGMMA)."""
    import shutil
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lib = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_hist
    k = sass_hist.histogram(lib)
    u8 = {n: c for n, c in k.items() if "match_u8_kernelE" in n}
    assert u8, "match_u8_kernel not in the library"
    for n, c in u8.items():
        assert c["IGMMA"] > 0 and c["UTMALDG"] > 0 and c["HGMMA"] == 0, n


# ------------------------------------------------------------------------------------------------------------- oracle

def oracle(l, r):
    """(n_left, 3) int32 rows (best, second, accept) of 8-bit sets l and r, from exact float64 distances"""
    l = np.asarray(l, np.float64).reshape(-1, 128)
    r = np.asarray(r, np.float64).reshape(-1, 128)
    out = np.zeros((len(l), 3), np.int32)
    if len(l) == 0 or len(r) == 0:
        return out
    rn = (r * r).sum(1)
    for s in range(0, len(l), 2048):
        a = l[s:s + 2048]
        d = (a * a).sum(1)[:, None] + rn[None, :] - 2.0 * (a @ r.T)
        rows = np.arange(len(a))
        i1 = np.argmin(d, 1)                                  # first occurrence: the smallest index among equal distances
        d1 = d[rows, i1].copy()
        if len(r) > 1:
            d[rows, i1] = np.inf
            i2 = np.argmin(d, 1)
            d2 = d[rows, i2]
        else:
            i2, d2 = np.zeros(len(a), np.int64), np.full(len(a), np.inf)
        with np.errstate(divide="ignore", invalid="ignore"):
            acc = (d1.astype(np.float32) / d2.astype(np.float32)) < np.float32(0.8)
        out[s:s + len(a)] = np.stack([i1, i2, acc.astype(np.int64)], 1)
    return out


def _rand_u8(rng, n, hi=64):
    return rng.integers(0, hi, size=(n, 128)).astype(np.uint8)


def _near(rng, x, scale=2):
    return np.clip(x.astype(np.int32) + rng.integers(-scale, scale + 1, size=x.shape), 0, 255).astype(np.uint8)


def _random_sets():
    rng = np.random.default_rng(17)
    sizes = [0, 1, 2, 127, 128, 129, 1000, 4097, 7000]
    sets = [_rand_u8(rng, n) for n in sizes]
    # planted near-duplicates: true matches between some of the sets
    sets[8][100:600] = _near(rng, sets[7][:500])
    sets[6][:120] = _near(rng, sets[5][:120])
    sets[7][3000:3900] = _near(rng, sets[6][:900], 1)
    sets[4][:2] = _near(rng, sets[2])
    return sets


# ------------------------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
def test_match_u8_pairs_equal_oracle():
    """Sizes {0, 1, 2, 127, 128, 129, 1000, 4097, 7000} with planted near-duplicates, all 81 ordered pairs (self pairs
    included) in one call under AUTO, TENSOR and EXACT: every pair's rows equal the numpy oracle and ps_match_batch(EXACT)
    on float32 copies."""
    sets = _random_sets()
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets))]
    want = [oracle(sets[i], sets[j]) for i, j in pairs]
    flt = api.match_pairs([s.astype(np.float32) for s in sets], pairs, EXACT)
    for p, f, w in zip(pairs, flt, want):
        assert np.array_equal(f, w), ("float exact", p, int((f != w).any(1).sum()))
    for flags in (AUTO, TENSOR, EXACT):
        got = api.match_pairs_u8(sets, pairs, flags)
        assert len(got) == len(pairs)
        for p, g, w in zip(pairs, got, want):
            assert g.shape == (len(sets[p[0]]), 3)
            assert np.array_equal(g, w), (flags, p, int((g != w).any(1).sum()))
    # the planted matches are found, and a self pair finds every (distinct) descriptor itself
    m = want[pairs.index((7, 8))]
    assert (m[:500, 0] == np.arange(100, 600)).all()
    s = want[pairs.index((7, 7))]
    assert (s[:, 0] == np.arange(len(sets[7]))).all()
    assert not want[pairs.index((6, 0))].any() and want[pairs.index((0, 6))].shape == (0, 3)


def _tie_case(rng, n, positions, dup=(), far=()):
    """A one-row left set a = 100 everywhere and an n-row right set: background rows far from a, tie rows at `positions`
    all exactly at distance 25 from a (+5 in a different component each), exact copies of a at `dup`, and rows at distance
    100 (+10 in one component) at `far`."""
    a = np.full((1, 128), 100, np.uint8)
    r = (100 + rng.choice([-1, 1], size=(n, 128)) * rng.integers(20, 60, size=(n, 128))).astype(np.uint8)
    for k, p in enumerate(positions):
        r[p] = 100
        r[p, k % 128] = 105
    for p in dup:
        r[p] = 100
    for k, p in enumerate(far):
        r[p] = 100
        r[p, k % 128] = 110
    return a, r


def _tie_cases():
    rng = np.random.default_rng(3)
    cases = [
        ("one thread's columns", 300, dict(positions=[8, 1, 0]), (0, 1, 0)),
        ("quad lanes", 300, dict(positions=[3, 5, 6]), (3, 5, 0)),
        ("quad lanes, reverse", 300, dict(positions=[6, 2]), (2, 6, 0)),
        ("quad lanes, lower index on a higher lane", 300, dict(positions=[8, 3, 9]), (3, 8, 0)),
        ("tiles", 1000, dict(positions=[129 + 128 * 3, 300, 130]), (130, 300, 0)),
        ("chunks, issue positions", 50000, dict(positions=[5, 130, 40000]), (5, 130, 0)),
        ("chunks only", 50000, dict(positions=[45000, 20000, 7000]), (7000, 20000, 0)),
        ("chunks, last column", 50000, dict(positions=[49999, 6300]), (6300, 49999, 0)),
        ("duplicates of the left row", 2000, dict(positions=[10], dup=[1500, 700, 1999]), (700, 1500, 0)),
        ("one duplicate and a farther row", 2000, dict(positions=[], dup=[1234], far=[77]), (1234, 77, 1)),
        ("one duplicate, ties behind it", 50000, dict(positions=[44000, 3], dup=[20000]), (20000, 3, 1)),
    ]
    out = []
    for name, n, kw, want in cases:
        a, r = _tie_case(rng, n, **kw)
        out.append((name, a, r, want))
    return out


@pytest.mark.gpu
def test_match_u8_ties_across_every_boundary():
    """Right descriptors at exactly the same distance from the left row, placed inside one thread's 32 columns, across the
    four lanes of a quad, across tiles and across the S = 8 chunks of a 50 000 set; exact duplicates of the left row
    (0 / 0: accept 0) and a single duplicate before farther rows (accept 1).  Expected: (lowest index, next index, accept)."""
    cases = _tie_cases()
    sets, pairs = [], []
    for _, a, r, _ in cases:
        pairs.append((len(sets), len(sets) + 1))
        sets += [a, r]
    for flags in (AUTO, TENSOR, EXACT):
        got = api.match_pairs_u8(sets, pairs, flags)
        for (name, a, r, want), g in zip(cases, got):
            assert tuple(g[0]) == want, (flags, name, tuple(g[0]))
            assert np.array_equal(g, oracle(a, r)), (flags, name)
            # alone, a one-row left set against 50 000 takes S = 8 (test_u8_planner_row_size)
            assert tuple(api.match_pairs_u8([a, r], [(0, 1)], flags)[0][0]) == want, (flags, name, "alone")


@pytest.mark.gpu
def test_match_u8_extremes():
    """All-255 against all-0 (distance 128 * 255^2 = 8 323 200, every row (0, 1, 0)); all-zero sets (every distance equal);
    right sets of one descriptor ((0, 0, 1)); an empty right set ((0, 0, 0))."""
    hi, lo = np.full((300, 128), 255, np.uint8), np.zeros((260, 128), np.uint8)
    one = np.full((1, 128), 7, np.uint8)
    rng = np.random.default_rng(8)
    sets = [hi, lo, one, _rand_u8(rng, 500, 256), np.zeros((0, 128), np.uint8)]
    pairs = [(0, 1), (1, 0), (1, 1), (0, 0), (0, 2), (3, 2), (2, 2), (3, 4), (2, 0)]
    for flags in (AUTO, TENSOR, EXACT):
        got = api.match_pairs_u8(sets, pairs, flags)
        for p, g in zip(pairs, got):
            assert np.array_equal(g, oracle(sets[p[0]], sets[p[1]])), (flags, p)
        for k in range(4):
            assert (got[k] == np.array([0, 1, 0])).all(), (flags, pairs[k])
        assert (got[4] == np.array([0, 0, 1])).all() and (got[5] == np.array([0, 0, 1])).all()
        assert not got[7].any() and got[7].shape == (500, 3)


@pytest.mark.gpu
def test_match_u8_work_split_equals_oracle():
    """64 x 60 000 and 200 x 50 000: the planner cuts each right set into S = 8 chunks (test_u8_planner_row_size)."""
    rng = np.random.default_rng(5)
    a, b, c, d = _rand_u8(rng, 64), _rand_u8(rng, 60000), _rand_u8(rng, 200), _rand_u8(rng, 50000)
    b[40000:40064] = _near(rng, a)
    d[7:207] = _near(rng, c)
    w1, w2 = oracle(a, b), oracle(c, d)
    assert (w1[:, 0] == np.arange(40000, 40064)).all() and (w2[:, 0] == np.arange(7, 207)).all()
    for flags in (AUTO, TENSOR, EXACT):
        g = api.match_pairs_u8([a, b, c, d], [(0, 1), (2, 3)], flags)
        assert np.array_equal(g[0], w1) and np.array_equal(g[1], w2), flags


_GROUP_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from popsift_b200 import api
z = np.load(sys.argv[2])
sets = [z["s%d" % i] for i in range(int(z["n"]))]
out = api.match_pairs_u8(sets, [tuple(p) for p in z["pairs"]], int(z["flags"]))
np.savez(sys.argv[3], *out)
"""


@pytest.mark.gpu
def test_match_u8_small_workspace_cap_gives_same_rows(tmp_path):
    """POPSIFT_B200_MATCH_WS small enough for at least three groups at 132-byte rows (checked with the planner), tie sets
    in several groups: the same rows as one group, and the oracle's."""
    rng = np.random.default_rng(9)
    sizes = [3000, 2500, 3100, 900, 0, 2000]
    sets = [_rand_u8(rng, n) for n in sizes]
    sets[1][:800] = _near(rng, sets[0][200:1000])
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if (i + j) % 2 == 0 or i == 5]
    # tie cases, each pair in its own group under the cap
    for _, a, r, _ in _tie_cases()[:4]:
        pairs.append((len(sets), len(sets) + 1))
        sets += [a, r]
    sizes = [len(s) for s in sets]
    cap = 1 << 20
    assert _plan(132, cap, sizes, pairs)[0] >= 3
    inp, res = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    for flags in (AUTO, TENSOR):
        np.savez(inp, n=len(sets), pairs=np.array(pairs, np.int32), flags=flags, **{"s%d" % i: s for i, s in enumerate(sets)})
        env = dict(os.environ, POPSIFT_B200_MATCH_WS=str(cap))
        subprocess.run([sys.executable, "-c", _GROUP_SCRIPT, ROOT, inp, res], env=env, check=True, timeout=300)
        z = np.load(res)
        forced = [z["arr_%d" % k] for k in range(len(pairs))]
        whole = api.match_pairs_u8(sets, pairs, flags)
        for p, f, w in zip(pairs, forced, whole):
            assert np.array_equal(f, w), (flags, p)
            assert np.array_equal(w, oracle(sets[p[0]], sets[p[1]])), (flags, p)


def _extract(seed, w=640, h=480, norm_multi=9):
    from popsift_b200.synth import make_frame
    cfg = api.Config()
    cfg.setNormalizationMultiplier(norm_multi)
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    fd = ps.enqueue(w, h, make_frame(w, h, seed)).getDev()
    return ps, fd


@pytest.mark.gpu
def test_descriptors_to_u8_rounding():
    """ps_descriptors_to_u8 equals floor(float64(v) + 0.5) clamped to [0, 255] (NaN -> 0) on the half-way cases, the
    saturating ones and the specials; on an extracted frame (norm_multi = 9) it is roundf of the downloaded floats
    wherever they are <= 255."""
    special = np.array([0.0, 0.49999997, 0.5, 1.5, 2.5, 254.5, 255.49, 255.5, 1e9, -3.0, np.inf, -np.inf, np.nan, -0.0,
                        0.5000001, 127.5, 1e-30, 3.4e38], np.float32)
    rng = np.random.default_rng(4)
    x = np.concatenate([special, (rng.random(128 * 40 - len(special)) * 300 - 20).astype(np.float32)]).reshape(-1, 128)
    with np.errstate(invalid="ignore"):
        want = np.clip(np.floor(np.nan_to_num(x.astype(np.float64), nan=0.0) + 0.5), 0, 255).astype(np.uint8)
    got = api.descriptors_to_u8(x)
    assert got.dtype == np.uint8 and got.shape == x.shape
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    assert got[0, 12] == 0 and got[0, 2] == 1 and got[0, 5] == 255 and got[0, 7] == 255
    ps, fd = _extract(31)
    try:
        _, desc, _ = fd.to_host()
        q = api.descriptors_to_u8(fd)
        assert len(desc) > 100 and q.shape == desc.shape
        m = desc <= 255
        assert m.mean() > 0.99 and desc.max() > 20          # norm_multi = 9 puts the components in the 8-bit range
        assert np.array_equal(q[m], np.floor(desc[m].astype(np.float64) + 0.5).astype(np.uint8))
        assert (q[~m] == 255).all()
    finally:
        del fd
        ps.uninit()


@pytest.mark.gpu
def test_match_pairs_u8_features_dev_equals_host_arrays():
    """api.match_pairs_u8 on FeaturesDev sets (quantised on the device) equals the same call on descriptors_to_u8 host
    arrays, and the oracle."""
    ps, a = _extract(41)
    _, b = _extract(42)
    try:
        host = [api.descriptors_to_u8(a), api.descriptors_to_u8(b)]
        pairs = [(0, 1), (1, 0), (0, 0), (1, 1)]
        for flags in (AUTO, TENSOR, EXACT):
            g_dev = api.match_pairs_u8([a, b], pairs, flags)
            g_host = api.match_pairs_u8(host, pairs, flags)
            for p, x, y in zip(pairs, g_dev, g_host):
                assert np.array_equal(x, y), (flags, p)
                assert np.array_equal(x, oracle(host[p[0]], host[p[1]])), (flags, p)
    finally:
        del a, b
        ps.uninit()


@pytest.mark.gpu
def test_cpp_match_pairs_u8_equals_float_exact(tmp_path):
    """popsift::matchPairsU8 (C++ API) on three frames extracted under Config::MatchingMode with norm_multi = 9, all nine
    pairs, under AUTO, EXACT and TENSOR: equals ps_match_batch(PS_MATCH_EXACT) on the quantised descriptors widened to float."""
    from popsift_b200 import build as B
    from popsift_b200.synth import make_frame
    exe = B.MATCH_U8_CHECK
    assert os.path.exists(exe), "build the product first (python -m popsift_b200.build)"
    w, h = 640, 480
    files = []
    for k in range(3):
        f = str(tmp_path / ("f%d.raw" % k))
        make_frame(w, h, 21 + k).tofile(f)
        files.append(f)
    out = subprocess.run([exe, str(w), str(h)] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK 9 "), out.stdout + out.stderr
    assert int(out.stdout.split()[3]) > 0                       # some matches pass the ratio test


@pytest.mark.gpu
def test_match_u8_batch_argument_errors():
    """A host pointer, a pointer that is not 16-byte aligned, a set index out of range and negative counts are refused
    with PS_ERR_ARG; so are bad ps_descriptors_to_u8 arguments."""
    lib = api.load_library()
    n = 300
    rng = np.random.default_rng(1)
    host = np.ascontiguousarray(_rand_u8(rng, n))
    d_set = lib.ps_dev_alloc(host.nbytes + 16)
    d_out = lib.ps_dev_alloc(3 * 4 * 2 * n)
    assert d_set and d_out
    try:
        assert lib.ps_host_to_dev(d_set, host.ctypes.data, host.nbytes) == 0
        def call(ptrs, counts, pairs):
            c_sets = (C.c_void_p * len(ptrs))(*ptrs)
            c_n = (C.c_int32 * len(counts))(*counts)
            c_p = (C.c_int32 * len(pairs))(*pairs)
            return lib.ps_match_u8_batch(0, len(ptrs), c_sets, c_n, len(pairs) // 2, c_p, d_out, 0)
        assert call([d_set], [n], [0, 0]) == 0                                    # the valid call
        assert call([host.ctypes.data], [n], [0, 0]) == -1                        # host pointer
        assert call([d_set + 8], [n], [0, 0]) == -1                               # not 16-byte aligned
        assert call([d_set, d_set + 4], [n, n], [0, 0]) == -1                     # ... even if no pair uses it
        assert call([d_set], [n], [0, 1]) == -1                                   # set index out of range
        assert call([d_set], [n], [-1, 0]) == -1
        assert call([d_set], [-5], [0, 0]) == -1                                  # negative count
        assert lib.ps_match_u8_batch(0, -1, None, None, 0, None, d_out, 0) == -1
        assert lib.ps_match_u8_batch(0, 1, (C.c_void_p * 1)(d_set), (C.c_int32 * 1)(n), -1, None, d_out, 0) == -1
        assert lib.ps_descriptors_to_u8(0, None, 3, d_out) == -1
        assert lib.ps_descriptors_to_u8(0, d_set, -1, d_out) == -1
        assert lib.ps_descriptors_to_u8(0, host.ctypes.data, 1, d_out) == -1     # host pointer
        assert lib.ps_descriptors_to_u8(0, d_set, 0, None) == 0                   # nothing to do
    finally:
        lib.ps_dev_free(d_set)
        lib.ps_dev_free(d_out)
