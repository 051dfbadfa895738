"""Batched descriptor matching (ps_match_batch / api.match_pairs / popsift::matchPairs): every pair's rows equal the
per-pair CUDA-core kernel (the reference's compute_distance order) and, on the reference's own runs, the reference's
lines.  The planner behind it (k_match_plan.h) is swept on the host."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from popsift_b200 import api

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = os.path.join(HERE, "golden")
EXACT, TENSOR, AUTO = api.FeaturesDev.MATCH_EXACT, api.FeaturesDev.MATCH_TENSOR, api.FeaturesDev.MATCH_AUTO


def _plan_check():
    from popsift_b200 import build as B
    B.build()
    return B.MATCH_PLAN_CHECK


def test_match_planner_covers_every_tile_pair_once():
    """Random set sizes (0, 1, 129, ...), pair lists with repeats and self pairs, 132 / 148 SMs, caps down to 3 MB:
    exact coverage, contiguous chunks, S bound, cap per group, output prefix sums, S = 1 once the left tiles fill the SMs."""
    exe = _plan_check()
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("OK"), out.stdout


def test_match_planner_single_pair_choices():
    """A 4K frame pair (16 330 descriptors a side, 128 left tiles) keeps one chunk per row on 132 SMs; one or two left
    tiles against 50 000+ right descriptors are cut into the maximum of 8 chunks."""
    exe = _plan_check()
    def plan(sms, cap, sizes, pairs):
        out = subprocess.run([exe, "plan", str(sms), str(cap), ",".join(map(str, sizes)), ",".join(str(v) for p in pairs for v in p)],
                             capture_output=True, text=True, check=True).stdout.strip()
        g, s = out.split()
        return int(g.split("=")[1]), [int(v) for v in s.split("=")[1].split(",") if v]
    assert plan(132, 1 << 30, [16330, 16330], [(0, 1)]) == (1, [1])
    assert plan(132, 1 << 30, [64, 60000], [(0, 1)]) == (1, [8])
    assert plan(132, 1 << 30, [200, 50000], [(0, 1)]) == (1, [8])
    # 16 frames of ~4000 descriptors, all 240 ordered pairs: 7680 left tiles fill the SMs, one group, one chunk
    pairs = [(i, j) for i in range(16) for j in range(16) if i != j]
    assert plan(132, 1 << 30, [4000] * 16, pairs) == (1, [1])


# ------------------------------------------------------------------------------------------------------------- GPU

def _unit(rng, n):
    d = np.abs(rng.normal(size=(n, 128))).astype(np.float32)
    return d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12).astype(np.float32)


def _random_sets():
    rng = np.random.default_rng(11)
    sizes = [0, 1, 2, 127, 129, 1000, 4097, 7000]
    sets = [_unit(rng, n) for n in sizes]
    # planted near-duplicates: true matches between some of the sets
    sets[7][100:600] = sets[6][:500] + rng.normal(scale=0.01, size=(500, 128)).astype(np.float32)
    sets[5][:120] = sets[4][:120] + rng.normal(scale=0.01, size=(120, 128)).astype(np.float32)
    sets[6][3000:3900] = sets[5][:900] + rng.normal(scale=0.005, size=(900, 128)).astype(np.float32)
    sets[3][:2] = sets[2] + rng.normal(scale=0.01, size=(2, 128)).astype(np.float32)
    return sets


@pytest.mark.gpu
def test_match_pairs_equal_per_pair_exact_kernel():
    """Sizes {0, 1, 2, 127, 129, 1000, 4097, 7000} with planted near-duplicates, all 64 ordered pairs (self pairs
    included) in one call under AUTO, TENSOR and EXACT: each pair's rows equal match_descriptors(l, r, EXACT)."""
    sets = _random_sets()
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets))]
    want = [api.match_descriptors(sets[i], sets[j], EXACT) for i, j in pairs]
    for flags in (AUTO, TENSOR, EXACT):
        got = api.match_pairs(sets, pairs, flags)
        assert len(got) == len(pairs)
        for (i, j), g, w in zip(pairs, got, want):
            assert g.shape == (len(sets[i]), 3)
            assert np.array_equal(g, w), (flags, i, j, int((g != w).any(1).sum()))
    # the planted matches are found, and a set's self pair finds every descriptor itself
    m = want[pairs.index((6, 7))]
    assert (m[:500, 0] == np.arange(100, 600)).mean() > 0.99 and m[:500, 2].mean() > 0.9
    s = want[pairs.index((6, 6))]
    assert (s[:, 0] == np.arange(len(sets[6]))).all()
    # empty right set: (0, 0, 0) rows; empty left set: no rows
    assert not want[pairs.index((5, 0))].any() and want[pairs.index((0, 5))].shape == (0, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("stem", ["match_640", "match_aff12"])
def test_match_pairs_reference_lines(stem):
    """The reference's own descriptors and match() lines (tests/golden/match_*.npz): in a batch of [(0, 1), (1, 0),
    (0, 0)] the first pair gives exactly the reference's (best, second, accept) for every descriptor."""
    z = np.load(os.path.join(G, stem + ".npz"))
    L = z["lines"]
    want = np.stack([L["r1"], L["r2"], L["accept"].astype(np.int32)], 1)
    sets = [z["desc0"], z["desc1"]]
    for flags in (AUTO, TENSOR, EXACT):
        got = api.match_pairs(sets, [(0, 1), (1, 0), (0, 0)], flags)
        assert np.array_equal(got[0], want), (flags, int((got[0] != want).any(1).sum()))
        assert np.array_equal(got[1], api.match_descriptors(sets[1], sets[0], EXACT))
        assert np.array_equal(got[2], api.match_descriptors(sets[0], sets[0], EXACT))


@pytest.mark.gpu
def test_match_work_split_equals_exact():
    """64 x 60 000 and 200 x 50 000: too few left tiles to fill the SMs, so each row's right set is cut into chunks
    (S = 8, see test_match_planner_single_pair_choices); ps_match and ps_match_batch both equal the exact kernel."""
    rng = np.random.default_rng(5)
    a, b, c, d = _unit(rng, 64), _unit(rng, 60000), _unit(rng, 200), _unit(rng, 50000)
    b[40000:40064] = a + rng.normal(scale=0.01, size=a.shape).astype(np.float32)
    d[7:207] = c + rng.normal(scale=0.01, size=c.shape).astype(np.float32)
    w1, w2 = api.match_descriptors(a, b, EXACT), api.match_descriptors(c, d, EXACT)
    assert (w1[:, 0] == np.arange(40000, 40064)).all() and (w2[:, 0] == np.arange(7, 207)).all()
    for flags in (AUTO, TENSOR):
        assert np.array_equal(api.match_descriptors(a, b, flags), w1), flags
        assert np.array_equal(api.match_descriptors(c, d, flags), w2), flags
        g = api.match_pairs([a, b, c, d], [(0, 1), (2, 3)], flags)
        assert np.array_equal(g[0], w1) and np.array_equal(g[1], w2), flags


_GROUP_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from popsift_b200 import api
z = np.load(sys.argv[2])
sets = [z["s%d" % i] for i in range(int(z["n"]))]
out = api.match_pairs(sets, [tuple(p) for p in z["pairs"]], int(z["flags"]))
np.savez(sys.argv[3], *out)
"""


@pytest.mark.gpu
def test_match_pairs_small_workspace_cap_gives_same_rows(tmp_path):
    """POPSIFT_B200_MATCH_WS small enough for at least three groups (checked with the planner): same rows as one group."""
    rng = np.random.default_rng(9)
    sizes = [3000, 2500, 3100, 900, 0, 2000]
    sets = [_unit(rng, n) for n in sizes]
    sets[1][:800] = sets[0][200:1000] + rng.normal(scale=0.01, size=(800, 128)).astype(np.float32)
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if (i + j) % 2 == 0 or i == 5]
    cap = 8 << 20
    exe = _plan_check()
    out = subprocess.run([exe, "plan", "132", str(cap), ",".join(map(str, sizes)), ",".join(str(v) for p in pairs for v in p)],
                         capture_output=True, text=True, check=True).stdout
    assert int(out.split()[0].split("=")[1]) >= 3, out
    inp, res = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    for flags in (AUTO, TENSOR):
        np.savez(inp, n=len(sets), pairs=np.array(pairs, np.int32), flags=flags, **{"s%d" % i: s for i, s in enumerate(sets)})
        env = dict(os.environ, POPSIFT_B200_MATCH_WS=str(cap))
        subprocess.run([sys.executable, "-c", _GROUP_SCRIPT, ROOT, inp, res], env=env, check=True, timeout=300)
        z = np.load(res)
        forced = [z["arr_%d" % k] for k in range(len(pairs))]
        whole = api.match_pairs(sets, pairs, flags)
        for p, f, w in zip(pairs, forced, whole):
            assert np.array_equal(f, w), (flags, p)
            assert np.array_equal(w, api.match_descriptors(sets[p[0]], sets[p[1]], EXACT)), (flags, p)


@pytest.mark.gpu
def test_cpp_match_pairs_equals_match_indices(tmp_path):
    """popsift::matchPairs (C++ API) on three frames extracted under Config::MatchingMode equals
    FeaturesDev::matchIndices pair by pair, self pairs included, under AUTO, EXACT and TENSOR."""
    from popsift_b200 import build as B
    from popsift_b200.synth import make_frame
    exe = B.MATCH_PAIRS_CHECK
    assert os.path.exists(exe), "build the product first (python -m popsift_b200.build)"
    w, h = 640, 480
    files = []
    for k in range(3):
        f = str(tmp_path / ("f%d.raw" % k))
        make_frame(w, h, 21 + k).tofile(f)
        files.append(f)
    out = subprocess.run([exe, str(w), str(h)] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK 9 "), out.stdout + out.stderr


@pytest.mark.gpu
def test_match_batch_argument_errors():
    """A host pointer as a set, a set index out of range and a negative count are refused with PS_ERR_ARG."""
    lib = api.load_library()
    n = 300
    rng = np.random.default_rng(1)
    host = np.ascontiguousarray(_unit(rng, n))
    d_set = lib.ps_dev_alloc(host.nbytes)
    d_out = lib.ps_dev_alloc(3 * 4 * 2 * n)
    assert d_set and d_out
    try:
        assert lib.ps_host_to_dev(d_set, host.ctypes.data, host.nbytes) == 0
        def call(ptrs, counts, pairs):
            c_sets = (C.c_void_p * len(ptrs))(*ptrs)
            c_n = (C.c_int32 * len(counts))(*counts)
            c_p = (C.c_int32 * len(pairs))(*pairs)
            return lib.ps_match_batch(0, len(ptrs), c_sets, c_n, len(pairs) // 2, c_p, d_out, 0)
        assert call([d_set], [n], [0, 0]) == 0                                    # the valid call
        assert call([host.ctypes.data], [n], [0, 0]) == -1                        # host pointer
        assert call([d_set], [n], [0, 1]) == -1                                   # set index out of range
        assert call([d_set], [n], [-1, 0]) == -1
        assert call([d_set], [-5], [0, 0]) == -1                                  # negative count
        assert lib.ps_match_batch(0, -1, None, None, 0, None, d_out, 0) == -1
        assert lib.ps_match_batch(0, 1, (C.c_void_p * 1)(d_set), (C.c_int32 * 1)(n), -1, None, d_out, 0) == -1
    finally:
        lib.ps_dev_free(d_set)
        lib.ps_dev_free(d_out)
