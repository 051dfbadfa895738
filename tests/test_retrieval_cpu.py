"""Image retrieval without a GPU: the new header's exports, the initial draw and the score chain of the host program built
on the kernels' own headers, the oracle's top-m rules, and the retrieval kernels' SASS."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import retrieval_oracle as ro
from popsift_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_exe():
    from popsift_b200 import build as B
    B.build()
    return B.RETRIEVAL_HOST


def host_scores(exe, v, plain):
    v = np.ascontiguousarray(v, np.float32)
    with tempfile.TemporaryDirectory() as d:
        inp, out = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(inp, "wb") as f:
            f.write(np.int32(v.shape[0]).tobytes() + np.int32(v.shape[1]).tobytes() + v.tobytes())
        r = subprocess.run([exe, "score", inp, out, "1" if plain else "0"], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        return np.fromfile(out, np.float32).reshape(len(v), len(v))


def test_header_exports():
    """every ps_*( of popsift_b200_retrieval.h is exported and listed in api.RETRIEVAL_EXPORTS, apart from the others"""
    hdr = open(os.path.join(ROOT, "include", "popsift_b200_retrieval.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    decl = sorted(set(re.findall(r"\b(ps_\w+)\(", hdr)))
    assert decl == sorted(api.RETRIEVAL_EXPORTS)
    assert not set(api.RETRIEVAL_EXPORTS) & set(api.EXPORTS)
    assert not set(api.RETRIEVAL_EXPORTS) & set(api.GUIDED_EXPORTS)
    lib = api.load_library()
    for name in api.RETRIEVAL_EXPORTS:
        assert hasattr(lib, name)


@pytest.mark.parametrize("seed", [0, 1, 0xFFFFFFFFFFFFFFFF])
@pytest.mark.parametrize("k", [1, 7, 64, 1024])
def test_draw_matches_header(host_exe, seed, k):
    """the oracle's initial draw equals the host program on k_verify_sample.h, for N = k, k + 1 and 10^5"""
    for N in (k, k + 1, 10 ** 5):
        r = subprocess.run([host_exe, "draw", str(seed), str(N), str(k)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr
        got = [int(v) for v in r.stdout.split()]
        want = ro.draw(seed, N, k)
        assert got == want
        assert len(set(got)) == k and all(0 <= v < N for v in got)


@pytest.mark.parametrize("dim", [4, 36, 128, 1028])
def test_score_chain_is_a_plain_fmaf_loop(host_exe, dim):
    """retrieve_score (k_retrieval.h) is bit for bit a scalar std::fmaf loop, and symmetric"""
    rng = np.random.default_rng(dim)
    v = rng.normal(size=(40, dim)).astype(np.float32)
    v[3] = v[5]
    v[7, : dim // 2] = 0.0
    a, b = host_scores(host_exe, v, False), host_scores(host_exe, v, True)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(a.view(np.uint32), a.T.view(np.uint32))
    # and it is not the float64 product rounded once: the order is a property of the result
    assert not np.array_equal(a, (v.astype(np.float64) @ v.T.astype(np.float64)).astype(np.float32))


def test_oracle_topm_rules():
    S = np.array([[0, 2, 2, np.nan, 5],
                  [2, 0, -0.0, 0.0, np.nan],
                  [2, -0.0, 0, -np.inf, 1],
                  [np.nan, 0.0, -np.inf, 0, np.nan],
                  [5, np.nan, 1, np.nan, 0]], np.float32)
    nbr, sc = ro.topm(S, 4)
    assert nbr[0].tolist() == [4, 1, 2, 3]                 # ties to the lower j, NaN last
    assert nbr[1].tolist() == [0, 2, 3, 4]                 # -0 and +0 tie: lower j first
    assert nbr[2].tolist() == [0, 4, 1, 3]                 # -inf above nothing but NaN
    assert nbr[3].tolist() == [1, 2, 0, 4]                 # NaNs ranked by j
    assert np.isnan(sc[3, 2]) and sc[2, 3] == -np.inf
    nbr, sc = ro.topm(S[:2, :2], 3)
    assert nbr.tolist() == [[1, -1, -1], [0, -1, -1]] and (sc[:, 1:] == -np.inf).all()
    assert ro.topm(np.zeros((1, 1), np.float32), 2)[0].tolist() == [[-1, -1]]
    assert ro.select_pairs([[1, 2], [0, -1], [0, 1]]) == [(0, 1), (0, 2), (1, 2)]
    assert api.select_pairs([[1, 2], [0, -1], [0, 1]]) == [(0, 1), (0, 2), (1, 2)]


def test_oracle_vlad_rules():
    rng = np.random.default_rng(0)
    x = rng.random((50, 128)).astype(np.float32)
    cb = x[:4].copy()
    a = ro.assign(x, cb)
    assert a[:4].tolist() == [0, 1, 2, 3]
    v = ro.vlad(x, cb, a)
    assert v.shape == (512,) and abs(np.linalg.norm(v) - 1) < 1e-12
    assert not ro.vlad(x[:0], cb, a[:0]).any()
    # equidistant centroids: the lower index wins
    assert ro.assign(np.zeros((1, 128), np.float32), np.stack([np.eye(128)[0], np.eye(128)[1]]).astype(np.float32)).tolist() == [0]


def test_shipped_sass_retrieval_kernels_no_local_memory():
    """the retrieval kernels keep everything in registers and shared memory; the score kernel loads its tiles by TMA"""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lib = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_hist
    k = sass_hist.histogram(lib)
    names = [n for n in k if re.search(r"vlad_\w+_kernel|retrieve_\w+_kernel", n)]
    assert len(names) == 8, names
    for n in names:
        c = k[n]
        assert c["LDL"] == 0 and c["STL"] == 0, n
    score = [n for n in names if "retrieve_score_kernel" in n]
    assert len(score) == 1 and k[score[0]]["UTMALDG"] > 0 and k[score[0]]["FFMA"] > 0
