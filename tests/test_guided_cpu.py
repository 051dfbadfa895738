"""Guided matching without a GPU: the kernels' eligibility test (k_guided.h, compiled for the host) against the float64
predicate, its empty cases, the masked 2-NN oracle's row rules, the new header's exports and the guided kernels' SASS."""
import os
import re
import shutil
import sys

import numpy as np
import pytest

import guided_oracle as go
from popsift_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mask_exe():
    from popsift_b200 import build as B
    B.build()
    return B.GUIDED_MASK


def _cases(kind, rng, n_models=48, n=150, w=3840, h=2160):
    """(model, t, left points, right points) with 4K pixel coordinates; the right points of a homography are the mapped
    left points plus noise of about t, so that many diagonal cases lie near the threshold"""
    for _ in range(n_models):
        t = float(np.exp(rng.uniform(np.log(1.0), np.log(1000.0))))
        pl = rng.uniform([0, 0], [w, h], (n, 2))
        if kind == go.HOMOGRAPHY:
            M = go.random_homography(rng, w, h)
            hl = np.c_[pl, np.ones(n)] @ M.T
            pr = hl[:, :2] / hl[:, 2:3] + rng.normal(0, t, (n, 2))
        else:
            M = go.random_fundamental(rng, w, h)
            pr = pl + rng.normal(0, 40, (n, 2))
        yield M.astype(np.float32), np.float32(t), pl.astype(np.float32), pr.astype(np.float32)


@pytest.mark.parametrize("kind", [go.HOMOGRAPHY, go.FUNDAMENTAL])
def test_mask_matches_float64_outside_band(mask_exe, kind):
    """about 10^6 (model, point pair) cases per model kind: the float32 mask equals the float64 predicate wherever the
    float64 error is more than 1e-3 t^2 away from t^2 (the band test_verify.py uses)"""
    rng = np.random.default_rng(5 + kind)
    total = near = elig = 0
    for M, t, pl, pr in _cases(kind, rng):
        got = go.mask_exact(kind, t, M, pl, pr, mask_exe)
        err = go.sq_err64(kind, M.astype(np.float64), pl.astype(np.float64), pr.astype(np.float64))
        t2 = float(t) ** 2
        far = np.abs(err - t2) > 1e-3 * t2
        assert np.array_equal(got[far], (err < t2)[far])
        total += err.size
        near += int((~far).sum())
        elig += int(got.sum())
    assert total > 10 ** 6
    assert 0.01 * total < elig < 0.99 * total          # both outcomes well represented
    assert near < 1e-3 * total


@pytest.mark.parametrize("kind", [go.HOMOGRAPHY, go.FUNDAMENTAL])
def test_zero_and_nan_models_give_empty_masks(mask_exe, kind):
    rng = np.random.default_rng(3)
    pl = rng.uniform(0, 4000, (64, 2)).astype(np.float32)
    pr = np.r_[pl, rng.uniform(0, 4000, (64, 2))].astype(np.float32)
    for M in (np.zeros(9, np.float32), np.full(9, np.nan, np.float32), np.r_[np.eye(3).ravel()[:8], np.nan].astype(np.float32)):
        assert not go.mask_exact(kind, 1e6, M, pl, pr, mask_exe).any()
    # NaN points (the kernels' padding rows) are never eligible either, even under H = I and a huge threshold
    eye = np.eye(3, dtype=np.float32).ravel()
    m = go.mask_exact(kind, 1e6, eye, np.r_[pl[:4], [[np.nan, np.nan]]], np.r_[pr[:4], [[np.nan, 1.0]]], mask_exe)
    assert not m[4].any() and not m[:, 4].any()
    if kind == go.HOMOGRAPHY:
        assert m[:4, :4].all()


def test_guided_rows_row_rules():
    """the masked 2-NN: nothing eligible -> (0, 0, 0); exactly one j -> (j, 0, 1); all eligible -> the unguided rows"""
    import match_oracle as mo
    rng = np.random.default_rng(1)
    l = rng.random((5, 128)).astype(np.float32)
    r = rng.random((9, 128)).astype(np.float32)
    none = go.guided_rows(l, r, np.zeros((5, 9), bool))
    assert (none == 0).all()
    one = np.zeros((5, 9), bool)
    one[np.arange(5), [3, 0, 8, 5, 5]] = True
    assert go.guided_rows(l, r, one).tolist() == [[3, 0, 1], [0, 0, 1], [8, 0, 1], [5, 0, 1], [5, 0, 1]]
    assert np.array_equal(go.guided_rows(l, r, np.ones((5, 9), bool)), mo.best_two(mo.sq_dist_matrix(l, r)))
    assert go.guided_rows(l, r[:0], np.zeros((5, 0), bool)).tolist() == [[0, 0, 0]] * 5


def test_header_exports():
    """every ps_*( of popsift_b200_guided.h is exported by the library and listed in api.GUIDED_EXPORTS, apart from
    api.EXPORTS (the entry points of popsift_b200.h)"""
    hdr = open(os.path.join(ROOT, "include", "popsift_b200_guided.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    decl = sorted(set(re.findall(r"\b(ps_\w+)\(", hdr)))
    assert decl == sorted(api.GUIDED_EXPORTS)
    assert not set(api.GUIDED_EXPORTS) & set(api.EXPORTS)
    lib = api.load_library()
    for name in api.GUIDED_EXPORTS:
        assert hasattr(lib, name)


def test_shipped_sass_guided_kernels_use_tma_and_mma():
    """the float guided kernel issues float warpgroup MMAs (HGMMA), the 8-bit one integer ones (IGMMA), both with TMA"""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    lib = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_hist
    k = sass_hist.histogram(lib)
    fl = {n: c for n, c in k.items() if "match_tc_guided_kernel" in n}
    u8 = {n: c for n, c in k.items() if "match_u8_guided_kernel" in n}
    assert len(fl) == 2 and len(u8) == 2, (list(fl), list(u8))           # homography and fundamental instantiations
    for n, c in fl.items():
        assert c["HGMMA"] > 0 and c["UTMALDG"] > 0 and c["IGMMA"] == 0, n
    for n, c in u8.items():
        assert c["IGMMA"] > 0 and c["UTMALDG"] > 0 and c["HGMMA"] == 0, n
