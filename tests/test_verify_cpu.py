"""Geometric verification without a GPU: the RANSAC sample hash against the kernel's own __host__ __device__ function
(compiled for the host), self-checks of the float64 oracle (tests/verify_oracle.py), and the C ABI's layout."""
import ctypes as C
import os
import subprocess

import numpy as np

import verify_oracle as vo
from popsift_b200 import api


def test_sample_hash_matches_kernel_function(tmp_path):
    """10^5 (seed, pair, sample, n) records, m = 4 and 7, n from m (every draw must be distinct) to 2^31 - 1: the oracle's
    indices and validity equal those of psb::verify_sample, the function the solve kernel calls."""
    from popsift_b200 import build as B
    B.build()
    rng = np.random.default_rng(11)
    N = 100_000
    rec = np.zeros(N, dtype=[("seed", "<u8"), ("p", "<i4"), ("s", "<i4"), ("n", "<u4"), ("m", "<i4")])
    rec["seed"] = rng.integers(0, 2 ** 63, N, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, N).astype(np.uint64)
    rec["seed"][:1000] = 0
    rec["p"] = rng.integers(0, 1 << 20, N)
    rec["s"] = rng.integers(0, 65536, N)
    rec["m"] = np.where(rng.random(N) < 0.5, 4, 7)
    kind = rng.integers(0, 4, N)
    rec["n"] = np.select([kind == 0, kind == 1, kind == 2], [rec["m"], rng.integers(rec["m"], 12), rng.integers(12, 200_000)],
                         rng.integers(200_000, 2 ** 31 - 1, N))
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    rec.tofile(inp)
    r = subprocess.run([B.VERIFY_SAMPLE_CHECK, str(inp), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("OK"), r.stdout + r.stderr
    got = np.fromfile(out, dtype=np.uint32).reshape(N, 8)
    for m in (4, 7):
        sel = rec["m"] == m
        ok, idx = vo.samples(rec["seed"][sel], rec["p"][sel], rec["s"][sel], rec["n"][sel], m)
        assert np.array_equal(ok, got[sel, 0] == 1)
        assert np.array_equal(idx, got[sel, 1:1 + m])
    # n == m: 64 draws usually find them all, but not always; the sample is then invalid on both sides
    small = rec["n"] == rec["m"]
    assert small.sum() > 10_000 and 0 < (got[small, 0] == 0).sum() < small.sum()
    assert (got[rec["n"] > 1000, 0] == 1).all()


def test_sample_indices_distinct_and_in_range():
    ok, idx = vo.samples(5, np.arange(2000) // 100, np.arange(2000) % 100, 10, 7)
    assert ok.mean() > 0.99
    for row in idx[ok]:
        assert len(set(row.tolist())) == 7 and row.max() < 10


def test_oracle_recovers_planted_homography():
    rng = np.random.default_rng(1)
    corr, H, inl, _ = vo.planted_homography(rng, 200, 1.0, sigma=0.0)
    s, cl, cr = vo.normalization(corr)
    pn = vo.normalize(corr, s, cl, cr)
    Hn = vo.solve_h4(pn[:4])
    assert Hn is not None
    assert np.allclose(vo.to_pixels(0, Hn, s, cl, cr), H, rtol=1e-3, atol=1e-6)
    assert np.allclose(vo.to_pixels(0, vo.refit(0, pn), s, cl, cr), H, rtol=1e-3, atol=1e-6)
    assert vo.transfer_error(H, corr).max() < 1e-3


def test_oracle_recovers_planted_fundamental():
    rng = np.random.default_rng(2)
    corr, F, inl, _, clean = vo.planted_fundamental(rng, 300, 1.0, sigma=0.0)
    s, cl, cr = vo.normalization(clean)
    pn = vo.normalize(clean, s, cl, cr)
    Fs = [vo.to_pixels(1, Fn, s, cl, cr) for Fn in vo.solve_f7(pn[:7])]
    assert 1 <= len(Fs) <= 3
    assert min(np.abs(G - F).max() for G in Fs) < 1e-6
    G = vo.to_pixels(1, vo.refit(1, pn), s, cl, cr)
    assert np.abs(G - F).max() < 1e-6
    assert vo.sampson(F, clean).max() < 1e-6


def test_errors_scale_by_s_under_common_normalization():
    """transfer error and Sampson distance in normalised coordinates are exactly s times the pixel ones"""
    rng = np.random.default_rng(3)
    for model in (0, 1):
        if model == 0:
            corr, M, _, _ = vo.planted_homography(rng, 500, 0.6)
        else:
            corr, M, _, _, _ = vo.planted_fundamental(rng, 500, 0.6)
        s, cl, cr = vo.normalization(corr)
        pn = vo.normalize(corr, s, cl, cr)
        Tl, Tr = vo.xform(s, cl), vo.xform(s, cr)
        Mn = Tr @ M @ np.linalg.inv(Tl) if model == 0 else np.linalg.inv(Tr).T @ M @ np.linalg.inv(Tl)
        e, en = vo.error(model, M, corr), vo.error(model, Mn, pn)
        fin = np.isfinite(e)
        assert np.allclose(en[fin], s * e[fin], rtol=1e-9, atol=1e-12)
        # the normalised points of both images together have mean distance sqrt(2) from their centroids
        d = (np.linalg.norm(pn[:, :2], axis=1).sum() + np.linalg.norm(pn[:, 2:], axis=1).sum()) / (2 * len(pn))
        assert abs(d - np.sqrt(2)) < 1e-9


def test_tie_rule():
    assert vo.select([3, 5, 5, -1]) == 1
    assert vo.select([-1, -1]) == -1
    assert vo.select([-1, 0, 0]) == 1
    assert vo.select([]) == -1


def test_collinear_samples_rejected():
    p = np.array([[0, 0, 0, 0], [1, 1, 1, 2], [2, 2, 3, 1], [0, 1, 5, 5]], np.float64)
    assert vo.solve_h4(p) is None
    p[:, 2:] = [[0, 0], [1, 0], [0, 1], [1, 1]]
    p[:, :2] = [[0, 0], [1, 0], [0, 1], [1, 1]]
    assert vo.solve_h4(p) is not None


def test_abi_layout_and_exports():
    assert C.sizeof(api.PsVerifyParams) == 24
    assert api.PsVerifyParams.seed.offset == 16
    lib = api.load_library()
    for name in ("ps_match_correspondences", "ps_verify_batch"):
        assert name in api.EXPORTS and hasattr(lib, name)
    assert len(api.EXPORTS) == len(set(api.EXPORTS)) == 41
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "popsift_b200.h")).read()
    assert "PS_GEOM_HOMOGRAPHY = 0, PS_GEOM_FUNDAMENTAL = 1" in hdr
