"""Geometric verification on the GPU (ps_match_correspondences / ps_verify_batch, api.verify_pairs, popsift::verifyPairs):
planted models, the float64 oracle (tests/verify_oracle.py) on the kernels' own hypothesis taps, the final mask,
determinism, the correspondence gather, an end-to-end run on synth.affine_set, large and ragged batches, argument errors
and the C++ API."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import verify_oracle as vo
from popsift_b200 import api
from popsift_b200.synth import affine_set, make_frame

pytestmark = pytest.mark.gpu

# points whose squared error is within this relative distance of t^2 may be classified either way.  Scoring runs in float32
# on normalised points, and the pixel model a tap or the output reports is a second float32 rounding: with image
# coordinates near 1000 the sums behind an error of a few pixels cancel to about 1e-3 of their terms, so the two
# roundings can move e^2 by a few 1e-4 of t^2 (one point in a 300-point pair was measured beyond 1e-4 on an H100).
BAND = 1e-3


def _band_ok(mask, err, t):
    """mask equals err < t outside the band around t^2"""
    e2, t2 = err.astype(np.float64) ** 2, t * t
    clear = np.abs(e2 - t2) > BAND * t2
    return np.array_equal(mask[clear], (e2 < t2)[clear])


def _count_bounds(err, t):
    e2, t2 = err.astype(np.float64) ** 2, t * t
    return int((e2 < t2 * (1 - BAND)).sum()), int((e2 < t2 * (1 + BAND)).sum())


def _corners_err(H, Ht, w=1920, h=1080):
    c = np.array([[0, 0, 1], [w, 0, 1], [0, h, 1], [w, h, 1]], np.float64)
    a, b = c @ np.asarray(H, np.float64).T, c @ np.asarray(Ht, np.float64).T
    return np.abs(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:]).max()


def _planted(model, sizes, fracs, reps, seed):
    rng = np.random.default_rng(seed)
    out = []
    for n in sizes:
        for f in fracs:
            for _ in range(reps if n < 10_000 else 2):
                if model == 0:
                    corr, M, inl, err = vo.planted_homography(rng, n, f)
                    out.append((corr, M, inl, err, None))
                else:
                    out.append((*vo.planted_fundamental(rng, n, f),))
    return out


@pytest.mark.parametrize("model", [0, 1])
def test_planted_models(model):
    """About 400 pairs per model in one call, n from 0 to 20 000, inlier fractions 1.0 .. 0.25 (H) / 1.0 .. 0.5 (F), 0.3 px
    noise, t = 2 px.  Where at least 40 (H) / 400 (F) planted inliers exist: every inlier with true error < t/2 is in the
    mask (F: at least 98 % of them), no outlier with true error > 2t is (F: at most 2 % of them), H maps the image corners within 1 px of the
    truth, F has Sampson distance < 2 px on the noise-free inliers.  (An F from 40 noisy inliers was measured at 0.70 px, and with it two outliers lay
    within t of their estimated epipolar lines: a point-to-line test cannot reject those.)  Below the sample size the result
    is zero."""
    t = 2.0
    fracs = [1.0, 0.75, 0.5, 0.25] if model == 0 else [1.0, 0.75, 0.5]
    data = _planted(model, [0, 3, 4, 6, 7, 8, 50, 1000, 20_000], fracs, 12 if model == 0 else 16, 100 + model)
    res = api.verify_correspondences([d[0] for d in data], model=model, threshold=t, n_samples=4096, seed=5)
    m = vo.SAMPLE_SIZE[model]
    checked = 0
    for (corr, M, inl, err, clean), (G, cnt, mask) in zip(data, res):
        n = len(corr)
        assert cnt == int(mask.sum())
        if n < m:
            assert cnt == 0 and not G.any() and not mask.any()
            continue
        if inl.sum() < 40:
            continue
        if model == 1 and inl.sum() < 400:
            continue
        checked += 1
        near = inl & (err < t / 2)
        far = ~inl & (err > 2 * t)
        if model == 0:
            assert mask[near].all(), (n, inl.mean())
            assert not mask[far].any(), (n, inl.mean())
            assert _corners_err(G, M) < 1.0, (n, inl.mean(), _corners_err(G, M))
        else:
            # the F winner is often the minimal-sample model (see the refit rule), and a point-to-line test cannot
            # separate everything: up to 2 such outliers of 228 were measured, and some near inliers were missed at 49 %
            assert mask[near].mean() >= 0.98, (n, inl.mean(), float(mask[near].mean()))
            assert mask[far].sum() <= max(2, 0.02 * far.sum()), (n, inl.mean(), int(mask[far].sum()))
            # 0.5 px where the refit was kept; a minimal-sample winner (refit rejected for losing an inlier) was measured at
            # 1.52 px on 749 inliers
            assert vo.sampson(G, clean[inl]).max() < 2.0, (n, inl.mean())
    assert checked > (60 if model == 0 else 40)


def _algebraic(model, M, pts):
    """sine of the angle between x_r and H x_l (H), or |x_r^T F x_l| / (|x_r| |F x_l|) (F): small for the sample's own points
    even where the pixel error is not (points near a homography's line at infinity)"""
    xl = np.hstack([pts[:, :2], np.ones((len(pts), 1))]).astype(np.float64)
    xr = np.hstack([pts[:, 2:], np.ones((len(pts), 1))]).astype(np.float64)
    a = xl @ np.asarray(M, np.float64).T
    if model == 0:
        return np.linalg.norm(np.cross(xr, a), axis=1) / (np.linalg.norm(xr, axis=1) * np.linalg.norm(a, axis=1))
    return np.abs((xr * a).sum(1)) / (np.linalg.norm(xr, axis=1) * np.linalg.norm(a, axis=1))


def _stable(solve, pts_n, rel=1e-7, gain=5.0):
    """the oracle's rating of a sample: its solutions move by less than gain x rel (relative) when the points move by rel,
    so a float32 solve can match them to about 1e-6"""
    base = solve(pts_n)
    if base is None or len(base) == 0:
        return False
    rng = np.random.default_rng(0)
    for _ in range(3):
        alt = solve(pts_n * (1 + rel * rng.choice([-1.0, 1.0], pts_n.shape)))
        if alt is None or len(alt) != len(base):
            return False
        for B in base:
            B = B / np.linalg.norm(B)
            d = min(min(np.abs(A / np.linalg.norm(A) - B).max(), np.abs(A / np.linalg.norm(A) + B).max()) for A in alt)
            if d > gain * rel * np.abs(B).max():
                return False
    return True


# relative agreement (largest entry difference over the largest entry) of the float32 pixel tap models with the oracle's
# float64 solvers on well-conditioned samples, measured on an H100: H up to 2.5e-5, F up to 4.3e-5 (Gauss-Jordan null
# space and closed-form cubic against SVD null space and companion roots) -- above the 1e-6 first aimed for.
TAP_MODEL_TOL = {0: 1e-4, 1: 1e-4}


def _tap_run(model, refine, seed=9, n_samples=None):
    rng = np.random.default_rng(40 + model)
    corrs = []
    for n in (8, 50, 300, 7, 4):
        for f in (1.0, 0.6, 0.3):
            for _ in range(3):
                corrs.append(vo.planted_homography(rng, n, f)[0] if model == 0 else vo.planted_fundamental(rng, n, f)[0])
    ns = n_samples or (256 if model == 0 else 128)
    res, (tc, tm) = api.verify_correspondences(corrs, model=model, threshold=2.0, n_samples=ns, seed=seed, refine=refine, taps=True)
    return corrs, ns, res, tc, tm


@pytest.mark.parametrize("model", [0, 1])
def test_taps_against_oracle(model):
    """Every valid hypothesis fits the oracle-drawn sample points (algebraic residual < 5e-2, which pins the hash on the
    device) and its validity equals the oracle's; on the samples the oracle rates well-conditioned (_stable) every tap count
    equals the float64 recount under the tap model outside the band and the tap models equal the oracle's solvers within
    TAP_MODEL_TOL (F as a set of roots); the output follows the tie rule over the taps."""
    t = 2.0
    corrs, ns, res, tc, tm = _tap_run(model, refine=0)
    m, k = vo.SAMPLE_SIZE[model], vo.ROOTS[model]
    worst, compared = 0.0, 0
    for p, corr in enumerate(corrs):
        n = len(corr)
        ok, idx = vo.samples(9, np.full(ns, p), np.arange(ns), np.full(ns, n), m)
        counts = tc[p].reshape(ns, k)
        assert (counts[~ok] == -1).all()
        s, cl, cr = vo.normalization(corr)
        pn = vo.normalize(corr, s, cl, cr)
        for si in np.nonzero(ok)[0]:
            pts = corr[idx[si]]
            valid = counts[si] >= 0
            for j in np.nonzero(valid)[0]:
                Mg = tm[p, si * k + j].astype(np.float64)
                # a wrong sample point gives an angle of order 1e-1; ill-conditioned solutions were measured up to 7.1e-3
                assert _algebraic(model, Mg, pts).max() < 5e-2, (p, si, j)
            if model == 0:
                Hn = vo.solve_h4(pn[idx[si]])
                assert (Hn is None) == (not valid[0]), (p, si)
                if Hn is None or not _stable(lambda q: [vo.solve_h4(q)] if vo.solve_h4(q) is not None else None, pn[idx[si]]):
                    continue
                want = [vo.to_pixels(0, Hn, s, cl, cr)]
            else:
                want = [vo.to_pixels(1, F, s, cl, cr) for F in vo.solve_f7(pn[idx[si]])]
                if len(want) != valid.sum() or not _stable(vo.solve_f7, pn[idx[si]]):
                    continue
            got = [tm[p, si * k + j].astype(np.float64) for j in np.nonzero(valid)[0]]
            # the recount under the float32 pixel model agrees with the tally only where that model is well-conditioned
            # (an ill-conditioned H was measured 3 points apart)
            for j in np.nonzero(valid)[0]:
                Mg = tm[p, si * k + j].astype(np.float64)
                if model == 0:
                    w = np.hstack([corr[:, :2], np.ones((len(corr), 1))]) @ Mg[2]
                    if w.min() <= 0.05 * np.abs(w).max():
                        continue        # the line at infinity crosses the image: rounding of H decides near it
                lo, hi = _count_bounds(vo.error(model, Mg, corr), t)
                assert lo <= counts[si, j] <= hi, (p, si, j, lo, counts[si, j], hi)
            for W in want:
                d = min(np.abs(G - W).max() for G in got) / np.abs(W).max()
                worst = max(worst, d)
            compared += 1
        win = vo.select(tc[p])
        G, cnt, mask = res[p]
        if win < 0:
            assert cnt == 0 and not G.any()
        else:
            assert np.array_equal(G, tm[p, win]) and cnt == tc[p, win]
    print("taps model %d: %d samples compared, largest relative difference %.3g" % (model, compared, worst))
    assert compared > 500, compared
    assert worst < TAP_MODEL_TOL[model], worst


@pytest.mark.parametrize("model", [0, 1])
def test_final_mask_and_refit(model):
    """The mask is the float64 inlier test under the output model outside the band, n_inliers its sum; refine = 1 never
    ends below the winner's count, refine = 0 returns the winner's tap model itself."""
    t = 2.0
    for refine in (0, 1):
        corrs, ns, res, tc, tm = _tap_run(model, refine=refine)
        for p, corr in enumerate(corrs):
            G, cnt, mask = res[p]
            assert cnt == int(mask.sum())
            win = vo.select(tc[p])
            if win < 0:
                continue
            assert _band_ok(mask, vo.error(model, G, corr), t), p
            if refine:
                assert cnt >= tc[p, win]
            else:
                assert np.array_equal(G, tm[p, win]) and cnt == tc[p, win]


def test_determinism():
    corrs, ns, res, tc, tm = _tap_run(1, refine=1)
    corrs2, _, res2, tc2, tm2 = _tap_run(1, refine=1)
    assert np.array_equal(tc, tc2) and np.array_equal(tm.view(np.uint32), tm2.view(np.uint32))
    for a, b in zip(res, res2):
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and a[1] == b[1] and np.array_equal(a[2], b[2])
    _, _, _, tc3, _ = _tap_run(1, refine=1, seed=10)
    assert not np.array_equal(tc, tc3)


def _extract_sets(images, w, h, norm_multi=0):
    cfg = api.Config()
    if norm_multi:
        cfg.setNormalizationMultiplier(norm_multi)
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    sets = [ps.enqueue(w, h, im).getDev() for im in images]
    return ps, sets


def _gather_numpy(hosts, pairs, matches):
    out = []
    for (l, r), rows in zip(pairs, matches):
        fl, _, rl = hosts[l]
        fr, _, rr = hosts[r]
        corr, src = [], []
        for i in range(len(rows)):
            b, _, acc = rows[i]
            if acc != 1 or len(rr) == 0:
                continue
            dup = any(i - d >= 0 and rows[i - d][2] == 1 and rl[i - d] == rl[i] and rr[rows[i - d][0]] == rr[b] for d in (1, 2, 3))
            if dup:
                continue
            corr.append((fl["x"][rl[i]], fl["y"][rl[i]], fr["x"][rr[b]], fr["y"][rr[b]]))
            src.append(i)
        out.append((np.array(corr, np.float32).reshape(-1, 4), np.array(src, np.int32)))
    return out


def test_correspondence_gather():
    """ps_match_correspondences equals a numpy restatement on float and u8 match rows, on rows with many duplicate
    (feature, feature) pairs, with an empty set and self pairs."""
    frames = [im for im, _ in affine_set(480, 360)[:2]] + [np.zeros((360, 480), np.uint8)]
    ps, sets = _extract_sets(frames, 480, 360, norm_multi=9)
    assert sets[0].getDescriptorCount() > 100 and sets[2].getDescriptorCount() == 0
    hosts = [s.to_host() for s in sets]
    pairs = [(0, 1), (1, 0), (0, 0), (2, 0), (0, 2), (1, 1), (2, 2)]
    rng = np.random.default_rng(3)
    fake = []
    for l, r in pairs:
        nl, nr = sets[l].getDescriptorCount(), sets[r].getDescriptorCount()
        rows = np.zeros((nl, 3), np.int32)
        if nr:
            rows[:, 0] = rng.integers(0, min(nr, 6), nl)          # few right rows: many repeats of the same right Feature
            rows[:, 2] = rng.random(nl) < 0.7
        fake.append(rows)
    for matches in (api.match_pairs(sets, pairs), api.match_pairs_u8(sets, pairs), fake):
        corr, src = api.match_correspondences(sets, pairs, matches)
        want = _gather_numpy(hosts, pairs, matches)
        for p in range(len(pairs)):
            assert np.array_equal(corr[p], want[p][0]), pairs[p]
            assert np.array_equal(src[p], want[p][1]), pairs[p]
    assert sum(len(c) for c in api.match_correspondences(sets, pairs, fake)[0]) < sum(int(f[:, 2].sum()) for f in fake)
    ps.uninit()


# inlier fractions of verify_pairs on affine_set (t = 2 px, 1024 samples, seed 1), measured on an H100 80GB HBM3:
# 375/409, 266/314, 492/508, 353/423, 143/208; asserted about 0.07 below
AFFINE_MIN_FRACTION = {1: 0.85, 2: 0.78, 3: 0.90, 4: 0.77, 5: 0.62}
# Corner accuracy.  The single refit is kept only when it loses no inlier; on k = 1, 2, 3 it loses 2 or 3 (a float64 refit of
# the same inliers: 373 < 375, 263 < 266, 489 < 492) and the minimal-sample winner stays, 1.95 / 2.02 / 2.24 px from A_k at
# the corners (the float64 refit would be 0.15 / 0.20 / 0.08 px).  The extraction's feature order differs from process to
# process, which reorders the correspondences and so the samples: over six runs the corner errors ranged 0.22 .. 2.84 px
# (ps_verify_batch itself gave identical bytes in three processes on identical input).  Asserted with a margin:
AFFINE_MAX_CORNER_PX = 4.0


def test_affine_set_end_to_end():
    """Extract synth.affine_set in MatchingMode, verify_pairs (0, k), k = 1..5, with a homography: the recovered H is within
    AFFINE_MAX_CORNER_PX of the known A_k at the corners, and the inlier fractions stay above the measured bounds."""
    data = affine_set()
    ps, sets = _extract_sets([im for im, _ in data], 800, 640)
    pairs = [(0, k) for k in range(1, 6)]
    out = api.verify_pairs(sets, pairs, model="homography", threshold=2.0, n_samples=1024, seed=1)
    matches = api.match_pairs(sets, pairs)
    corr, src = api.match_correspondences(sets, pairs, matches)
    for (_, k), (G, cnt, rows), c, sr in zip(pairs, out, corr, src):
        A = np.vstack([data[k][1], [0, 0, 1.0]])
        err = _corners_err(G, A, 800, 640)
        frac = cnt / max(len(c), 1)
        print("affine k=%d: corner error %.3f px, %d / %d inliers (%.3f)" % (k, err, cnt, len(c), frac))
        assert err < AFFINE_MAX_CORNER_PX, (k, err)
        assert frac >= AFFINE_MIN_FRACTION[k], (k, frac)
        assert len(rows) == cnt and set(rows.tolist()) <= set(sr.tolist())
    ps.uninit()


def test_large_and_ragged_batch():
    """10 000 pairs of 200 correspondences (60 % inliers) and one pair of 200 000 (30 %) in one call, against the planted
    truth: the masks hold every inlier with true error < t/2 and no outlier beyond 2t; the corners are within 1.5 px (largest
    of the 10 001 measured on an H100: 1.27 px, 99.9th percentile 0.59 px)."""
    rng = np.random.default_rng(77)
    data = [vo.planted_homography(rng, 200, 0.6) for _ in range(10_000)]
    data.insert(5000, vo.planted_homography(rng, 200_000, 0.3))
    res = api.verify_correspondences([d[0] for d in data], model="homography", threshold=2.0, n_samples=256, seed=3)
    bad = 0
    for (corr, H, inl, err), (G, cnt, mask) in zip(data, res):
        assert cnt == int(mask.sum())
        ok = _corners_err(G, H) < 1.5 and mask[inl & (err < 1.0)].all() and not mask[~inl & (err > 4.0)].any()
        bad += not ok
    assert _corners_err(res[5000][0], data[5000][1]) < 1.0
    assert bad == 0, bad


def test_argument_errors():
    lib = api.load_library()
    bufs = api._DevBuffers(lib)
    try:
        d_corr, d_models, d_n, d_mask = bufs.alloc(64 * 16), bufs.alloc(36 * 2), bufs.alloc(8), bufs.alloc(64)
        start = np.array([0, 32], np.int32)
        n = np.array([32, 32], np.int32)

        def call(prm=None, P=2, corr=d_corr, st=start, nn=n, models=d_models, cnt=d_n, mask=d_mask, taps=None, **kw):
            prm = prm or api._verify_params(**kw)
            return lib.ps_verify_batch(0, P, corr, st.ctypes.data, nn.ctypes.data, C.byref(prm), models, cnt, mask, taps)

        host = np.zeros(64, np.float32)
        assert call() == 0
        assert call(P=0) == 0
        assert call(prm=api.PsVerifyParams(2, 16, 2.0, 1, 0)) == -1
        for thr in (0.0, -1.0, float("nan"), float("inf")):
            assert call(threshold=thr) == -1
        for ns in (0, 65537, -5):
            assert call(n_samples=ns) == -1
        assert call(n_samples=65536, threshold=1.0, model="homography", P=1) == 0
        assert call(prm=api.PsVerifyParams(0, 16, 2.0, 2, 0)) == -1
        assert call(P=-1) == -1
        assert call(nn=np.array([32, -1], np.int32)) == -1
        assert call(st=np.array([-1, 0], np.int32)) == -1
        assert call(corr=None) == -1 and call(mask=None) == -1 and call(models=None) == -1 and call(cnt=None) == -1
        assert call(corr=host.ctypes.data) == -1
        assert call(taps=C.byref(api.PsVerifyTaps(None, None))) == -1
        assert lib.ps_verify_batch(0, 1, d_corr, start.ctypes.data, n.ctypes.data, None, d_models, d_n, d_mask, None) == -1
        # correspondences: negative counts, set index out of range, null / host pointers
        c_n = (C.c_int32 * 1)(5)
        c_p = (C.c_int32 * 2)(0, 0)
        feat = (C.c_void_p * 1)(bufs.alloc(5 * 72))
        rev = (C.c_void_p * 1)(bufs.alloc(20))
        out_n = np.zeros(1, np.int32)
        m = bufs.alloc(60)
        assert lib.ps_match_correspondences(0, 1, feat, rev, c_n, 1, c_p, m, d_corr, d_n, out_n.ctypes.data) == 0
        assert lib.ps_match_correspondences(0, -1, feat, rev, c_n, 1, c_p, m, d_corr, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, feat, rev, (C.c_int32 * 1)(-1), 1, c_p, m, d_corr, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, feat, rev, c_n, 1, (C.c_int32 * 2)(0, 1), m, d_corr, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, feat, rev, c_n, 1, c_p, None, d_corr, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, feat, rev, c_n, 1, c_p, m, host.ctypes.data, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, (C.c_void_p * 1)(host.ctypes.data), rev, c_n, 1, c_p, m, d_corr, d_n, out_n.ctypes.data) == -1
        assert lib.ps_match_correspondences(0, 1, feat, rev, c_n, 1, c_p, m, d_corr, d_n, None) == -1
        assert lib.ps_match_correspondences(0, 0, None, None, None, 0, None, None, None, None, None) == 0
    finally:
        bufs.free()
    with pytest.raises(api.PopSiftError):
        api.verify_correspondences([np.zeros((10, 4), np.float32)], model="affine")


def test_cpp_verify_pairs(tmp_path):
    """popsift::verifyPairs (C++ API) equals ps_match_correspondences + ps_verify_batch on the same pairs."""
    from popsift_b200 import build as B
    exe = B.VERIFY_CHECK
    assert os.path.exists(exe), "build the product first (python -m popsift_b200.build)"
    data = affine_set(640, 480)
    files = []
    for k in (0, 1, 4):
        f = tmp_path / ("%d.raw" % k)
        data[k][0].tofile(f)
        files.append(str(f))
    out = subprocess.run([exe, "640", "480"] + files, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK 7"), out.stdout + out.stderr
    counts = [int(v) for v in out.stdout.split()[2:]]
    assert len(counts) == 14 and min(counts[:6]) > 50
