"""ps_relative_pose_batch on the GPU against tests/pose_oracle.py and planted truth."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import pose_oracle as po          # noqa: E402
import verify_oracle as vo        # noqa: E402
from popsift_b200 import api      # noqa: E402
from popsift_b200.synth import make_frame   # noqa: E402
import tracks_oracle as to        # noqa: E402

pytestmark = pytest.mark.gpu

THR = 2.0
PS_ERR_ARG = -1


def _scenes(seed, sizes, fracs):
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(sizes):
        out.append(po.planted_pose(rng, n, fracs[i % len(fracs)], 0.3))
    return out


@pytest.fixture(scope="module")
def planted():
    sizes = [0, 4, 5, 6, 50, 1000, 20000] + [1000] * 40 + [300] * 120 + [2000] * 130
    fr = [1.0, 0.8, 0.6, 0.5, 0.4]
    sc = _scenes(1, sizes, fr)
    res, taps = api.relative_pose_correspondences([s[0] for s in sc], [s[1] for s in sc], threshold=THR, n_samples=1024, seed=7,
                                                  points=True, taps=True)
    return sc, res, taps


def test_planted_accuracy(planted):
    sc, res, _ = planted
    worst = dict(rot=0.0, tr=0.0, keep=1.0, leak=0.0, front=1.0)
    where = {}
    for p, ((corr, cams, R, t, inl, err, clean), r) in enumerate(zip(sc, res)):
        n = len(corr)
        if n < 5:
            assert r.n_inliers == 0 and r.n_front == 0 and not r.mask.any() and not r.E.any() and not r.R.any()
            continue
        if inl.sum() < 100:
            continue
        worst["rot"] = max(worst["rot"], po.rot_angle(r.R, R))
        worst["tr"] = max(worst["tr"], po.dir_angle(r.t, t))
        good = inl & (err < THR / 2)
        bad = (~inl) & (err > 2 * THR)
        worst["keep"] = min(worst["keep"], (r.mask[good] & 1).mean())
        if bad.any():
            worst["leak"] = max(worst["leak"], (r.mask[bad] & 1).mean())
        worst["front"] = min(worst["front"], r.n_front / max(r.n_inliers, 1))
        ang = po.rot_angle(r.R, R)
        if ang >= worst["rot"]:
            where["rot"] = (p, n, int(inl.sum()), ang, po.dir_angle(r.t, t), r.n_inliers)
    print("worst", worst, "worst-rotation pair (p, n, planted inliers, rot, dir, n_inliers)", where.get("rot"))
    # worst over the pairs with >= 100 planted inliers, H100: rotation 0.83 deg, translation direction 1.68 deg, kept clear
    # inliers 0.986, accepted clear outliers 0.046, n_front / n_inliers 0.972.  The worst rotation is pair 96 (300 rows, 240
    # inliers, f = 2 200 px, sideways motion): its winner has 241 inliers and the refit is kept only at >= 241, while the
    # inlier count is flat over almost a degree under that narrow field of view (DESIGN.md 4.12)
    assert worst["rot"] < 1.0
    assert worst["tr"] < 2.0
    assert worst["keep"] >= 0.98
    assert worst["leak"] <= 0.05
    assert worst["front"] >= 0.95


def test_outputs_consistent(planted):
    sc, res, _ = planted
    for (corr, cams, R, t, inl, err, clean), r in zip(sc, res):
        if r.n_inliers == 0:
            continue
        Rr = r.R.astype(np.float64)
        assert abs(np.linalg.det(Rr) - 1) < 1e-5 and np.abs(Rr @ Rr.T - np.eye(3)).max() < 1e-5
        assert abs(np.linalg.norm(r.t) - 1) < 1e-6
        E = po.essential(Rr, r.t.astype(np.float64))
        assert np.abs(E - r.E).max() < 1e-6
        F = po.pixels_f(E, cams[0], cams[1])
        assert np.abs(F - r.F).max() < 1e-5
        m = r.mask
        assert set(np.unique(m).tolist()) <= {0, 1, 3}
        assert r.n_inliers == int((m & 1).sum()) and r.n_front == int(((m & 2) != 0).sum())
        rows, t2 = po.calibrate(corr, cams[0], cams[1], THR)
        # bit 0: the float64 Sampson test under the output E, outside a band around the threshold
        s2 = vo.sampson(r.E.astype(np.float64), rows) ** 2
        clear = np.abs(s2 - t2) > 1e-3 * t2
        assert ((s2 < t2)[clear] == ((m & 1) != 0)[clear]).all()
        # bit 1: cheirality under the output R, t, except rows within a relative 1e-6 of a cut
        det, ref, dl, dr, X = po.triangulate(Rr, r.t, rows)
        front = (det > 1e-12 * ref) & (dl > 0) & (dr > 0)
        # per row, relative to its own scale: the depths against the row's |t| / sqrt(det / (a.a b.b)) (1 for |t| = 1)
        with np.errstate(invalid="ignore", divide="ignore"):
            dscale = 1.0 / np.sqrt(np.maximum(det, 0) / ref)
            near = ~np.isfinite(dl) | ~np.isfinite(dr) | (np.abs(det - 1e-12 * ref) <= 1e-6 * ref) | \
                (np.abs(dl) <= 1e-6 * dscale) | (np.abs(dr) <= 1e-6 * dscale)
        in0 = (m & 1) != 0
        assert ((front & in0)[~near] == ((m & 2) != 0)[~near]).all()
        pts = r.points
        b1 = (m & 2) != 0
        assert (pts[~b1] == 0).all()
        assert np.allclose(pts[b1, :3], X[b1], rtol=1e-4, atol=1e-4 * np.abs(X[b1]).max()) and (pts[b1, 3] == 1).all()


def test_taps(planted):
    sc, res, (tc, tm) = planted
    ns = 1024
    n_valid = n_slots = n_stable = n_agree = 0
    for p, ((corr, cams, R, t, inl, err, clean), r) in enumerate(zip(sc, res)):
        n = len(corr)
        if n < 5:
            assert (tc[p] == -1).all()
            continue
        valid, idx = vo.samples(7, p, np.arange(ns), n, 5)
        cnt = tc[p].reshape(ns, 10)
        assert (cnt[~valid] == -1).all()
        n_valid += int((cnt >= 0).sum())
        n_slots += cnt[valid].size
        rows, t2 = po.calibrate(corr, cams[0], cams[1], THR)
        # every valid tap's E nearly satisfies its sample's epipolar constraints (pins the hash on the device)
        for s in np.nonzero(valid)[0][:16]:
            q = rows[idx[s]].astype(np.float64)
            xl = np.hstack([q[:, :2], np.ones((5, 1))]); xr = np.hstack([q[:, 2:], np.ones((5, 1))])
            for j in np.nonzero(cnt[s] >= 0)[0]:
                E = tm[p, 10 * s + j].astype(np.float64)
                assert np.abs((xr * (xl @ E.T)).sum(1)).max() < 5e-2
        # counts: the float64 recount, outside the band
        for h in np.nonzero(tc[p] >= 0)[0][:8]:
            s2 = vo.sampson(tm[p, h].astype(np.float64), rows) ** 2
            lo, hi = int((s2 < t2 * (1 - 1e-3)).sum()), int((s2 < t2 * (1 + 1e-3)).sum())
            assert lo <= tc[p, h] <= hi
        # on stable samples the valid taps are the oracle's solution set (float32 E against float64)
        for s in np.nonzero(valid)[0][:24]:
            S, stable = po.five_point(rows[idx[s]].astype(np.float64), info=True)
            if not stable:
                continue
            taps_s = [tm[p, 10 * s + j].astype(np.float64) for j in np.nonzero(cnt[s] >= 0)[0]]
            n_stable += 1
            n_agree += po.same_set(taps_s, S, 1e-4)
    frac = n_valid / max(n_slots, 1)
    print("valid slot fraction", frac, "stable samples", n_stable, "agreeing with the oracle", n_agree)
    # measured on the H100: valid slot fraction 0.451; 7 054 of 7 060 stable samples agree at 1e-4
    assert 0.3 < frac < 0.6
    assert n_stable > 1000 and n_agree >= 0.99 * n_stable


def test_refine_and_tie_rule():
    sc = _scenes(2, [500] * 12, [0.7])
    corrs, cams = [s[0] for s in sc], [s[1] for s in sc]
    r0, (tc, tm) = api.relative_pose_correspondences(corrs, cams, threshold=THR, n_samples=128, seed=3, refine=False, taps=True)
    r1, (tc1, _) = api.relative_pose_correspondences(corrs, cams, threshold=THR, n_samples=128, seed=3, refine=True, taps=True)
    assert (tc == tc1).all()
    for p in range(len(sc)):
        w = vo.select(tc[p])
        rows, t2 = po.calibrate(corrs[p], cams[p][0], cams[p][1], THR)
        k, Rc, tcand, _ = po.choose(tm[p, w].astype(np.float64), rows[(vo.sampson(tm[p, w].astype(np.float64), rows) ** 2) < t2])
        assert po.rot_angle(r0[p].R, Rc) < 1e-3
        assert r1[p].n_inliers >= tc[p, w] - 2     # the refit is kept only when it keeps as many inliers (float rounding of E)


def test_determinism_and_independence():
    sc = _scenes(3, [800, 40, 3000, 0, 700], [0.6])
    corrs, cams = [s[0] for s in sc], [s[1] for s in sc]
    a = api.relative_pose_correspondences(corrs, cams, threshold=THR, n_samples=200, seed=5, points=True)
    b = api.relative_pose_correspondences(corrs, cams, threshold=THR, n_samples=200, seed=5, points=True)
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert np.array_equal(np.asarray(u), np.asarray(v))
    p = 2
    lone = [np.zeros((0, 4), np.float32)] * len(corrs)
    lone[p] = corrs[p]
    c = api.relative_pose_correspondences(lone, cams, threshold=THR, n_samples=200, seed=5, points=True)
    for u, v in zip(a[p], c[p]):
        assert np.array_equal(np.asarray(u), np.asarray(v))


def test_large_ragged():
    rng = np.random.default_rng(4)
    P = 10001
    base = _scenes(5, [60, 7, 200, 0, 33], [0.7])
    corrs = [base[i % 5][0] for i in range(P)]
    cams = [base[i % 5][1] for i in range(P)]
    big = api.relative_pose_correspondences(corrs, cams, threshold=THR, n_samples=32, seed=9)
    for p in (0, 1, 2, 3, 4, 5000, 10000):
        lone = [np.zeros((0, 4), np.float32)] * (p + 1)
        lone[p] = corrs[p]
        small = api.relative_pose_correspondences(lone, cams[:p + 1], threshold=THR, n_samples=32, seed=9)[p]
        for u, v in zip(big[p], small):
            assert np.array_equal(np.asarray(u), np.asarray(v))


def test_argument_errors():
    lib = api.load_library()
    bufs = api._DevBuffers(lib)
    try:
        d_corr, d_out, d_mask, d_pts = bufs.alloc(160), bufs.alloc(128), bufs.alloc(16), bufs.alloc(160)
        start = np.zeros(1, np.int32); n = np.full(1, 10, np.int32)
        cams = np.array([[1000, 1000, 500, 400]] * 2, np.float32)
        prm = api._pose_params(2.0, 16)

        def call(P=1, corr=d_corr, st=start, nc=n, cm=cams, pr=prm, out=d_out, mask=d_mask, pts=None, taps=None):
            return lib.ps_relative_pose_batch(0, P, corr, st.ctypes.data if st is not None else None,
                                              nc.ctypes.data if nc is not None else None, cm.ctypes.data if cm is not None else None,
                                              C.byref(pr) if pr is not None else None, out, mask, pts, taps)
        assert call() == 0 and call(pts=d_pts) == 0
        assert call(P=0, st=None, nc=None, cm=None) == 0
        host = np.zeros(64, np.uint8)
        for kw in (dict(P=-1), dict(pr=None), dict(pr=api._pose_params(2.0, 0)), dict(pr=api._pose_params(2.0, 65537)),
                   dict(pr=api._pose_params(float("nan"), 16)), dict(pr=api._pose_params(0.0, 16)),
                   dict(pr=api.PsPoseParams(16, 2.0, 2, 0, 0)), dict(st=None), dict(nc=None), dict(cm=None),
                   dict(st=np.full(1, -1, np.int32)), dict(nc=np.full(1, -1, np.int32)),
                   dict(out=host.ctypes.data), dict(pts=host.ctypes.data), dict(corr=host.ctypes.data), dict(mask=host.ctypes.data),
                   dict(corr=d_corr + 4)):
            assert call(**kw) == PS_ERR_ARG, kw
        for bad in ((0, 1000, 500, 400), (-5, 1000, 500, 400), (1000, float("inf"), 500, 400), (1000, 1000, float("nan"), 400),
                    (1000, 1000, 500, float("inf"))):
            cm = cams.copy(); cm[1] = bad
            assert call(cm=cm) == PS_ERR_ARG, bad
    finally:
        bufs.free()


# ---- end to end: a rendered piecewise-planar scene through extraction, pose, guided matching and tracks ----

W, H = 1280, 960
CAMS = [np.array([1000.0, 1000.0, 640.0, 480.0], np.float32), np.array([1150.0, 1150.0, 630.0, 490.0], np.float32)]


def _rot(axis, deg):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    th = np.radians(deg)
    return np.cos(th) * np.eye(3) + np.sin(th) * vo._skew(a) + (1 - np.cos(th)) * np.outer(a, a)


# planes n . X = d in the left frame, each with its own texture and in-plane axes
PLANES = [((1.0, 0.0, 0.0), -2.2), ((0.0, 1.0, 0.0), 1.3), ((-0.35, 0.2, 1.0), 7.0), ((-1.0, 0.0, 0.25), -1.4)]


def _cast(cam, R, t, x, y):
    """(Z in the left frame, texture value) of the rays through pixels (x, y) of a camera with X_cam = R X_l + t"""
    d = np.linalg.solve(po.K(cam), np.stack([x, y, np.ones_like(x)]))
    o, dirs = -R.T @ t, R.T @ d
    best = np.full(x.shape, np.inf)
    val = np.zeros(x.shape)
    Z = np.zeros(x.shape)
    for k, (n, dist) in enumerate(PLANES):
        n = np.asarray(n) / np.linalg.norm(n)
        dist = dist / np.linalg.norm(PLANES[k][0])
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = (dist - n @ o) / (n @ dirs)
        lam = np.where(np.isfinite(lam) & (lam > 0), lam, np.inf)
        hit = lam < best
        P = o[:, None] + np.where(hit, lam, 0.0) * dirs
        e1 = np.cross(n, [0.0, 0.0, 1.0] if abs(n[2]) < 0.9 else [0.0, 1.0, 0.0]); e1 /= np.linalg.norm(e1)
        e2 = np.cross(n, e1)
        tex = _TEX[k]
        a, b = (e1 @ P) * 230.0, (e2 @ P) * 230.0
        a0, b0 = np.floor(a), np.floor(b)
        fa, fb = a - a0, b - b0
        S = tex.shape[0]
        i0, j0 = np.mod(b0, S).astype(np.int64), np.mod(a0, S).astype(np.int64)
        i1, j1 = (i0 + 1) % S, (j0 + 1) % S
        v = (tex[i0, j0] * (1 - fa) + tex[i0, j1] * fa) * (1 - fb) + (tex[i1, j0] * (1 - fa) + tex[i1, j1] * fa) * fb
        val = np.where(hit, v, val)
        Z = np.where(hit, P[2], Z)
        best = np.where(hit, lam, best)
    return Z, val


_TEX = [make_frame(1536, 1536, 40 + k).astype(np.float64) for k in range(len(PLANES))]
R_TRUE = _rot((0.2, 1.0, 0.1), 4.0)
C_TRUE = np.array([0.6, 0.05, 0.2])              # right camera centre in the left frame
T_TRUE = -R_TRUE @ C_TRUE


@pytest.fixture(scope="module")
def rendered():
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    imgs = []
    for cam, R, t in ((CAMS[0], np.eye(3), np.zeros(3)), (CAMS[1], R_TRUE, T_TRUE)):
        _, v = _cast(cam, R, t, x.ravel(), y.ravel())
        imgs.append(np.clip(np.rint(v), 0, 255).astype(np.uint8).reshape(H, W))
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=W, max_height=H, slots=1)
    sets = [ps.enqueue(W, H, im).getDev() for im in imgs]
    yield imgs, sets
    ps.uninit()


def test_end_to_end_rendered(rendered, tmp_path):
    imgs, sets = rendered
    pairs = [(0, 1)]
    (two, in_rows, front_rows), = api.relative_poses(sets, pairs, CAMS, threshold=THR, n_samples=1024, seed=1, points=True)
    rot, tdir = po.rot_angle(two.R, R_TRUE), po.dir_angle(two.t, T_TRUE)
    # depths of the in-front rows against the ray-cast truth at their left keypoints, after scaling by the baseline
    lib = api.load_library()
    bufs = api._DevBuffers(lib)
    try:
        _, dev, rows, d_match, d_corr, d_src, start, n_corr = api._matched_rows(lib, bufs, sets, pairs, None, 0, False, None, False)
        prm = api._pose_params(THR, 1024, 1, True)
        d_out, d_mask, tv, mask, pts = api._pose_dev(lib, bufs, dev, d_corr, start, n_corr, api._c_cameras(CAMS), prm, points=True)
        n = int(n_corr[0])
        corr = bufs.download(d_corr, (rows, 4), np.float32)[:n]
        src = bufs.download(d_src, rows, np.int32)
        match = bufs.download(d_match, (rows, 3), np.int32)
        # relative_poses is this chain: same record, mask, points and rows
        for f in ("E", "F", "R", "t"):
            assert np.array_equal(getattr(two, f), tv[0][f]), f
        assert (two.n_inliers, two.n_front) == (int(tv[0]["n_inliers"]), int(tv[0]["n_front"]))
        assert np.array_equal(two.mask, mask[:n]) and np.array_equal(two.points, pts[:n])
        assert np.array_equal(in_rows, src[:n][(mask[:n] & 1) != 0]) and np.array_equal(front_rows, src[:n][(mask[:n] & 2) != 0])
        # guided matching on d_out[0].F, straight from the device record (byte offset 36), no host copy
        descs = api._desc_sets(lib, bufs, sets, dev)
        d_g = api._match_guided_dev(lib, bufs, sets, descs, pairs, d_out + 36, 1, THR, 0, False)
        d_gc, _, _, g_n = api._correspondences_dev(lib, bufs, sets, pairs, d_g, dev)
        gcorr = bufs.download(d_gc, (rows, 4), np.float32)[:int(g_n[0])]
        # the pose mask as the tracks' inlier mask, against the explicit bit-0 edges
        n_feat = [s.getFeatureCount() for s in sets]
        n_desc = [s.getDescriptorCount() for s in sets]
        c_corr = np.ascontiguousarray(n_corr, np.int32)
        via_mask = api._tracks_dev(lib, bufs, n_feat, 2, lambda of, st, mem, cnt: lib.ps_tracks_from_matches(
            dev, 2, (C.c_int32 * 2)(*n_feat), (C.c_void_p * 2)(*[s.getReverseMap() for s in sets]), (C.c_int32 * 2)(*n_desc), 1,
            api._c_pairs(pairs), d_match, d_src, c_corr.ctypes.data, d_mask, 2, of, st, mem, C.byref(cnt)))
    finally:
        bufs.free()
    b1 = (two.mask & 2) != 0
    Zt, _ = _cast(CAMS[0], np.eye(3), np.zeros(3), corr[b1, 0].astype(np.float64), corr[b1, 1].astype(np.float64))
    depth_err = np.median(np.abs(two.points[b1, 2] * np.linalg.norm(T_TRUE) - Zt) / Zt)
    gs = vo.sampson(two.F.astype(np.float64), gcorr)
    print("rendered: corr", n, "inliers", two.n_inliers, "front", two.n_front, "rot", rot, "dir", tdir, "median depth err", depth_err,
          "guided", len(gcorr), "max guided Sampson", gs.max() if len(gs) else None)
    # measured on the H100: 3 122 correspondences, 2 911 inliers, 2 910 in front, rotation 0.20 deg, direction 1.18 deg,
    # median depth error 3.5 %, 3 471 guided correspondences with the largest Sampson distance 1.9989 px
    assert two.n_inliers > 500
    assert rot < 0.5
    assert tdir < 3.0
    assert two.n_front >= 0.9 * two.n_inliers
    assert depth_err < 0.05
    assert len(gcorr) > two.n_inliers // 2 and (gs < THR * 1.001).all()
    rev = [s.to_host()[2] for s in sets]
    e = to.chain_edges(pairs, n_desc, n_feat, match, src, n_corr, mask & 1, rev)
    off = to.offsets(n_feat)
    se = np.searchsorted(off, e, side="right") - 1
    via_edges = api.build_tracks(n_feat, np.stack([se[:, 0], e[:, 0] - off[se[:, 0]], se[:, 1], e[:, 1] - off[se[:, 1]]], 1), 2)
    assert len(via_mask.start) > 100
    for f in via_mask._fields:
        a, b = getattr(via_mask, f), getattr(via_edges, f)
        if f == "track_of":
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
        else:
            assert np.array_equal(a, b), f
    # the C++ API on the same frames against the C ABI
    from popsift_b200 import build as B
    files = []
    for k, im in enumerate(imgs):
        f = tmp_path / ("v%d.raw" % k)
        im.tofile(f)
        files.append(str(f))
    args = [B.POSE_CHECK, str(W), str(H)] + files + ["%.9g" % v for c in CAMS for v in c]
    out = subprocess.run(args, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
