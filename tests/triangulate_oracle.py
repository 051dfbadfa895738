"""Float64 numpy restatement of ps_triangulate_tracks (include/popsift_b200_triangulate.h) for the tests; nothing in the
package imports it.

Every expression follows the header's order of operations with elementwise float64 operations, and the lane-strided sums
of the device (a partial sum per lane of a warp, then an xor butterfly) are restated as such, so the oracle is meant to
give the device's bits.  The sample hash is verify_oracle's.  It also plants scenes: posed cameras around a point cloud,
noisy observations and outliers."""
from __future__ import annotations

import math

import numpy as np

import verify_oracle as vo

OK, TOO_FEW_OBS, NO_HYPOTHESIS, TOO_FEW_INLIERS, SMALL_ANGLE = range(5)
POINT_DTYPE = np.dtype([("X", "<f8", 3), ("error", "<f4"), ("angle", "<f4"), ("n_inliers", "<i4"), ("status", "<i4")])


# ---- the per-observation math (k_triangulate.h) ----------------------------------------------------------------------

def centre(R, t):
    """C = -R^T t, (..., 3)"""
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    return np.stack([-(R[..., 0, k] * t[..., 0] + R[..., 1, k] * t[..., 1] + R[..., 2, k] * t[..., 2]) for k in range(3)], -1)


def unit(v):
    """v / sqrt(v.v) componentwise; (ok, u)"""
    n = np.sqrt(v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])
    ok = (n > 0) & np.isfinite(n)
    with np.errstate(invalid="ignore", divide="ignore"):
        return ok, v / n[..., None]


def direction(cam, R, x, y):
    """(ok, d): the unit ray R^T ((x - cx) / fx, (y - cy) / fy, 1) of pixels (x, y); cam (..., 4) float32 fx, fy, cx, cy"""
    c = np.asarray(cam, np.float32).astype(np.float64)
    R = np.asarray(R, np.float64)
    xn = (np.asarray(x, np.float32).astype(np.float64) - c[..., 2]) / c[..., 0]
    yn = (np.asarray(y, np.float32).astype(np.float64) - c[..., 3]) / c[..., 1]
    u = np.stack([R[..., 0, k] * xn + R[..., 1, k] * yn + R[..., 2, k] for k in range(3)], -1)
    return unit(u)


def dot3(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def hypothesis(Ca, da, Cb, db, cos_min):
    """(ok, X): the two-ray rule (pose_two_rays) with t = C_a - C_b and the midpoint"""
    w = Ca - Cb
    aa, bb, ab = dot3(da, da), dot3(db, db), dot3(da, db)
    at, bt = dot3(da, w), dot3(db, w)
    det = aa * bb - ab * ab
    with np.errstate(invalid="ignore", divide="ignore"):
        sa = (ab * bt - at * bb) / det
        sb = (aa * bt - ab * at) / det
    ok = (det > 1e-12 * (aa * bb)) & (sa > 0) & (sb > 0) & (ab <= cos_min)
    X = 0.5 * ((Ca + sa[..., None] * da) + (Cb + sb[..., None] * db))
    return ok, X


def residual(cam, R, t, X, x, y, jac=False):
    """(front, ex, ey[, Jx, Jy]) of pixels (x, y) under points X (broadcast)"""
    c = np.asarray(cam, np.float32).astype(np.float64)
    fx, fy, cx, cy = c[..., 0], c[..., 1], c[..., 2], c[..., 3]
    x = np.asarray(x, np.float32).astype(np.float64)
    y = np.asarray(y, np.float32).astype(np.float64)
    Xc = [R[..., r, 0] * X[..., 0] + R[..., r, 1] * X[..., 1] + R[..., r, 2] * X[..., 2] + t[..., r] for r in range(3)]
    front = Xc[2] > 0
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        iz = 1.0 / Xc[2]
        p, q = Xc[0] * iz, Xc[1] * iz
        ex = fx * p + cx - x
        ey = fy * q + cy - y
        if not jac:
            return front, ex, ey
        Jx = np.stack([fx * ((R[..., 0, k] - p * R[..., 2, k]) * iz) for k in range(3)], -1)
        Jy = np.stack([fy * ((R[..., 1, k] - q * R[..., 2, k]) * iz) for k in range(3)], -1)
    return front, ex, ey, Jx, Jy


def error2(cam, R, t, X, x, y):
    """(front, e2)"""
    front, ex, ey = residual(cam, R, t, X, x, y)
    with np.errstate(invalid="ignore", over="ignore"):
        return front, ex * ex + ey * ey


def step(S):
    """(ok, dX) of the Gauss-Newton sums S (J^T J as 00 01 02 11 12 22, then -J^T e) by Cramer's rule"""
    a, b, c, d, e, f, g0, g1, g2 = (float(v) for v in S[:9])
    m0, m1, m2 = d * f - e * e, b * f - e * c, b * e - d * c
    det = a * m0 - b * m1 + c * m2
    if not (det > 0.0) or not math.isfinite(det):
        return False, np.zeros(3)
    return True, np.array([(g0 * m0 - b * (g1 * f - e * g2) + c * (g1 * e - d * g2)) / det,
                           (a * (g1 * f - e * g2) - g0 * m1 + c * (b * g2 - g1 * c)) / det,
                           (a * (d * g2 - g1 * e) - b * (b * g2 - g1 * c) + g0 * m2) / det])


def warp_sum(v):
    """the device's lane-strided sum: v[j] goes to lane j % 32 in order, then an xor butterfly"""
    v = np.asarray(v, np.float64)
    lanes = np.zeros(32)
    for j in range(len(v)):
        lanes[j % 32] += v[j]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return float(lanes[0])


# ---- hypotheses ------------------------------------------------------------------------------------------------------

def exhaustive(L, n_samples):
    return L * (L - 1) // 2 <= n_samples


def hypothesis_pairs(L, n_samples, seed, track):
    """(valid (H,), a (H,), b (H,)): every pair in lexicographic order, or n_samples drawn pairs (smaller position first)"""
    if exhaustive(L, n_samples):
        a, b = np.triu_indices(L, 1)
        return np.ones(len(a), bool), a, b
    valid, idx = vo.samples(seed, track, np.arange(n_samples), L, 2)
    return valid, np.minimum(idx[:, 0], idx[:, 1]).astype(np.int64), np.maximum(idx[:, 0], idx[:, 1]).astype(np.int64)


# ---- one track -------------------------------------------------------------------------------------------------------

def triangulate_track(x, y, cam, R, t, t_index, max_error, min_angle, min_views, n_samples, refine_iters, seed, info=False):
    """The track's (record, mask (L,) uint8, err (L,) float32[, info]).  x, y (L,) float32 pixels; cam (L, 4) float32;
    R (L, 3, 3), t (L, 3) double: member k's camera.  info: the hypothesis counts, the winner, e2 of every hypothesis
    and member, and the refinement's trail, for the tests' exclusions."""
    L = len(x)
    thr2 = float(np.float32(max_error)) * float(np.float32(max_error))
    cos_min = math.cos(float(np.float32(min_angle)) * (3.141592653589793 / 180.0))
    rec = np.zeros((), POINT_DTYPE)
    mask = np.zeros(L, np.uint8)
    err = np.full(L, np.inf, np.float32)
    inf = dict(counts=None, win=-1, e2=None, thr2=thr2, cos_min=cos_min)
    R = np.asarray(R, np.float64).reshape(L, 3, 3)
    t = np.asarray(t, np.float64).reshape(L, 3)
    cam = np.asarray(cam, np.float32).reshape(L, 4)
    if L < min_views:
        rec["status"] = TOO_FEW_OBS
        return (rec, mask, err, inf) if info else (rec, mask, err)
    C = centre(R, t)
    _, d = direction(cam, R, x, y)
    valid, a, b = hypothesis_pairs(L, n_samples, seed, t_index)
    ok, Xh = hypothesis(C[a], d[a], C[b], d[b], cos_min)
    ok &= valid
    front, e2 = error2(cam[None], R[None], t[None], Xh[:, None, :], np.asarray(x)[None], np.asarray(y)[None])
    inl = front & (e2 <= thr2)
    counts = np.where(ok, inl.sum(1), -1)
    inf.update(counts=counts, e2=np.where(front, e2, np.inf), hyp_ok=ok)
    if not ok.any():
        rec["status"] = NO_HYPOTHESIS
        return (rec, mask, err, inf) if info else (rec, mask, err)
    w = int(np.argmax(counts))              # first of the largest: ties to the smallest h
    bc = int(counts[w])
    X = Xh[w].copy()
    inf["win"] = w
    if refine_iters > 0:
        S0 = inl[w]

        def sums(Xq):
            fr, ex, ey, Jx, Jy = residual(cam, R, t, Xq[None], x, y, jac=True)
            m = S0 & fr
            z = lambda v: np.where(m, v, 0.0)   # noqa: E731
            S = [warp_sum(z(Jx[:, i] * Jx[:, j] + Jy[:, i] * Jy[:, j])) for i, j in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
            S += [-warp_sum(z(Jx[:, k] * ex + Jy[:, k] * ey)) for k in range(3)]
            S.append(warp_sum(z(ex * ex + ey * ey)) if not (S0 & ~fr).any() else math.inf)
            return np.array(S)

        Xr = X.copy()
        S = sums(Xr)
        trail = [S[9]]
        for _ in range(refine_iters):
            good, dX = step(S)
            if not good:
                break
            Xn = np.array([Xr[0] + dX[0], Xr[1] + dX[1], Xr[2] + dX[2]])
            Sn = sums(Xn)
            trail.append(Sn[9])
            if not (Sn[9] < S[9]):
                break
            Xr, S = Xn, Sn
        fr, e2r = error2(cam, R, t, Xr[None], x, y)
        rc = int((fr & (e2r <= thr2)).sum())
        inf.update(trail=trail, refit_count=rc, refit_e2=np.where(fr, e2r, np.inf))
        if rc >= bc:
            X = Xr
    fr, e2f = error2(cam, R, t, X[None], x, y)
    inl_f = fr & (e2f <= thr2)
    mask[:] = inl_f
    with np.errstate(invalid="ignore"):
        err[:] = np.where(fr, np.sqrt(np.where(fr, e2f, 0.0)), np.inf).astype(np.float32)
    n_in = int(inl_f.sum())
    esum = warp_sum(np.where(inl_f, np.sqrt(np.where(fr, e2f, 0.0)), 0.0))
    _, U = unit(C - X[None])
    cmin = 2.0
    ii = np.nonzero(inl_f)[0]
    if len(ii) > 1:
        Ui = U[ii]
        G = Ui[:, None, 0] * Ui[None, :, 0] + Ui[:, None, 1] * Ui[None, :, 1] + Ui[:, None, 2] * Ui[None, :, 2]
        cmin = float(G[np.triu_indices(len(ii), 1)].min())
    rec["X"] = X
    rec["n_inliers"] = n_in
    rec["error"] = np.float32(esum / n_in) if n_in else np.float32(0)
    rec["angle"] = np.float32(math.degrees(math.acos(min(1.0, max(-1.0, cmin))))) if n_in > 1 else np.float32(0)
    rec["status"] = TOO_FEW_INLIERS if n_in < min_views else (SMALL_ANGLE if cmin > cos_min else OK)
    inf.update(final_e2=np.where(fr, e2f, np.inf), cmin=cmin)
    return (rec, mask, err, inf) if info else (rec, mask, err)


def triangulate(feats, cams, poses, start, members, max_error=4.0, min_angle=1.5, min_views=2, n_samples=256, refine_iters=10, seed=0,
                info=False):
    """All tracks: feats[i] (n_i, 2) float32 pixels of set i, cams (n_sets, 4), poses a list of (R, t); start / members
    as ps_triangulate_tracks takes them.  Returns (points, mask, err[, infos])"""
    n_feat = [len(f) for f in feats]
    off = np.concatenate([[0], np.cumsum(n_feat)]).astype(np.int64)
    allxy = np.concatenate([np.asarray(f, np.float32).reshape(-1, 2) for f in feats]) if feats else np.zeros((0, 2), np.float32)
    members = np.asarray(members, np.int64)
    sets = np.searchsorted(off, members, side="right") - 1
    Rs = np.stack([np.asarray(p[0], np.float64) for p in poses]) if poses else np.zeros((0, 3, 3))
    ts = np.stack([np.asarray(p[1], np.float64) for p in poses]) if poses else np.zeros((0, 3))
    cams = np.asarray(cams, np.float32).reshape(-1, 4)
    T = len(start) - 1
    pts = np.zeros(T, POINT_DTYPE)
    mask = np.zeros(len(members), np.uint8)
    err = np.full(len(members), np.inf, np.float32)
    infos = []
    for k in range(T):
        s0, s1 = int(start[k]), int(start[k + 1])
        st = sets[s0:s1]
        xy = allxy[members[s0:s1]]
        r = triangulate_track(xy[:, 0], xy[:, 1], cams[st], Rs[st], ts[st], k, max_error, min_angle, min_views, n_samples, refine_iters,
                              seed, info=info)
        pts[k], mask[s0:s1], err[s0:s1] = r[0], r[1], r[2]
        if info:
            infos.append(r[3])
    return (pts, mask, err, infos) if info else (pts, mask, err)


# ---- planted scenes --------------------------------------------------------------------------------------------------

def look_at(centre_, target, rng):
    """(R, t) of a camera at centre_ looking at target, with a random roll"""
    z = np.asarray(target, np.float64) - centre_
    z /= np.linalg.norm(z)
    up = rng.normal(size=3)
    x = np.cross(up, z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ centre_


def project(cam, R, t, X):
    Xc = X @ R.T + t
    return np.stack([cam[0] * Xc[:, 0] / Xc[:, 2] + cam[2], cam[1] * Xc[:, 1] / Xc[:, 2] + cam[3]], 1)


def planted_scene(rng, n_cams, lengths, noise=0.5, outliers=0.2, radius=10.0, spread=2.0, shift=(0.0, 0.0, 0.0), sets=None):
    """Cameras on a sphere of `radius` around a cloud of `spread`, one track per entry of `lengths` (that many distinct
    cameras), pixel noise, and a fraction of outlier observations (uniform over the image).  The world frame is translated
    by `shift`.  `sets`, when given, is one array of distinct cameras per track (lengths must be their sizes): the cameras
    that see it, so that a test can set every camera's observation count exactly; the observations are then drawn in bulk.
    Returns dict(feats, cams, poses, start, members, Xtrue, outlier (members,) bool)."""
    shift = np.asarray(shift, np.float64)
    cams, poses = _cameras(rng, n_cams, radius, shift)
    T = len(lengths)
    X = rng.normal(scale=spread / 2, size=(T, 3)) + shift
    if sets is not None:
        return _planted_sets(rng, cams, poses, X, lengths, noise, outliers, sets)
    obs_set, obs_xy, obs_track, outl = [], [], [], []
    for k, L in enumerate(lengths):
        cs = np.sort(rng.choice(n_cams, size=int(L), replace=False))
        for c in cs:
            uv = project(cams[c].astype(np.float64), poses[c][0], poses[c][1], X[k:k + 1])[0] + rng.normal(scale=noise, size=2)
            o = rng.random() < outliers
            if o:
                uv = rng.uniform([0, 0], [640, 480])
            obs_set.append(c); obs_xy.append(uv); obs_track.append(k); outl.append(o)
    return _pack(cams, poses, X, lengths, obs_set, obs_xy, outl)


def _cameras(rng, n_cams, radius, shift):
    cams = np.zeros((n_cams, 4), np.float32)
    poses = []
    for i in range(n_cams):
        c = rng.normal(size=3); c *= radius / np.linalg.norm(c)
        R, t = look_at(c + shift, shift + rng.normal(scale=0.2, size=3), rng)
        f = rng.uniform(600, 1400)
        cams[i] = (f, f * rng.uniform(0.98, 1.02), rng.uniform(300, 340), rng.uniform(230, 250))
        poses.append((R, t))
    return cams, poses


def _planted_sets(rng, cams, poses, X, lengths, noise, outliers, sets):
    """planted_scene's observations for the given cameras of every track, drawn in bulk"""
    sets = [np.sort(np.asarray(s, np.int64)) for s in sets]
    assert [len(s) for s in sets] == [int(L) for L in lengths] and all(len(np.unique(s)) == len(s) for s in sets)
    obs_set = np.concatenate(sets) if sets else np.zeros(0, np.int64)
    obs_track = np.repeat(np.arange(len(sets)), [len(s) for s in sets])
    uv = np.zeros((len(obs_set), 2))
    for c in np.unique(obs_set):
        m = obs_set == c
        uv[m] = project(cams[c].astype(np.float64), poses[c][0], poses[c][1], X[obs_track[m]])
    uv += rng.normal(scale=noise, size=uv.shape)
    outl = rng.random(len(uv)) < outliers
    uv[outl] = rng.uniform([0, 0], [640, 480], size=(int(outl.sum()), 2))
    return _pack(cams, poses, X, lengths, obs_set, uv, outl)


def _pack(cams, poses, X, lengths, obs_set, obs_xy, outl):
    n_cams = len(cams)
    obs_set = np.asarray(obs_set, np.int64)
    obs_xy = np.asarray(obs_xy, np.float32).reshape(-1, 2)
    order = np.lexsort((np.arange(len(obs_set)), obs_set))     # features of each set in observation order
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order))
    n_feat = np.bincount(obs_set, minlength=n_cams)
    off = np.concatenate([[0], np.cumsum(n_feat)])
    feats = [obs_xy[order[off[i]:off[i + 1]]] for i in range(n_cams)]
    members = rank.astype(np.int32)          # observations are already grouped by track, ascending by set
    start = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    return dict(feats=feats, cams=cams, poses=poses, start=start, members=members, Xtrue=X, outlier=np.asarray(outl, bool))
