"""float64 numpy statement of ps_two_view_config_batch's contract (include/popsift_b200_twoview.h): the classification of
step 2, Kabsch's rotation and the rotation test of step 3, the homography's normalisation, sign and decomposition of step 4,
and the triangulation angle and lower median of step 6."""
import numpy as np

import pose_oracle as po

DEGENERATE, GENERAL, PLANAR, PANORAMIC, UNCALIBRATED = range(5)
NO_PARALLAX = 1e-9


def classify(n_e, n_f, n_h, min_inliers=15, min_ef_ratio=0.95, max_h_ratio=0.8, allow_h=True):
    """step 2; PLANAR stands for "planar or panoramic: step 3" """
    calibrated = n_e >= min_inliers and n_e >= min_ef_ratio * n_f
    m = n_e if calibrated else n_f
    if allow_h and n_h >= min_inliers and n_h > max_h_ratio * m:
        return PLANAR
    if calibrated:
        return GENERAL
    return UNCALIBRATED if n_f >= min_inliers else DEGENERATE


def rays(xy):
    """unit rays (x, y, 1) / |(x, y, 1)| of (n, 2) calibrated points"""
    h = np.hstack([np.asarray(xy, np.float64).reshape(-1, 2), np.ones((len(xy), 1))])
    return h / np.linalg.norm(h, axis=1, keepdims=True)


def kabsch_sum(rows):
    """B = sum b a^T over calibrated rows (x_l, y_l, x_r, y_r)"""
    r = np.asarray(rows, np.float64).reshape(-1, 4)
    return rays(r[:, 2:]).T @ rays(r[:, :2])


def kabsch(B):
    """the rotation U diag(1, 1, det(U V^T)) V^T of B = U S V^T"""
    U, _, Vt = np.linalg.svd(np.asarray(B, np.float64).reshape(3, 3))
    return U @ np.diag([1.0, 1.0, np.linalg.det(U @ Vt)]) @ Vt


def rotation_ok(R0, cam_r, rows, corr, threshold):
    """step 3's test per row: w = R0 (x^_l, y^_l, 1), w_z > 0 and the pixel transfer error below threshold"""
    r = np.asarray(rows, np.float64).reshape(-1, 4)
    c = np.asarray(corr, np.float32).astype(np.float64).reshape(-1, 4)
    w = np.hstack([r[:, :2], np.ones((len(r), 1))]) @ np.asarray(R0, np.float64).T
    fx, fy, cx, cy = (float(v) for v in np.asarray(cam_r, np.float32))
    with np.errstate(divide="ignore", invalid="ignore"):
        du = fx * (w[:, 0] / w[:, 2]) + cx - c[:, 2]
        dv = fy * (w[:, 1] / w[:, 2]) + cy - c[:, 3]
        return (w[:, 2] > 0) & (du * du + dv * dv < float(threshold) ** 2)


def h_calibrated(H, cam_l, cam_r):
    return np.linalg.inv(po.K(cam_r)) @ np.asarray(H, np.float64).reshape(3, 3) @ po.K(cam_l)


def h_svd(H):
    """singular values (descending) and right singular vectors (rows), each signed so that its first entry of largest
    magnitude is positive"""
    _, s, Vt = np.linalg.svd(np.asarray(H, np.float64).reshape(3, 3))
    V = Vt.copy()
    for k in range(3):
        if V[k, np.argmax(np.abs(V[k]))] < 0:
            V[k] = -V[k]
    return s, V


def h_normalise(H):
    s, _ = h_svd(H)
    return np.asarray(H, np.float64).reshape(3, 3) / s[1]


def h_signed(Hn, rows):
    """Hn negated when fewer than half of the rows have x_r^T Hn x_l > 0"""
    r = np.asarray(rows, np.float64).reshape(-1, 4)
    xl = np.hstack([r[:, :2], np.ones((len(r), 1))])
    xr = np.hstack([r[:, 2:], np.ones((len(r), 1))])
    npos = int(((xr * (xl @ Hn.T)).sum(1) > 0).sum())
    return -Hn if 2 * npos < len(r) else Hn


def h_decompose(H):
    """the four (R, t, n) of a normalised, signed H in the contract's order; [] without parallax"""
    H = np.asarray(H, np.float64).reshape(3, 3)
    s, V = h_svd(H)
    if not s[0] - s[2] > NO_PARALLAX * s[1]:
        return []
    d13 = s[0] ** 2 - s[2] ** 2
    a, b = np.sqrt(max(s[1] ** 2 - s[2] ** 2, 0.0) / d13), np.sqrt(max(s[0] ** 2 - s[1] ** 2, 0.0) / d13)
    v1, v2, v3 = V
    out = []
    for sg in (1.0, -1.0):
        u = a * v1 + sg * b * v3
        U = np.stack([v2, u, np.cross(v2, u)], 1)
        W = np.stack([H @ v2, H @ u, np.cross(H @ v2, H @ u)], 1)
        R = W @ U.T
        n = np.cross(v2, u)
        out.append((R, (H - R) @ n, n))
    return out + [(R, -t, -n) for R, t, n in out]


def prune(cands):
    """indices of the candidates with n_z > 0, in order"""
    return [k for k, (_, _, n) in enumerate(cands) if n[2] > 0]


def choose(cands, rows):
    """(index into cands, unit t, counts): the most rows in front under pose_front with (R, t / |t|), ties to the lower index"""
    counts = [int(po.in_front(R, t / np.linalg.norm(t), rows).sum()) for R, t, _ in cands]
    k = int(np.argmax(counts))
    return k, cands[k][1] / np.linalg.norm(cands[k][1]), counts


def angle(X, R, t):
    """degrees at X between the rays from 0 and from c = -R^T t"""
    X = np.asarray(X, np.float64).reshape(-1, 3)
    c = -np.asarray(R, np.float64).T @ np.asarray(t, np.float64)
    v = X - c
    return np.degrees(np.arctan2(np.linalg.norm(np.cross(X, v), axis=1), (X * v).sum(1)))


def lower_median(a):
    """rank floor((k - 1) / 2) of k values; 0 for none"""
    a = np.sort(np.asarray(a, np.float32))
    return np.float32(a[(len(a) - 1) // 2]) if len(a) else np.float32(0.0)


def random_rotation(rng, lo_deg=0.0, hi_deg=30.0):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    th = np.radians(rng.uniform(lo_deg, hi_deg))
    Kx = po.skew(ax)
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def planted_plane(rng, n, frac=1.0, sigma=0.3, w=1920, h=1080, rotation_only=False, f=None):
    """(corr (n, 4) float32, (cam_l, cam_r), R, t (unit, zero for rotation_only), plane normal (left frame), inlier flags,
    t / d (the calibrated homography is R + (t / d) n^T)):
    n points on one plane 4-10 units in front of the left camera (or any depths, under a pure rotation), seen by two
    cameras with different intrinsics, sigma pixels of noise on the inliers and uniform outliers"""
    f = f if f is not None else rng.uniform(800, 1600)
    cam_l = np.array([f, f * rng.uniform(0.98, 1.02), w / 2 + rng.uniform(-20, 20), h / 2 + rng.uniform(-20, 20)], np.float32)
    cam_r = np.array([f * rng.uniform(0.9, 1.1), f * rng.uniform(0.9, 1.1), w / 2 + rng.uniform(-20, 20), h / 2 + rng.uniform(-20, 20)],
                     np.float32)
    R = random_rotation(rng, 2.0, 12.0)
    nrm = np.array([rng.normal(0, 0.3), rng.normal(0, 0.3), 1.0])
    nrm /= np.linalg.norm(nrm)
    d = rng.uniform(4.0, 10.0)
    C = np.zeros(3) if rotation_only else rng.normal(size=3) * np.array([1.0, 0.5, 0.3])
    if not rotation_only:
        C *= rng.uniform(0.6, 1.5) / np.linalg.norm(C)
    t = -R @ C
    Kl, Kr = po.K(cam_l), po.K(cam_r)
    xl, X, k = [], [], 0
    while len(xl) < n and k < 100:
        k += 1
        px = np.stack([rng.uniform(0, w, 4 * n), rng.uniform(0, h, 4 * n), np.ones(4 * n)], 1)
        ray = px @ np.linalg.inv(Kl).T
        depth = d / (ray @ nrm) if not rotation_only else rng.uniform(2.0, 20.0, 4 * n)
        P = ray * depth[:, None]
        Pr = P @ R.T + t
        pr = Pr @ Kr.T
        ok = (depth > 0) & (Pr[:, 2] > 0.1)
        pr = pr[ok] / pr[ok][:, 2:3]
        ok2 = (pr[:, 0] >= 0) & (pr[:, 0] < w) & (pr[:, 1] >= 0) & (pr[:, 1] < h)
        xl += list(px[ok][ok2][:, :2])
        X += list(pr[ok2][:, :2])
    xl, xr = np.array(xl[:n]), np.array(X[:n])
    corr = np.hstack([xl, xr]) + rng.normal(0, sigma, (n, 4))
    inl = rng.random(n) < frac
    m = int((~inl).sum())
    corr[~inl] = np.stack([rng.uniform(0, w, m), rng.uniform(0, h, m), rng.uniform(0, w, m), rng.uniform(0, h, m)], 1)
    tu = np.zeros(3) if rotation_only else t / np.linalg.norm(t)
    return corr.astype(np.float32), (cam_l, cam_r), R, tu, nrm, inl, (np.zeros(3) if rotation_only else t / d)
