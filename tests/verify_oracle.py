"""Float64 numpy restatement of ps_verify_batch (include/popsift_b200.h) for the tests; nothing in the package imports it.

It restates the sample hash, the common-scale normalisation, the 4-point and 7-point solvers, both error functions, the
selection rule and the refit, and it plants homographies and fundamental matrices with known truth."""
from __future__ import annotations

import numpy as np

HOMOGRAPHY, FUNDAMENTAL = 0, 1
SAMPLE_SIZE = {HOMOGRAPHY: 4, FUNDAMENTAL: 7}
ROOTS = {HOMOGRAPHY: 1, FUNDAMENTAL: 3}
COLLINEAR_EPS = 1e-7
U64 = np.uint64


# ---- the sample hash -------------------------------------------------------------------------------------------------

def mix(z):
    """splitmix64's finaliser on uint64 arrays"""
    z = np.asarray(z, dtype=U64)
    with np.errstate(over="ignore"):
        z = z + U64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def sample_key(seed, p, s):
    seed = np.asarray(seed, dtype=U64)
    ps = (np.asarray(p, dtype=np.int64).astype(U64) << U64(32)) | np.asarray(s, dtype=np.int64).astype(U64)
    return mix(seed ^ mix(ps))


def draw(key, c, n):
    with np.errstate(over="ignore"):
        r = mix(np.asarray(key, dtype=U64) + U64(c))
    return ((r >> U64(32)) * np.asarray(n, dtype=U64)) >> U64(32)


def samples(seed, p, s, n, m):
    """(valid (N,), idx (N, m) uint32) of samples (p[i], s[i]) of pairs with n[i] correspondences, m indices each: draws in
    order, repeated indices skipped, at most 64 draws; idx keeps the draws made when the sample is invalid, zeros after"""
    p, s, n = np.broadcast_arrays(np.asarray(p), np.asarray(s), np.asarray(n))
    key = sample_key(np.broadcast_to(np.asarray(seed, dtype=U64), p.shape), p, s)
    N = p.size
    key, n = key.reshape(N), n.reshape(N)
    idx = np.zeros((N, m), np.uint32)
    got = np.zeros(N, np.int64)
    rows = np.arange(N)
    for c in range(64):
        v = draw(key, c, n).astype(np.uint32)
        dup = ((idx == v[:, None]) & (np.arange(m)[None, :] < got[:, None])).any(1)
        take = (~dup) & (got < m)
        idx[rows[take], got[take]] = v[take]
        got += take
    return got == m, idx


# ---- normalisation and errors ----------------------------------------------------------------------------------------

def normalization(corr):
    """(s, c_l, c_r) of the common-scale similarity: centroids, s = sqrt(2) / mean distance over both images"""
    c = np.asarray(corr, np.float64).reshape(-1, 4)
    if len(c) == 0:
        return 1.0, np.zeros(2), np.zeros(2)
    cl, cr = c[:, :2].mean(0), c[:, 2:].mean(0)
    d = (np.linalg.norm(c[:, :2] - cl, axis=1).sum() + np.linalg.norm(c[:, 2:] - cr, axis=1).sum()) / (2 * len(c))
    s = np.sqrt(2.0) / d if d > 0 else 1.0
    return s, cl, cr


def normalize(corr, s, cl, cr):
    c = np.asarray(corr, np.float64).reshape(-1, 4)
    return np.hstack([s * (c[:, :2] - cl), s * (c[:, 2:] - cr)])


def xform(s, c):
    return np.array([[s, 0, -s * c[0]], [0, s, -s * c[1]], [0, 0, 1.0]])


def transfer_error(H, corr):
    """||x_r - pi(H x_l)||, the one-sided transfer error (cv::findHomography's)"""
    c = np.asarray(corr, np.float64).reshape(-1, 4)
    x = np.hstack([c[:, :2], np.ones((len(c), 1))]) @ np.asarray(H, np.float64).T
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.hypot(x[:, 0] / x[:, 2] - c[:, 2], x[:, 1] / x[:, 2] - c[:, 3])
    return np.where(np.isfinite(e), e, np.inf)


def sampson(F, corr):
    """Sampson distance of x_r^T F x_l = 0"""
    c = np.asarray(corr, np.float64).reshape(-1, 4)
    F = np.asarray(F, np.float64)
    xl = np.hstack([c[:, :2], np.ones((len(c), 1))])
    xr = np.hstack([c[:, 2:], np.ones((len(c), 1))])
    a = xl @ F.T
    b = xr @ F
    e = (xr * a).sum(1)
    den = a[:, 0] ** 2 + a[:, 1] ** 2 + b[:, 0] ** 2 + b[:, 1] ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.sqrt(e * e / den)
    return np.where(np.isfinite(d), d, np.inf)


def error(model, M, corr):
    return transfer_error(M, corr) if model == HOMOGRAPHY else sampson(M, corr)


# ---- solvers ---------------------------------------------------------------------------------------------------------

def _cross(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def collinear(pts_n):
    """three of the four sample points collinear in either image (normalised coordinates)"""
    for t in range(4):
        tri = [j for j in range(4) if j != t]
        for o in (0, 2):
            a, b, c = (pts_n[j, o:o + 2] for j in tri)
            if abs(_cross(a, b, c)) < COLLINEAR_EPS:
                return True
    return False


def solve_h4(pts_n):
    """4-point DLT (SVD of the 8 x 9 system) in normalised coordinates; None when collinear"""
    if collinear(pts_n):
        return None
    A = []
    for x, y, xr, yr in pts_n:
        A.append([x, y, 1, 0, 0, 0, -xr * x, -xr * y, -xr])
        A.append([0, 0, 0, x, y, 1, -yr * x, -yr * y, -yr])
    return np.linalg.svd(np.array(A))[2][-1].reshape(3, 3)


def _f_rows(pts_n):
    x, y, xr, yr = (pts_n[:, k] for k in range(4))
    return np.stack([xr * x, xr * y, xr, yr * x, yr * y, yr, x, y, np.ones_like(x)], 1)


def solve_f7(pts_n):
    """7-point method: the real roots of det(l F1 + (1 - l) F2) = 0 over the SVD null space (list of 3 x 3)"""
    V = np.linalg.svd(_f_rows(pts_n))[2]
    F1, F2 = V[-1].reshape(3, 3), V[-2].reshape(3, 3)
    D = [np.linalg.det(F2 + l * (F1 - F2)) for l in (0.0, 1.0, -1.0, 2.0)]
    b = 0.5 * (D[1] + D[2]) - D[0]
    a = (D[3] - 4 * b - D[0] - (D[1] - D[2])) / 6.0
    c = 0.5 * (D[1] - D[2]) - a
    r = np.roots([a, b, c, D[0]])
    lam = np.sort(r[np.abs(r.imag) <= 1e-9 * np.maximum(1.0, np.abs(r))].real)
    return [l * F1 + (1 - l) * F2 for l in lam]


def refit(model, pts_n):
    """normalised DLT (H) or 8-point method with rank-2 enforcement (F): smallest eigenvector of the normal matrix"""
    if model == HOMOGRAPHY:
        x, y, xr, yr = (pts_n[:, k] for k in range(4))
        o, z = np.ones_like(x), np.zeros_like(x)
        A = np.vstack([np.stack([x, y, o, z, z, z, -xr * x, -xr * y, -xr], 1), np.stack([z, z, z, x, y, o, -yr * x, -yr * y, -yr], 1)])
    else:
        A = _f_rows(pts_n)
    w, V = np.linalg.eigh(A.T @ A)
    M = V[:, 0].reshape(3, 3)
    if model == FUNDAMENTAL:
        U, S, Vt = np.linalg.svd(M)
        M = U @ np.diag([S[0], S[1], 0.0]) @ Vt
    return M


def to_pixels(model, Mn, s, cl, cr):
    """normalised model -> pixels, scaled like the output (H22 = 1 / Frobenius 1 with the largest entry positive)"""
    Tl, Tr = xform(s, cl), xform(s, cr)
    M = np.linalg.inv(Tr) @ Mn @ Tl if model == HOMOGRAPHY else Tr.T @ Mn @ Tl
    return scale_output(model, M)


def scale_output(model, M):
    M = np.asarray(M, np.float64)
    n = np.linalg.norm(M)
    if not (n > 0 and np.isfinite(n)):
        return np.zeros((3, 3))
    if model == HOMOGRAPHY:
        return M / M[2, 2] if abs(M[2, 2]) >= 1e-8 * n else M / n
    f = M.ravel()
    big = f[np.argmax(np.abs(f))]
    return M / n * (1.0 if big >= 0 else -1.0)


def select(counts):
    """the winner: most inliers, ties to the smallest h; -1 when every hypothesis is invalid"""
    counts = np.asarray(counts)
    if counts.size == 0 or counts.max() < 0:
        return -1
    return int(np.argmax(counts))


# ---- planted models --------------------------------------------------------------------------------------------------

def planted_homography(rng, n, frac, sigma=0.3, w=1920, h=1080):
    """(corr (n, 4) float32, H, inlier flags, true errors): left points uniform, inliers H x + N(0, sigma), outliers
    uniform in the right image"""
    cx, cy = w / 2, h / 2
    th = rng.uniform(-0.3, 0.3)
    sc = rng.uniform(0.8, 1.25)
    A = np.array([[sc * np.cos(th), -sc * np.sin(th) + rng.uniform(-0.1, 0.1), 0], [sc * np.sin(th), sc * np.cos(th), 0], [0, 0, 1.0]])
    A[2, :2] = rng.uniform(-2e-4, 2e-4, 2)
    T0 = np.array([[1, 0, -cx], [0, 1, -cy], [0, 0, 1.0]])
    T1 = np.array([[1, 0, cx + rng.uniform(-50, 50)], [0, 1, cy + rng.uniform(-50, 50)], [0, 0, 1.0]])
    H = T1 @ A @ T0
    H /= H[2, 2]
    xl = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1)
    p = np.hstack([xl, np.ones((n, 1))]) @ H.T
    xr = p[:, :2] / p[:, 2:]
    inl = rng.random(n) < frac
    xr = np.where(inl[:, None], xr + rng.normal(0, sigma, (n, 2)), np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1))
    corr = np.hstack([xl, xr]).astype(np.float32)
    return corr, H, inl, transfer_error(H, corr)


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def planted_fundamental(rng, n, frac, sigma=0.3, w=1920, h=1080):
    """(corr, F, inlier flags, true Sampson distances, noise-free corr): two seeded cameras looking at 3D points"""
    f = rng.uniform(0.8, 1.2) * w
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1.0]])
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = rng.uniform(0.05, 0.2)
    R = np.cos(ang) * np.eye(3) + np.sin(ang) * _skew(ax) + (1 - np.cos(ang)) * np.outer(ax, ax)
    t = np.array([rng.uniform(-1, 1), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    X = np.stack([rng.uniform(-4, 4, n), rng.uniform(-2.5, 2.5, n), rng.uniform(6, 14, n)], 1)
    pl = X @ K.T
    pr = (X @ R.T + t) @ K.T
    xl, xr = pl[:, :2] / pl[:, 2:], pr[:, :2] / pr[:, 2:]
    Ki = np.linalg.inv(K)
    F = Ki.T @ _skew(t) @ R @ Ki
    F = scale_output(FUNDAMENTAL, F)
    clean = np.hstack([xl, xr])
    inl = rng.random(n) < frac
    xln = xl + rng.normal(0, sigma, (n, 2))
    xrn = np.where(inl[:, None], xr + rng.normal(0, sigma, (n, 2)), np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1))
    corr = np.hstack([np.where(inl[:, None], xln, xl), xrn]).astype(np.float32)
    return corr, F, inl, sampson(F, corr), clean
