"""Float64 numpy restatement of ps_relative_pose_batch (include/popsift_b200_pose.h) for the tests; nothing in the package
imports it.

The five-point solver here is independent of the device's arithmetic: an SVD null space, the ten cubics in graded reverse
lexicographic order, one linear solve and the eigenvectors of the 10 x 10 action matrix of x (Stewenius), where the
device uses Gauss-Jordan eliminations and the real roots of a degree-10 polynomial (Nister).  The rest restates the
contract: calibration, projection onto the essential matrices, the four-candidate decomposition, triangulation and
cheirality, the midpoint, and planted scenes with known truth."""
from __future__ import annotations

import numpy as np

import verify_oracle as vo

SLOTS = 10


# ---- calibration -----------------------------------------------------------------------------------------------------

def calibrate(corr, cam_l, cam_r, threshold):
    """(rows (n, 4) float32 calibrated, t2 float32): x^ = (x - cx) / fx in double, rounded once"""
    c = np.asarray(corr, np.float32).astype(np.float64).reshape(-1, 4)
    fl = np.asarray(cam_l, np.float32).astype(np.float64)
    fr = np.asarray(cam_r, np.float32).astype(np.float64)
    rows = np.stack([(c[:, 0] - fl[2]) / fl[0], (c[:, 1] - fl[3]) / fl[1], (c[:, 2] - fr[2]) / fr[0], (c[:, 3] - fr[3]) / fr[1]], 1)
    fbar = (fl[0] + fl[1] + fr[0] + fr[1]) / 4.0
    return rows.astype(np.float32), np.float32((np.float64(np.float32(threshold)) / fbar) ** 2)


def K(cam):
    fx, fy, cx, cy = (float(v) for v in np.asarray(cam, np.float32))
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])


# ---- five-point (action matrix) --------------------------------------------------------------------------------------

# graded reverse lexicographic monomials of degree <= 3 in (x, y, z): the ten cubics, then the basis of the quotient ring
_MONS = [(3, 0, 0), (2, 1, 0), (2, 0, 1), (1, 2, 0), (1, 1, 1), (1, 0, 2), (0, 3, 0), (0, 2, 1), (0, 1, 2), (0, 0, 3),
         (2, 0, 0), (1, 1, 0), (1, 0, 1), (0, 2, 0), (0, 1, 1), (0, 0, 2), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
_IDX = {m: i for i, m in enumerate(_MONS)}
_LIN = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]


def _pmul(a, b):
    out = {}
    for ma, ca in a.items():
        for mb, cb in b.items():
            m = (ma[0] + mb[0], ma[1] + mb[1], ma[2] + mb[2])
            out[m] = out.get(m, 0.0) + ca * cb
    return out


def _padd(a, b, s=1.0):
    out = dict(a)
    for m, c in b.items():
        out[m] = out.get(m, 0.0) + s * c
    return out


def _constraints(basis):
    """the 10 x 20 coefficient matrix of det E = 0 and 2 E E^T E - tr(E E^T) E = 0, E = x X + y Y + z Z + W"""
    E = [[{_LIN[k]: basis[k][3 * i + j] for k in range(4)} for j in range(3)] for i in range(3)]
    EEt = [[_padd(_padd(_pmul(E[i][0], E[j][0]), _pmul(E[i][1], E[j][1])), _pmul(E[i][2], E[j][2])) for j in range(3)] for i in range(3)]
    tr = _padd(_padd(EEt[0][0], EEt[1][1]), EEt[2][2])
    eqs = []
    for i in range(3):
        for j in range(3):
            acc = {}
            for k in range(3):
                acc = _padd(acc, _pmul(EEt[i][k], E[k][j]), 2.0)
            eqs.append(_padd(acc, _pmul(tr, E[i][j]), -1.0))
    det = {}
    for (a, b, c), s in (((0, 1, 2), 1), ((0, 2, 1), -1), ((1, 0, 2), -1), ((1, 2, 0), 1), ((2, 0, 1), 1), ((2, 1, 0), -1)):
        det = _padd(det, _pmul(_pmul(E[0][a], E[1][b]), E[2][c]), s)
    eqs.append(det)
    A = np.zeros((10, 20))
    for r, q in enumerate(eqs):
        for m, c in q.items():
            A[r, _IDX[m]] += c
    return A


def five_point(rows5, info=False):
    """essential matrices (list of 3 x 3, Frobenius 1, largest entry positive) through five calibrated rows; with info=True
    also whether the sample is stable: a well-conditioned elimination, and every eigenvalue clearly real or clearly not,
    and clearly apart from the others"""
    r = np.asarray(rows5, np.float64).reshape(5, 4)
    Q = np.stack([r[:, 2] * r[:, 0], r[:, 2] * r[:, 1], r[:, 2], r[:, 3] * r[:, 0], r[:, 3] * r[:, 1], r[:, 3], r[:, 0], r[:, 1],
                  np.ones(5)], 1)
    V = np.linalg.svd(Q)[2]
    basis = V[5:9]
    A = _constraints(basis)
    stable = True
    try:
        cond = np.linalg.cond(A[:, :10])
        B = np.linalg.solve(A[:, :10], A[:, 10:])
    except np.linalg.LinAlgError:
        return ([], False) if info else []
    if not np.isfinite(cond) or cond > 1e7:
        stable = False
    M = np.zeros((10, 10))
    M[:6] = -B[:6]
    for row, col in ((6, 0), (7, 1), (8, 2), (9, 6)):
        M[row, col] = 1.0
    w, vec = np.linalg.eig(M)
    sols = []
    scale = max(1.0, np.abs(w).max())
    real = np.abs(w.imag) <= 1e-8 * scale
    if (np.abs(w.imag)[~real] < 1e-5 * scale).any():
        stable = False
    wr = np.sort(w.real[real])
    if len(wr) > 1 and np.diff(wr).min() < 1e-5 * scale:
        stable = False
    for k in np.nonzero(real)[0]:
        v = vec[:, k].real
        if abs(v[9]) < 1e-12 * np.abs(v).max():
            stable = False
            continue
        x, y, z = v[6] / v[9], v[7] / v[9], v[8] / v[9]
        E = (x * basis[0] + y * basis[1] + z * basis[2] + basis[3]).reshape(3, 3)
        sols.append(vo.scale_output(vo.FUNDAMENTAL, E))
    return (sols, stable) if info else sols


def contains(sols, E, rtol):
    """E (scaled as the contract's hypotheses) is within rtol (Frobenius) of one of sols"""
    E = vo.scale_output(vo.FUNDAMENTAL, E)
    return any(np.linalg.norm(np.asarray(S, np.float64) - E) <= rtol for S in sols)


def same_set(a, b, rtol):
    return len(a) == len(b) and all(contains(b, E, rtol) for E in a)


# ---- projection, decomposition, triangulation ------------------------------------------------------------------------

def project_essential(M):
    U, S, Vt = np.linalg.svd(np.asarray(M, np.float64).reshape(3, 3))
    return vo.scale_output(vo.FUNDAMENTAL, U @ np.diag([1.0, 1.0, 0.0]) @ Vt)


def candidates(E):
    """the four (R, t) of E in the contract's order, U and V with det +1"""
    U, S, Vt = np.linalg.svd(np.asarray(E, np.float64).reshape(3, 3))
    if np.linalg.det(U) < 0:
        U[:, 2] *= -1
    if np.linalg.det(Vt) < 0:
        Vt[2] *= -1
    W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    R1, R2, u3 = U @ W @ Vt, U @ W.T @ Vt, U[:, 2]
    return [(R1, u3), (R1, -u3), (R2, u3), (R2, -u3)]


def triangulate(R, t, rows):
    """(det, a.a * b.b, d_l, d_r, midpoints (n, 3)) of each calibrated row under (R, t)"""
    r = np.asarray(rows, np.float64).reshape(-1, 4)
    R = np.asarray(R, np.float64).reshape(3, 3)
    t = np.asarray(t, np.float64).reshape(3)
    xl = np.hstack([r[:, :2], np.ones((len(r), 1))])
    b = np.hstack([r[:, 2:], np.ones((len(r), 1))])
    a = xl @ R.T
    aa, bb, ab = (a * a).sum(1), (b * b).sum(1), (a * b).sum(1)
    at, bt = a @ t, b @ t
    det = aa * bb - ab * ab
    with np.errstate(divide="ignore", invalid="ignore"):
        dl = (ab * bt - at * bb) / det
        dr = (aa * bt - ab * at) / det
    X = 0.5 * (dl[:, None] * xl + (dr[:, None] * b - t) @ R)
    return det, aa * bb, dl, dr, X


def in_front(R, t, rows):
    det, ref, dl, dr, _ = triangulate(R, t, rows)
    return (det > 1e-12 * ref) & (dl > 0) & (dr > 0)


def choose(E, rows):
    """(index, R, t, counts) of the candidate with the most rows in front, ties to the lower index"""
    cands = candidates(E)
    counts = [int(in_front(R, t, rows).sum()) for R, t in cands]
    k = int(np.argmax(counts))
    return k, cands[k][0], cands[k][1], counts


def skew(t):
    return vo._skew(np.asarray(t, np.float64))


def essential(R, t):
    return skew(t) @ np.asarray(R, np.float64) / np.sqrt(2.0)


def pixels_f(E, cam_l, cam_r):
    return vo.scale_output(vo.FUNDAMENTAL, np.linalg.inv(K(cam_r)).T @ np.asarray(E, np.float64) @ np.linalg.inv(K(cam_l)))


def sampson_calibrated(E, rows):
    return vo.sampson(E, rows)


def rot_angle(Ra, Rb):
    """degrees between two rotations (|Ra - Rb|_F = 2 sqrt(2) sin(angle / 2), accurate for small angles)"""
    d = np.linalg.norm(np.asarray(Ra, np.float64) - np.asarray(Rb, np.float64))
    return np.degrees(2 * np.arcsin(min(1.0, d / (2 * np.sqrt(2)))))


def dir_angle(a, b):
    """degrees between two directions (accurate for small angles)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a, b = a / np.linalg.norm(a), b / np.linalg.norm(b)
    return np.degrees(2 * np.arcsin(min(1.0, np.linalg.norm(a - b) / 2)))


# ---- planted scenes --------------------------------------------------------------------------------------------------

def _rotation(rng, lo_deg=2.0, hi_deg=12.0):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = np.radians(rng.uniform(lo_deg, hi_deg))
    return np.cos(ang) * np.eye(3) + np.sin(ang) * vo._skew(ax) + (1 - np.cos(ang)) * np.outer(ax, ax)


def planted_pose(rng, n, frac, sigma=0.3, w=1920, h=1080, forward=None):
    """(corr (n, 4) float32, (cam_l, cam_r), R, t (unit), inlier flags, true errors in pixels, clean corr): two cameras with
    different intrinsics, a rotation of 2-12 degrees, sideways or forward / backward translation (forward=None: either),
    3-D points at depths 4-15 seen by both; outliers uniform in the right image"""
    cams = []
    for _ in range(2):
        f = rng.uniform(0.7, 1.3) * w
        cams.append(np.array([f * rng.uniform(0.97, 1.03), f, w / 2 + rng.uniform(-20, 20), h / 2 + rng.uniform(-20, 20)], np.float32))
    R = _rotation(rng)
    fwd = rng.random() < 0.5 if forward is None else forward
    if fwd:
        t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.choice([-1.0, 1.0]) * rng.uniform(0.5, 1.0)])
    else:
        t = np.array([rng.choice([-1.0, 1.0]) * rng.uniform(0.5, 1.0), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    t /= np.linalg.norm(t)
    Kl, Kr = K(cams[0]), K(cams[1])
    X = np.zeros((0, 3))
    while len(X) < n:
        m = 4 * n + 16
        z = rng.uniform(4, 15, m)
        u = rng.uniform(0, w, m); v = rng.uniform(0, h, m)
        P = np.linalg.solve(Kl, np.stack([u, v, np.ones(m)])).T * z[:, None]
        Pr = P @ R.T + t
        pr = Pr @ Kr.T
        with np.errstate(divide="ignore", invalid="ignore"):
            ur, vr = pr[:, 0] / pr[:, 2], pr[:, 1] / pr[:, 2]
        ok = (Pr[:, 2] > 1.0) & (ur >= 0) & (ur < w) & (vr >= 0) & (vr < h)
        X = np.vstack([X, P[ok]])
    X = X[:n]
    pl = X @ Kl.T
    pr = (X @ R.T + t) @ Kr.T
    xl, xr = pl[:, :2] / pl[:, 2:], pr[:, :2] / pr[:, 2:]
    clean = np.hstack([xl, xr])
    inl = rng.random(n) < frac
    xln = xl + rng.normal(0, sigma, (n, 2))
    xrn = np.where(inl[:, None], xr + rng.normal(0, sigma, (n, 2)), np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1))
    corr = np.hstack([np.where(inl[:, None], xln, xl), xrn]).astype(np.float32)
    F = pixels_f(essential(R, t), cams[0], cams[1])
    return corr, (cams[0], cams[1]), R, t, inl, vo.sampson(F, corr), clean
