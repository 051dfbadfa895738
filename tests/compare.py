"""Set-based comparison of SIFT outputs (SURVEY.md section 8c parity protocol) -- test helper."""
from __future__ import annotations

import numpy as np


def match_keypoints(kp_a: np.ndarray, kp_b: np.ndarray, tol_xy=0.5, tol_sig=0.05, tol_th=0.1):
    """One-to-one greedy matching of rows (x, y, sigma, theta) in input-image coordinates.

    Returns (pairs[(i, j)], precision, recall, f1); a is the candidate, b the reference."""
    na, nb = len(kp_a), len(kp_b)
    if na == 0 or nb == 0:
        return [], 0.0 if na else 1.0, 0.0 if nb else 1.0, 1.0 if na == nb else 0.0
    order = np.argsort(kp_b[:, 0], kind="stable")
    bx = kp_b[order, 0]
    cands = []
    for i in range(na):
        lo = np.searchsorted(bx, kp_a[i, 0] - tol_xy, "left")
        hi = np.searchsorted(bx, kp_a[i, 0] + tol_xy, "right")
        for jj in range(lo, hi):
            j = order[jj]
            if abs(kp_a[i, 1] - kp_b[j, 1]) >= tol_xy:
                continue
            if abs(kp_a[i, 2] - kp_b[j, 2]) >= tol_sig * kp_b[j, 2]:
                continue
            dth = abs(kp_a[i, 3] - kp_b[j, 3]) % (2 * np.pi)
            dth = min(dth, 2 * np.pi - dth)
            if dth >= tol_th:
                continue
            d = np.hypot(kp_a[i, 0] - kp_b[j, 0], kp_a[i, 1] - kp_b[j, 1]) + dth
            cands.append((d, i, j))
    cands.sort()
    used_a, used_b, pairs = set(), set(), []
    for d, i, j in cands:
        if i in used_a or j in used_b:
            continue
        used_a.add(i); used_b.add(j); pairs.append((i, j))
    prec = len(pairs) / na
    rec = len(pairs) / nb
    f1 = 2 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0
    return pairs, prec, rec, f1


def descriptor_l2(desc_a, desc_b, pairs):
    if not pairs:
        return np.zeros(0)
    ia = np.array([p[0] for p in pairs]); ib = np.array([p[1] for p in pairs])
    # a fixture that keeps a sample of the reference's descriptors marks the others as all-NaN rows: pairs are compared
    # where the reference row is stored
    kept = ~np.isnan(desc_b[ib]).all(axis=1)
    ia, ib = ia[kept], ib[kept]
    return np.linalg.norm(desc_a[ia].astype(np.float64) - desc_b[ib].astype(np.float64), axis=1)


def report(kp_a, desc_a, kp_b, desc_b, **tol):
    pairs, p, r, f1 = match_keypoints(kp_a, kp_b, **tol)
    l2 = descriptor_l2(desc_a, desc_b, pairs)
    return {"n_a": len(kp_a), "n_b": len(kp_b), "matched": len(pairs), "precision": p, "recall": r,
            "f1": f1, "desc_compared": len(l2), "desc_l2_max": float(l2.max()) if len(l2) else 0.0,
            "desc_l2_median": float(np.median(l2)) if len(l2) else 0.0,
            "desc_l2_p99": float(np.percentile(l2, 99)) if len(l2) else 0.0}
