"""Float64 numpy statement of ps_view_graph_filter (include/popsift_b200_viewgraph.h) for the tests; nothing in the
package imports it.

Steps 1-6 of the header: the used pairs and their orthonormal rotations (global_oracle's), the triangles of the used
pairs, each cycle error with the products written out in the order of k_viewgraph.h (no BLAS, so every rounding is the
kernel's but for the libm of sqrt and atan2), the per-pair statistics and the one-pass decision.  Also plants graphs:
view graphs with outliers, complete graphs, trees and the "doppelganger" case."""
from __future__ import annotations

import math

import numpy as np

import global_oracle as go

DEG = math.pi / 180.0


def used_pairs(pairs, Rp, n_front, min_inliers):
    """step 1: (used (P,) bool, R (P, 3, 3) the orthonormal rotations of the used pairs, identity elsewhere)"""
    Rp = np.asarray(Rp, np.float32).reshape(-1, 3, 3)
    P = len(pairs)
    used = np.zeros(P, bool)
    R = np.tile(np.eye(3), (P, 1, 1))
    for p, (l, r) in enumerate(pairs):
        used[p] = int(n_front[p]) >= min_inliers and np.isfinite(Rp[p]).all() and l != r
        if used[p]:
            R[p] = go.orthonormal(Rp[p])
    return used, R


def has_duplicates(pairs):
    keys = [(min(a, b), max(a, b)) for a, b in pairs]
    return len(set(keys)) != len(keys)


def triangles(n_sets, pairs, used):
    """step 3: every triangle of the used pairs as (a, b, c) with a < b < c and its pairs (p_ab, p_bc, p_ca): two (T, 3)
    int64 arrays, sorted by (a, b, c)"""
    pid = np.full((n_sets, n_sets), -1, np.int64)
    for p in np.flatnonzero(used):
        l, r = pairs[p]
        pid[l, r] = pid[r, l] = p
    adj = pid >= 0
    tri, tp = [], []
    for a in range(n_sets):
        nb = np.flatnonzero(adj[a])
        nb = nb[nb > a]
        for b in nb:
            cs = np.flatnonzero(adj[a] & adj[b])
            cs = cs[cs > b]
            if len(cs):
                tri.append(np.stack([np.full(len(cs), a), np.full(len(cs), b), cs], 1))
                tp.append(np.stack([np.full(len(cs), pid[a, b]), pid[b, cs], pid[cs, a]], 1))
    if not tri:
        return np.zeros((0, 3), np.int64), np.zeros((0, 3), np.int64)
    return np.concatenate(tri).astype(np.int64), np.concatenate(tp).astype(np.int64)


def _mul(A, B):
    """gl_mul on stacks: each entry summed in k order, no contraction"""
    C = np.empty(np.broadcast_shapes(A.shape, B.shape))
    for i in range(3):
        for j in range(3):
            C[..., i, j] = A[..., i, 0] * B[..., 0, j] + A[..., i, 1] * B[..., 1, j] + A[..., i, 2] * B[..., 2, j]
    return C


def directed(R, pairs, p, x):
    """R(x -> y) of the pairs p (T,) leaving sets x (T,): R_p when stored as (x, .), R_p^T otherwise"""
    ends = np.asarray(pairs, np.int64).reshape(-1, 2)
    Rs = R[p]
    flip = ends[p, 0] != x
    Rs = Rs.copy()
    Rs[flip] = np.swapaxes(Rs[flip], 1, 2)
    return Rs


def cycle_errors(pairs, R, tri, tp):
    """vg_cycle_error of every triangle, degrees: |Log(R(c->a) (R(b->c) R(a->b)))|"""
    if len(tri) == 0:
        return np.zeros(0)
    A = directed(R, pairs, tp[:, 0], tri[:, 0])
    B = directed(R, pairs, tp[:, 1], tri[:, 1])
    Cm = directed(R, pairs, tp[:, 2], tri[:, 2])
    w = go.log_batch(_mul(Cm, _mul(B, A)))
    return np.sqrt(w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1] + w[:, 2] * w[:, 2]) / DEG


def cycle_error(Rab, t_ab, Rbc, t_bc, Rca, t_ca):
    """one triangle, the arguments of vg_cycle_error"""
    f = lambda M, t: np.asarray(M, np.float64).T if t else np.asarray(M, np.float64)   # noqa: E731
    w = go.log(_mul(f(Rca, t_ca), _mul(f(Rbc, t_bc), f(Rab, t_ab))))
    return math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]) / DEG


def view_graph_filter(n_sets, pairs, Rp, n_front, max_cycle_error=3.0, min_consistent=1, min_fraction=0.0, keep_untested=False,
                      min_inliers=15):
    """ps_view_graph_filter: dict(keep, n_triangles, n_consistent, min_error (float64, +inf: none), used, report, errors,
    triangles)"""
    pairs = [(int(a), int(b)) for a, b in pairs]
    assert not has_duplicates(pairs)
    P = len(pairs)
    used, R = used_pairs(pairs, Rp, n_front, min_inliers)
    tri, tp = triangles(n_sets, pairs, used)
    e = cycle_errors(pairs, R, tri, tp)
    ok = e <= max_cycle_error
    flat = tp.reshape(-1)
    nt = np.bincount(flat, minlength=P)[:P].astype(np.int64)
    nc = np.bincount(flat, weights=np.repeat(ok, 3).astype(np.float64), minlength=P)[:P].astype(np.int64)
    mn = np.full(P, np.inf)
    np.minimum.at(mn, flat, np.repeat(e, 3))
    keep = used & np.where(nt > 0, (nc >= min_consistent) & (nc.astype(np.float64) >= min_fraction * nt.astype(np.float64)),
                           bool(keep_untested))
    report = dict(n_triangles=len(tri), n_consistent_triangles=int(ok.sum()), n_used=int(used.sum()), n_kept=int(keep.sum()),
                  n_untested=int((used & (nt == 0)).sum()))
    return dict(keep=keep, n_triangles=nt, n_consistent=nc, min_error=mn, used=used, report=report, errors=e, triangles=tri)


# ---- planted graphs --------------------------------------------------------------------------------------------------

def planted(rng, n_cams, n_pairs, noise_deg=0.5, outliers=0.1, hub=None):
    """global_oracle.view_graph with every pair's n_front drawn from 30 to 500 (outliers too, so n_front says nothing about
    them): (R_true, pairs, Rp, n_front, is_outlier)"""
    Rt, pairs, Rp, _, out = go.view_graph(rng, n_cams, n_pairs, noise_deg=noise_deg, outliers=outliers, hub=hub)
    nf = rng.integers(30, 501, size=len(pairs))
    return Rt, pairs, np.asarray(Rp), nf, np.asarray(out, bool)


def exact_pairs(Rt, pairs, rng=None, noise_deg=0.0):
    """R_p = R_r R_l^T (turned by noise_deg about a random axis when rng is given)"""
    out = []
    for l, r in pairs:
        M = Rt[r] @ Rt[l].T
        if rng is not None and noise_deg > 0:
            M = go.exp(_axis(rng) * noise_deg * DEG) @ M
        out.append(M)
    return np.stack(out) if out else np.zeros((0, 3, 3))


def _axis(rng):
    w = rng.normal(size=3)
    return w / np.linalg.norm(w)


def complete(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def tree(rng, n):
    return [(int(rng.integers(0, i)), i) for i in range(1, n)]


def doppelganger(rng, n_true=8, n_group=3, wrong_deg=40.0, noise_deg=0.2):
    """set 0 joined to its true neighbours 1 + n_group .. n_group + n_true and to a group G = 1 .. n_group; the whole cluster
    is complete.  The pairs (0, g), g in G, use the rotation set 0 would have if it were turned by wrong_deg: wrong for 0,
    consistent across G.  Returns (R_true, pairs, Rp, n_front, the (0, g) pair indices)"""
    n = 1 + n_group + n_true
    Rt = np.stack([go.random_rotation(rng) for _ in range(n)])
    R0 = go.exp(_axis(rng) * wrong_deg * DEG) @ Rt[0]
    pairs = complete(n)
    Rp, bad = [], []
    for p, (l, r) in enumerate(pairs):
        Rl = R0 if (l == 0 and 1 <= r <= n_group) else Rt[l]
        if l == 0 and 1 <= r <= n_group:
            bad.append(p)
        Rp.append(go.exp(_axis(rng) * noise_deg * DEG) @ Rt[r] @ Rl.T)
    return Rt, pairs, np.stack(Rp), np.full(len(pairs), 200), np.array(bad)
