"""Float64 numpy statement of ps_rotation_averaging and ps_global_positioning (include/popsift_b200_global.h) for the
tests; nothing in the package imports it.

The rotation logarithm and the observation rule follow k_global.h; Exp and the losses are bundle_oracle's, the rays
triangulate_oracle's.  Every linear system is solved densely, so the device (preconditioned CG) agrees with it to the CG
tolerance, not bit for bit.  It also plants view graphs: random rotations, noisy relative rotations and outlier pairs."""
from __future__ import annotations

import math

import numpy as np

import bundle_oracle as bo
import triangulate_oracle as tro

RA_MAX_ITERS, RA_STEP_TOL, RA_NO_PAIRS = range(3)
GP_MAX_ITERS, GP_FUNCTION_TOL, GP_NO_OBSERVATIONS = range(3)
DEG = math.pi / 180.0


# ---- rotations (k_global.h) ------------------------------------------------------------------------------------------

def log(M):
    """gl_log: the rotation vector of a rotation matrix"""
    M = np.asarray(M, np.float64)
    c = min(1.0, max(-1.0, 0.5 * ((M[0, 0] + M[1, 1] + M[2, 2]) - 1.0)))
    s = np.array([0.5 * (M[2, 1] - M[1, 2]), 0.5 * (M[0, 2] - M[2, 0]), 0.5 * (M[1, 0] - M[0, 1])])
    sn = math.sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])
    th = math.atan2(sn, c)
    if c > -0.99:
        f = 1.0 + sn * sn / 6.0 if sn < 1e-8 else th / sn
        return f * s
    B = 0.5 * (M + M.T)
    k = 0
    if B[1, 1] > B[k, k]:
        k = 1
    if B[2, 2] > B[k, k]:
        k = 2
    omc = 1.0 - c
    a = np.zeros(3)
    a[k] = math.sqrt(max(0.0, (B[k, k] - c) / omc))
    for j in range(3):
        if j != k:
            a[j] = B[j, k] / (omc * a[k])
    sg = -1.0 if a[0] * s[0] + a[1] * s[1] + a[2] * s[2] < 0.0 else 1.0
    return th * (sg * a)


def exp(w):
    return bo.rodrigues(w)


def orthonormal(m):
    """gl_orthonormal: the rotation of the unit quaternion of a float32 matrix (Shepperd's branches)"""
    a = np.asarray(m, np.float32).astype(np.float64).reshape(9)
    tr = a[0] + a[4] + a[8]
    if tr > 0.0:
        s = 2.0 * math.sqrt(tr + 1.0)
        w, x, y, z = 0.25 * s, (a[7] - a[5]) / s, (a[2] - a[6]) / s, (a[3] - a[1]) / s
    elif a[0] > a[4] and a[0] > a[8]:
        s = 2.0 * math.sqrt(1.0 + a[0] - a[4] - a[8])
        w, x, y, z = (a[7] - a[5]) / s, 0.25 * s, (a[1] + a[3]) / s, (a[2] + a[6]) / s
    elif a[4] > a[8]:
        s = 2.0 * math.sqrt(1.0 + a[4] - a[0] - a[8])
        w, x, y, z = (a[2] - a[6]) / s, (a[1] + a[3]) / s, 0.25 * s, (a[5] + a[7]) / s
    else:
        s = 2.0 * math.sqrt(1.0 + a[8] - a[0] - a[4])
        w, x, y, z = (a[3] - a[1]) / s, (a[2] + a[6]) / s, (a[5] + a[7]) / s, 0.25 * s
    n = math.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w)],
                     [2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w)],
                     [2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)]])


def pair_residual(Rl, Rr, Rp):
    return log(np.asarray(Rr).T @ (np.asarray(Rp) @ np.asarray(Rl)))


def _find(par, a):
    while par[a] != a:
        par[a] = par[par[a]]
        a = par[a]
    return a


def start(n_sets, pairs, Rp, n_front, min_inliers):
    """steps 1-3 of ps_rotation_averaging: (used (P,) bool, registered (S,) bool, root, R (S, 3, 3))"""
    P = len(pairs)
    used = np.zeros(P, bool)
    par = list(range(n_sets))
    for p, (l, r) in enumerate(pairs):
        used[p] = n_front[p] >= min_inliers and np.isfinite(Rp[p]).all() and l != r
        if used[p]:
            a, b = _find(par, l), _find(par, r)
            if a != b:
                par[max(a, b)] = min(a, b)
    comp = np.array([_find(par, i) for i in range(n_sets)], np.int64)
    size = np.bincount(comp, minlength=n_sets)
    root = int(np.argmax(size)) if n_sets else -1     # the first (smallest) component root of the largest size
    reg = comp == root if n_sets else np.zeros(0, bool)
    for p, (l, _) in enumerate(pairs):
        used[p] = used[p] and reg[l]
    R = np.tile(np.eye(3), (n_sets, 1, 1))
    order = sorted(np.flatnonzero(used), key=lambda p: (-int(n_front[p]), p))
    par = list(range(n_sets))
    adj = [[] for _ in range(n_sets)]
    for p in order:
        l, r = pairs[p]
        a, b = _find(par, l), _find(par, r)
        if a == b:
            continue
        par[a] = b
        adj[l].append(p)
        adj[r].append(p)
    if n_sets:
        known = np.zeros(n_sets, bool)
        known[root] = True
        stack = [root]
        while stack:
            i = stack.pop()
            for p in adj[i]:
                l, r = pairs[p]
                o = r if l == i else l
                if known[o]:
                    continue
                if o == r:
                    R[r] = Rp[p] @ R[l]
                else:
                    R[l] = Rp[p].T @ R[r]
                known[o] = True
                stack.append(o)
    return used, reg, root, R


def laplacian_solve(n, ends, W, g, root, n_cam=None):
    """the weighted Laplacian (x) I3 system of the header with node `root` and the nodes of zero degree held: x (n, 3).
    Dense; n_cam (where the point nodes start, see LaplacianSystem) is not needed here."""
    D = np.zeros(n)
    b = np.zeros((n, 3))
    for (a, c), w, ge in zip(ends, W, g):
        if w == 0.0:
            continue
        D[a] += w
        D[c] += w
        b[a] += ge
        b[c] -= ge
    free = [i for i in range(n) if i != root and D[i] > 0.0]
    idx = {i: k for k, i in enumerate(free)}
    L = np.zeros((len(free), len(free)))
    for (a, c), w in zip(ends, W):
        if w == 0.0:
            continue
        for u, v in ((a, c), (c, a)):
            if u in idx:
                L[idx[u], idx[u]] += w
                if v in idx:
                    L[idx[u], idx[v]] -= w
    x = np.zeros((n, 3))
    if free:
        x[free] = np.linalg.solve(L, b[free])
    return x


class LaplacianSystem:
    """laplacian_solve's system with the point nodes (n_cam and up) eliminated, assembled with bincount.  A point node joins
    only camera nodes, so its row is D_j x_j - sum_e w_e x_c(e) = b_j and x_j = (b_j + sum_e w_e x_c(e)) / D_j; putting that
    into the camera rows leaves S x_c = b_c with S = L_cc - sum_j sum_{e, f at j} w_e w_f / D_j and
    b_c = b_c + sum_j sum_{e at j} w_e b_j / D_j, over the free camera nodes (not the root, degree > 0)."""

    def __init__(self, n, ends, W, g, root, n_cam=None):
        n_cam = n if n_cam is None else n_cam
        ends = np.asarray(ends, np.int64).reshape(-1, 2)
        W, g = np.asarray(W, np.float64), np.asarray(g, np.float64).reshape(-1, 3)
        on = W != 0.0
        ends, W, g = ends[on], W[on], g[on]
        a, c = ends[:, 0], ends[:, 1]
        assert not ((a >= n_cam) & (c >= n_cam)).any(), "an edge between two point nodes"
        D = np.bincount(a, weights=W, minlength=n) + np.bincount(c, weights=W, minlength=n)
        b = np.stack([np.bincount(a, weights=g[:, k], minlength=n) - np.bincount(c, weights=g[:, k], minlength=n) for k in range(3)], 1)
        free = (D > 0.0) & (np.arange(n) != root)
        self.n, self.n_cam, self.D, self.bfull, self.free = n, n_cam, D, b, free
        cams = np.flatnonzero(free[:n_cam])
        idx = np.full(n, -1, np.int64)
        idx[cams] = np.arange(len(cams))
        self.cams, self.idx = cams, idx
        m = len(cams)
        # camera-camera edges
        cc = (a < n_cam) & (c < n_cam)
        Lf = np.bincount(idx[cams] * m + idx[cams], weights=D[cams], minlength=m * m)
        for u, v in ((a[cc], c[cc]), (c[cc], a[cc])):
            k = (idx[u] >= 0) & (idx[v] >= 0)
            Lf -= np.bincount(idx[u[k]] * m + idx[v[k]], weights=W[cc][k], minlength=m * m)
        # camera-point edges, grouped by point: every pair (e, f) at a free point
        pe = ~cc
        pt = np.where(a[pe] >= n_cam, a[pe], c[pe])
        cm = np.where(a[pe] >= n_cam, c[pe], a[pe])
        wp = W[pe]
        o = np.argsort(pt, kind="stable")
        pt, cm, wp = pt[o], cm[o], wp[o]
        self.pt, self.cm, self.wp = pt, cm, wp
        bc = b[cams].copy()
        if len(pt):
            fp = free[pt]
            k = fp & (idx[cm] >= 0)
            for q in range(3):
                bc[:, q] += np.bincount(idx[cm[k]], weights=wp[k] * b[pt[k], q] / D[pt[k]], minlength=m)
            uniq, first, cnt = np.unique(pt, return_index=True, return_counts=True)
            for L in np.unique(cnt):
                sel = first[cnt == L]
                e = (sel[:, None, None] + np.arange(L)[None, :, None]).repeat(L, 2).reshape(-1)
                f = (sel[:, None, None] + np.arange(L)[None, None, :]).repeat(L, 1).reshape(-1)
                k = free[pt[e]] & (idx[cm[e]] >= 0) & (idx[cm[f]] >= 0)
                e, f = e[k], f[k]
                Lf -= np.bincount(idx[cm[e]] * m + idx[cm[f]], weights=wp[e] * wp[f] / D[pt[e]], minlength=m * m)
        self.S, self.b = Lf.reshape(m, m), bc

    def points(self, xc):
        """every node's x from the free cameras' x (m, 3): the held nodes 0, each free point by its row"""
        x = np.zeros((self.n, 3))
        x[self.cams] = xc
        if len(self.pt):
            s = np.stack([np.bincount(self.pt, weights=self.wp * x[self.cm, q], minlength=self.n) for q in range(3)], 1)
            pts = np.flatnonzero(self.free & (np.arange(self.n) >= self.n_cam))
            x[pts] = (self.bfull[pts] + s[pts]) / self.D[pts][:, None]
        return x

    def solve(self):
        return self.points(np.linalg.solve(self.S, self.b) if len(self.cams) else np.zeros((0, 3)))


def laplacian_solve_reduced(n, ends, W, g, root, n_cam=None):
    """laplacian_solve by LaplacianSystem: the same x (n, 3), to rounding"""
    return LaplacianSystem(n, ends, W, g, root, n_cam).solve()


def log_batch(M):
    """log of each (..., 3, 3): gl_log's branch c > -0.99 vectorised, the rest one by one"""
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    c = np.clip(0.5 * ((M[:, 0, 0] + M[:, 1, 1] + M[:, 2, 2]) - 1.0), -1.0, 1.0)
    s = np.stack([0.5 * (M[:, 2, 1] - M[:, 1, 2]), 0.5 * (M[:, 0, 2] - M[:, 2, 0]), 0.5 * (M[:, 1, 0] - M[:, 0, 1])], 1)
    sn = np.sqrt(s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1] + s[:, 2] * s[:, 2])
    th = np.arctan2(sn, c)
    with np.errstate(invalid="ignore", divide="ignore"):
        f = np.where(sn < 1e-8, 1.0 + sn * sn / 6.0, th / sn)
    out = f[:, None] * s
    for k in np.flatnonzero(~(c > -0.99)):
        out[k] = log(M[k])
    return out


def rotation_averaging(n_sets, pairs, Rp, n_front, loss="cauchy", loss_scale=5.0, max_iters=100, step_tol=1e-4, min_inliers=15,
                       solve=laplacian_solve):
    """ps_rotation_averaging, each Laplacian system by solve(n, ends, W, g, root) (default dense; laplacian_solve_reduced
    for large graphs): (R (S, 3, 3), registered, pair_error (deg), report dict)"""
    pairs = [(int(a), int(b)) for a, b in pairs]
    Rp = np.asarray(Rp, np.float32).reshape(-1, 3, 3)
    Rp = np.stack([orthonormal(m) if np.isfinite(m).all() else m.astype(np.float64) for m in Rp]) if len(Rp) else np.zeros((0, 3, 3))
    used, reg, root, R = start(n_sets, pairs, Rp, np.asarray(n_front), min_inliers)
    s2 = (loss_scale * DEG) ** 2
    rep = dict(iterations=0, n_pairs=int(used.sum()), n_registered=int(reg.sum()), termination=RA_MAX_ITERS, initial_cost=0.0,
               final_cost=0.0)

    ends = np.asarray(pairs, np.int64).reshape(-1, 2)

    def lin(R):
        W, g, err = np.zeros(len(pairs)), np.zeros((len(pairs), 3)), np.full(len(pairs), np.inf)
        u = np.flatnonzero(used)
        l, r = ends[u, 0], ends[u, 1]
        res = log_batch(np.matmul(np.swapaxes(R[r], 1, 2), np.matmul(Rp[u], R[l])))
        r2 = (res * res).sum(1)
        rho, w = bo.loss(loss, r2 / s2)
        W[u], g[u], err[u] = w, -w[:, None] * res, np.sqrt(r2) / DEG
        return W, g, err, float(np.sum(0.5 * (s2 * rho)))

    if not used.any():
        rep["termination"] = RA_NO_PAIRS
        return R, reg, np.full(len(pairs), np.inf), rep
    W, g, err, cost = lin(R)
    rep["initial_cost"] = cost
    for _ in range(max_iters):
        x = solve(n_sets, ends, W, g, root)
        for i in np.flatnonzero(reg):
            if i != root:
                R[i] = R[i] @ exp(x[i])
        rep["iterations"] += 1
        W, g, err, cost = lin(R)
        if np.sqrt((x * x).sum(1)).max() < step_tol * DEG:
            rep["termination"] = RA_STEP_TOL
            break
    rep["final_cost"] = cost
    return R, reg, err, rep


# ---- global positioning ----------------------------------------------------------------------------------------------

def obs(v, X, c):
    """gl_obs: (d, e) of rows"""
    u = X - c
    uu = (u * u).sum(-1)
    vu = (v * u).sum(-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.where(uu > 0.0, np.maximum(0.0, vu) / np.where(uu > 0.0, uu, 1.0), 0.0)
    return d, v - d[:, None] * u


class Positioning:
    """the used observations of a scene under rotations R and the registered flags (member order)"""

    def __init__(self, feats, cams, R, registered, start, members, loss="huber", loss_scale=0.1, solve=laplacian_solve):
        """solve(n, ends, W, g, root, n_cam) solves each Laplacian system: laplacian_solve (dense), or for large scenes
        laplacian_solve_reduced, the point nodes eliminated"""
        self.solve = solve
        n_feat = [len(f) for f in feats]
        off = np.concatenate([[0], np.cumsum(n_feat)]).astype(np.int64)
        allxy = np.concatenate([np.asarray(f, np.float32).reshape(-1, 2) for f in feats])
        members = np.asarray(members, np.int64)
        self.start = np.asarray(start, np.int64)
        self.S, self.T = len(feats), len(self.start) - 1
        self.set = np.searchsorted(off, members, side="right") - 1
        self.track = np.repeat(np.arange(self.T), np.diff(self.start))
        self.R = np.asarray(R, np.float64).reshape(-1, 3, 3)
        cams = np.asarray(cams, np.float32).reshape(-1, 4)
        xy = allxy[members]
        ok, self.v = tro.direction(cams[self.set], self.R[self.set], xy[:, 0], xy[:, 1])
        o = ok & np.asarray(registered, bool)[self.set]
        cnt = np.bincount(self.track, weights=o, minlength=self.T)
        self.tpart = cnt >= 2
        self.used = o & self.tpart[self.track]
        self.v = np.where(self.used[:, None], self.v, 0.0)
        self.positioned = np.bincount(self.set[self.used], minlength=self.S) > 0
        self.root = int(np.flatnonzero(self.positioned)[0]) if self.positioned.any() else -1
        self.ends = np.stack([self.S + self.track, self.set], 1)
        self.loss, self.s2 = loss, float(loss_scale) ** 2

    def lin(self, pos, init=False):
        """(W, g, cost) at positions pos (S + T, 3)"""
        X, c = pos[self.S + self.track], pos[self.set]
        if init:
            d, w = np.ones(len(X)), np.ones(len(X))
            e = self.v - (X - c)
            cost = 0.0
        else:
            d, e = obs(self.v, X, c)
            rho, w = bo.loss(self.loss, (e * e).sum(1) / self.s2)
            cost = float(np.sum(np.where(self.used, 0.5 * (self.s2 * rho), 0.0)))
        W = np.where(self.used, w * d * d, 0.0)
        g = np.where(self.used[:, None], e * (w * d)[:, None], 0.0)
        return W, g, cost

    def cost(self, pos):
        return self.lin(pos)[2]

    def step(self, pos, init=False):
        W, g, _ = self.lin(pos, init)
        return pos + self.solve(self.S + self.T, self.ends, W, g, self.root, n_cam=self.S)

    def extended_step(self, pos, max_doublings=20):
        """the header's iteration: the majorise-minimise step x, then pos + 2^k x for k = 1 .. 20 while the cost keeps
        decreasing (the device adds x, x, 2x, 4x, ... in place, so the two agree to rounding): (positions, cost)"""
        W, g, _ = self.lin(pos)
        x = self.solve(self.S + self.T, self.ends, W, g, self.root, n_cam=self.S)
        best = pos + x
        bc, a = self.cost(best), 1.0
        for _ in range(max_doublings):
            a *= 2.0
            cand = pos + a * x
            c = self.cost(cand)
            if not c < bc:
                break
            best, bc = cand, c
        return best, bc

    def run(self, max_iters=100, function_tol=1e-8):
        """(positions, report dict) of the header's loop"""
        pos = np.zeros((self.S + self.T, 3))
        rep = dict(iterations=0, termination=GP_MAX_ITERS, n_obs=int(self.used.sum()), n_points=int(self.tpart.sum()),
                   n_cams=int(self.positioned.sum()), initial_cost=0.0, final_cost=0.0)
        if not self.used.any():
            rep["termination"] = GP_NO_OBSERVATIONS
            return pos, rep
        pos = self.step(pos, init=True)
        cost = self.cost(pos)
        rep["initial_cost"] = cost
        for _ in range(max_iters):
            pos, new = self.extended_step(pos)
            rep["iterations"] += 1
            small = not (cost - new >= function_tol * cost)
            cost = new
            if small:
                rep["termination"] = GP_FUNCTION_TOL
                break
        rep["final_cost"] = cost
        return pos, rep

    def outputs(self, pos):
        """(poses [(R, t)], X (T, 3)) after the header's scaling"""
        c = pos[:self.S]
        ss = float((c[self.positioned] ** 2).sum())
        n = int(self.positioned.sum())
        scale = 1.0 / math.sqrt(ss / n) if n > 1 and ss > 0.0 else 1.0
        poses = [(self.R[i], -(self.R[i] @ (scale * c[i])) if self.positioned[i] else np.zeros(3)) for i in range(self.S)]
        X = np.where(self.tpart[:, None], scale * pos[self.S:], 0.0)
        return poses, X

    def free_gradient(self, pos, h=1e-7):
        """central differences of the reduced cost over every free coordinate (root and unpositioned nodes excluded)"""
        nodes = [i for i in range(self.S) if self.positioned[i] and i != self.root] + [self.S + t for t in np.flatnonzero(self.tpart)]
        gr = []
        for n in nodes:
            for k in range(3):
                a, b = pos.copy(), pos.copy()
                a[n, k] += h
                b[n, k] -= h
                gr.append((self.cost(a) - self.cost(b)) / (2 * h))
        return np.array(gr)


# ---- planted view graphs and alignment -------------------------------------------------------------------------------

def random_rotation(rng):
    """a uniform random rotation from a unit quaternion"""
    w, x, y, z = rng.normal(size=4)
    n = math.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def view_graph(rng, n_cams, n_pairs, noise_deg=0.5, outliers=0.2, hub=None):
    """random true rotations, n_pairs distinct pairs over a connected graph (a random tree first), R_p = R_r R_l^T turned
    by noise_deg about a random axis, or a random rotation for the outlier fraction; n_front from 30 to 500, outliers
    below 100.  hub = (node, degree): that node gets pairs with `degree` distinct others (added after the tree).
    Returns (R_true, pairs, Rp, n_front, is_outlier)."""
    Rt = np.stack([random_rotation(rng) for _ in range(n_cams)])
    perm = rng.permutation(n_cams)
    edges = set()
    for i in range(1, n_cams):
        j = int(rng.integers(0, i))
        a, b = int(perm[i]), int(perm[j])
        edges.add((min(a, b), max(a, b)))
    if hub is not None:
        h, deg = hub
        others = [int(o) for o in rng.permutation(n_cams) if o != h]
        have = {a if b == h else b for a, b in edges if h in (a, b)}
        for o in others:
            if len(have) >= deg:
                break
            have.add(o)
            edges.add((min(h, o), max(h, o)))
    while len(edges) < n_pairs:
        a, b = rng.choice(n_cams, 2, replace=False)
        edges.add((int(min(a, b)), int(max(a, b))))
    pairs = sorted(edges)
    out = rng.random(len(pairs)) < outliers
    Rp, nf = [], []
    for (l, r), o in zip(pairs, out):
        if o:
            Rp.append(random_rotation(rng))
            nf.append(int(rng.integers(15, 100)))
        else:
            Rp.append(bo.small_rotation(rng, noise_deg) @ Rt[r] @ Rt[l].T)
            nf.append(int(rng.integers(30, 500)))
    return Rt, pairs, np.stack(Rp), np.array(nf), out


def rotation_errors(R, Rt):
    """per-rotation angles (degrees, |Log|) after the best global alignment R_i ~ Rt_i G (G from the SVD of sum Rt^T R)"""
    M = sum(np.asarray(b).T @ np.asarray(a) for a, b in zip(R, Rt))
    U, _, Vt = np.linalg.svd(M)
    G = U @ np.diag([1.0, 1.0, np.linalg.det(U @ Vt)]) @ Vt
    return np.array([math.degrees(np.linalg.norm(log(np.asarray(a) @ (np.asarray(b) @ G).T))) for a, b in zip(R, Rt)])


def align_centres(C, Ct):
    """the similarity (s, Q, o) minimising sum |s Q C_i + o - Ct_i|^2 (Umeyama); returns the aligned centres"""
    C, Ct = np.asarray(C, np.float64), np.asarray(Ct, np.float64)
    mc, mt = C.mean(0), Ct.mean(0)
    A, B = C - mc, Ct - mt
    U, sv, Vt = np.linalg.svd(B.T @ A)
    D = np.diag([1.0, 1.0, np.linalg.det(U @ Vt)])
    Q = U @ D @ Vt
    s = np.trace(np.diag(sv) @ D) / (A * A).sum()
    return s * (Q @ A.T).T + mt
