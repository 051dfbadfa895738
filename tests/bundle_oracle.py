"""Float64 numpy statement of ps_bundle_adjust (include/popsift_b200_bundle.h) for the tests; nothing in the package
imports it.

The residual is triangulate_oracle's; the pose and point Jacobians, the three losses, the cost and its IRLS gradient, one
Levenberg-Marquardt step by a dense solve of the whole damped system (and by the Schur complement onto the cameras, for
checking the dense one), and a dense LM to convergence for small problems follow the header's rules.  The device solves
the same system by preconditioned CG, so the two agree to the CG tolerance, not bit for bit.  It also plants scenes:
triangulate_oracle.planted_scene with the poses and points perturbed."""
from __future__ import annotations

import math

import numpy as np

import triangulate_oracle as tro

LOSSES = ("squared", "huber", "cauchy")
MAX_ITERS, FUNCTION_TOL, LAMBDA, NO_OBSERVATIONS, NONFINITE_START = range(5)


# ---- per observation (k_bundle.h) ------------------------------------------------------------------------------------

def loss(kind, z):
    """(rho(z), rho'(z)) elementwise"""
    z = np.asarray(z, np.float64)
    if kind == "huber":
        r = np.sqrt(np.maximum(z, 1.0))
        return np.where(z <= 1.0, z, 2.0 * r - 1.0), np.where(z <= 1.0, 1.0, 1.0 / r)
    if kind == "cauchy":
        return np.log1p(z), 1.0 / (1.0 + z)
    return z.copy(), np.ones_like(z)


def jacobian(cam, R, t, X, x, y):
    """(front, e (U, 2), Jc (U, 2, 6), Jp (U, 2, 3)) of observations: cam (U, 4), R (U, 3, 3), t (U, 3), X (U, 3)"""
    front, ex, ey, Jx, Jy = tro.residual(cam, R, t, X, x, y, jac=True)
    c = np.asarray(cam, np.float32).astype(np.float64)
    fx, fy = c[:, 0], c[:, 1]
    Xc = np.stack([R[:, r, 0] * X[:, 0] + R[:, r, 1] * X[:, 1] + R[:, r, 2] * X[:, 2] + t[:, r] for r in range(3)], 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        iz = 1.0 / Xc[:, 2]
        p, q = Xc[:, 0] * iz, Xc[:, 1] * iz
    v = Xc - t
    zero = np.zeros_like(iz)
    a = np.stack([np.stack([fx * iz, zero, -(fx * p) * iz], 1), np.stack([zero, fy * iz, -(fy * q) * iz], 1)], 1)   # (U, 2, 3)
    Jc = np.zeros((len(iz), 2, 6))
    for r in range(2):
        ar = a[:, r]
        Jc[:, r, 0] = v[:, 1] * ar[:, 2] - v[:, 2] * ar[:, 1]
        Jc[:, r, 1] = v[:, 2] * ar[:, 0] - v[:, 0] * ar[:, 2]
        Jc[:, r, 2] = v[:, 0] * ar[:, 1] - v[:, 1] * ar[:, 0]
        Jc[:, r, 3:] = ar
    return front, np.stack([ex, ey], 1), Jc, np.stack([Jx, Jy], 1)


def rodrigues(w):
    w = np.asarray(w, np.float64)
    th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2]
    if th2 < 1e-16:
        A, B = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        th = math.sqrt(th2)
        A, B = math.sin(th) / th, (1.0 - math.cos(th)) / th2
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.eye(3) + A * W + B * (np.outer(w, w) - th2 * np.eye(3))


def pose_update(R, t, d):
    E = rodrigues(d[:3])
    Rn = np.array([[E[i, 0] * R[0, j] + E[i, 1] * R[1, j] + E[i, 2] * R[2, j] for j in range(3)] for i in range(3)])
    return Rn, np.asarray(t, np.float64) + np.asarray(d[3:], np.float64)


def damp(d, lam):
    return d + lam * np.minimum(np.maximum(d, 1e-6), 1e32)


# ---- a problem -------------------------------------------------------------------------------------------------------

class Problem:
    """the used observations of a scene (member order), the cameras, the fixed flags and the gauge"""

    def __init__(self, feats, cams, start, members, status, mask, fixed, loss_kind="squared", loss_scale=1.0, scale_set=-1, scale_axis=0):
        n_feat = [len(f) for f in feats]
        off = np.concatenate([[0], np.cumsum(n_feat)]).astype(np.int64)
        allxy = np.concatenate([np.asarray(f, np.float32).reshape(-1, 2) for f in feats])
        members = np.asarray(members, np.int64)
        start = np.asarray(start, np.int64)
        track = np.repeat(np.arange(len(start) - 1), np.diff(start))
        used = (np.asarray(status)[track] == tro.OK) & (np.asarray(mask) != 0)
        self.S, self.T = len(feats), len(start) - 1
        self.set = (np.searchsorted(off, members, side="right") - 1)[used]
        self.track = track[used]
        self.xy = allxy[members[used]]
        self.cams = np.asarray(cams, np.float32).reshape(-1, 4)
        self.fixed = np.asarray(fixed, bool)
        self.loss, self.s = loss_kind, float(loss_scale)
        has = np.bincount(self.set, minlength=self.S) > 0
        self.free = [i for i in range(self.S) if not self.fixed[i] and has[i]]
        self.points = np.unique(self.track)
        self.held = {scale_set: 3 + scale_axis} if scale_set >= 0 and not self.fixed[scale_set] else {}
        # parameter columns: each free camera's 6 (minus a held one), then each point's 3
        self.cam_cols, col = {}, 0
        for i in self.free:
            cols = [col + k if k != self.held.get(i, -1) else -1 for k in range(6)]
            col += sum(c >= 0 for c in cols)
            self.cam_cols[i] = cols
        self.n_cam = col
        self.pt_col = {int(j): col + 3 * k for k, j in enumerate(self.points)}
        self.n = col + 3 * len(self.points)

    def residuals(self, poses, X):
        R = np.stack([np.asarray(p[0], np.float64) for p in poses])[self.set]
        t = np.stack([np.asarray(p[1], np.float64) for p in poses])[self.set]
        return jacobian(self.cams[self.set], R, t, np.asarray(X, np.float64)[self.track], self.xy[:, 0], self.xy[:, 1])

    def cost(self, poses, X):
        front, e, _, _ = self.residuals(poses, X)
        if not front.all():
            return math.inf
        s2 = self.s * self.s
        rho, _ = loss(self.loss, (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) / s2)
        return float(np.sum(0.5 * (s2 * rho)))

    def system(self, poses, X):
        """(J (2U, n) weighted by sqrt(w), e (2U,) weighted): H = J^T J, g = J^T e"""
        front, e, Jc, Jp = self.residuals(poses, X)
        s2 = self.s * self.s
        _, w = loss(self.loss, (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) / s2)
        sw = np.sqrt(w)
        U = len(self.set)
        J = np.zeros((2 * U, self.n))
        for u in range(U):
            i, j = int(self.set[u]), int(self.track[u])
            for r in range(2):
                if i in self.cam_cols:
                    for k, c in enumerate(self.cam_cols[i]):
                        if c >= 0:
                            J[2 * u + r, c] = sw[u] * Jc[u, r, k]
                J[2 * u + r, self.pt_col[j]:self.pt_col[j] + 3] = sw[u] * Jp[u, r]
        return J, (e * sw[:, None]).reshape(-1)

    def gradient(self, poses, X):
        J, e = self.system(poses, X)
        return J.T @ e

    def apply(self, poses, X, d):
        poses = [(np.asarray(R, np.float64).copy(), np.asarray(t, np.float64).copy()) for R, t in poses]
        X = np.asarray(X, np.float64).copy()
        for i, cols in self.cam_cols.items():
            di = np.array([d[c] if c >= 0 else 0.0 for c in cols])
            poses[i] = pose_update(poses[i][0], poses[i][1], di)
        X[self.points] = X[self.points] + np.asarray(d[self.n_cam:], np.float64).reshape(-1, 3)
        return poses, X

    def step(self, poses, X, lam, schur=False):
        """one damped step: (d, pred)"""
        J, e = self.system(poses, X)
        H, g = J.T @ J, J.T @ e
        Hd = H.copy()
        Hd[np.diag_indices(self.n)] = damp(np.diag(H), lam)
        d = schur_solve(Hd, -g, self.n_cam) if schur else np.linalg.solve(Hd, -g)
        pred = -(g @ d + 0.5 * d @ H @ d)
        return d, pred

    def schur_step(self, poses, X, lam):
        """step()'s damped step by the Schur complement onto the cameras, vectorised: (d, pred, ReducedSystem)"""
        sys_ = ReducedSystem(self, poses, X, lam)
        d = sys_.solve()
        return d, sys_.pred(d), sys_


class ReducedSystem:
    """One LM step's reduced camera system S x = b (S = U + lambda D - sum_j W_j V_j^-1 W_j^T, the points eliminated),
    assembled without a dense Jacobian: per-set blocks U_i and g_i, per-track blocks V_j and g_j with step()'s damping, and
    S from every within-track pair of observations.  The columns are the problem's camera columns (a held component and
    the fixed and unobserved sets have none)."""

    def __init__(self, prob, poses, X, lam):
        front, e, Jc, Jp = prob.residuals(poses, X)
        _, w = loss(prob.loss, (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) / (prob.s * prob.s))
        sw = np.sqrt(w)
        e, Jc, Jp = e * sw[:, None], Jc * sw[:, None, None], Jp * sw[:, None, None]
        # camera columns: cam[u, k] is the column of observation u's pose component k, or -1
        colmap = np.full((prob.S, 6), -1, np.int64)
        for i, cols in prob.cam_cols.items():
            colmap[i] = cols
        cam = colmap[prob.set]
        Jc = np.where((cam >= 0)[:, None, :], Jc, 0.0)
        self.prob, self.nc, self.cam = prob, prob.n_cam, cam
        nc = self.nc
        # points: k = the index of observation u's point among prob.points
        pk = np.searchsorted(prob.points, prob.track)
        nP = len(prob.points)
        self.pk, self.Jc, self.Jp, self.e = pk, Jc, Jp, e
        V = np.zeros((nP, 3, 3))
        np.add.at(V, pk, np.einsum("ura,urb->uab", Jp, Jp))
        self.gp = np.zeros((nP, 3))
        np.add.at(self.gp, pk, np.einsum("ura,ur->ua", Jp, e))
        Vd = V.copy()
        for a in range(3):
            Vd[:, a, a] = damp(V[:, a, a], lam)
        self.Vi = np.linalg.inv(Vd)
        # U and g over the camera columns (observation u's 6 x 6 block scattered to its columns)
        Wu = np.einsum("ura,urb->uab", Jc, Jp)                 # (U, 6, 3): Jc^T Jp
        self.Wu = Wu
        gc_u = np.einsum("ura,ur->ua", Jc, e)
        self.gc = np.bincount(cam[cam >= 0], weights=gc_u[cam >= 0], minlength=nc)
        Uu = np.einsum("ura,urb->uab", Jc, Jc)
        ok = (cam[:, :, None] >= 0) & (cam[:, None, :] >= 0)
        flat = (cam[:, :, None] * nc + cam[:, None, :])[ok]
        Uc = np.bincount(flat, weights=Uu[ok], minlength=nc * nc).reshape(nc, nc)
        self.Ud = Uc.copy()
        self.Ud[np.diag_indices(nc)] = damp(np.diag(Uc), lam)
        self.Uc = Uc
        # S = Ud - sum over within-track pairs (u, v) of W_u Vi W_v^T; b = -g_c + sum_u W_u Vi g_p
        WVi = np.einsum("uab,ubc->uac", Wu, self.Vi[pk])      # (U, 6, 3)
        self.WVi = WVi
        bu = np.einsum("uab,ub->ua", WVi, self.gp[pk])
        self.b = -self.gc + np.bincount(cam[cam >= 0], weights=bu[cam >= 0], minlength=nc)
        start = np.searchsorted(pk, np.arange(nP + 1))          # observations are track-major, so each point's are a run
        L = np.diff(start)
        S = self.Ud.copy().reshape(-1)
        for n in np.unique(L):                                  # tracks of one length at a time, in chunks
            tr = np.flatnonzero(L == n)
            for c0 in range(0, len(tr), max(1, 200000 // (n * n))):
                base = start[tr[c0:c0 + max(1, 200000 // (n * n))]]
                uu = (base[:, None, None] + np.arange(n)[None, :, None]).repeat(n, 2).reshape(-1)
                vv = (base[:, None, None] + np.arange(n)[None, None, :]).repeat(n, 1).reshape(-1)
                blk = np.einsum("pac,pbc->pab", WVi[uu], Wu[vv])
                ca, cb = cam[uu][:, :, None], cam[vv][:, None, :]
                m = (ca >= 0) & (cb >= 0)
                S -= np.bincount((ca * nc + cb)[m], weights=blk[m], minlength=nc * nc)
        self.S = S.reshape(nc, nc)
        self.pstart = start

    def solve(self):
        """the damped step in the problem's columns: the cameras by Cholesky, then the points by back-substitution"""
        from scipy.linalg import cho_factor, cho_solve
        xc = cho_solve(cho_factor(self.S), self.b) if self.nc else np.zeros(0)
        return np.concatenate([xc, self.back(xc).reshape(-1)])

    def back(self, xc):
        """the points' step for a camera step xc: dX_j = -Vi_j (g_j + sum_u W_u^T xc)"""
        xu = np.where(self.cam >= 0, np.asarray(xc, np.float64)[np.maximum(self.cam, 0)], 0.0)
        s = np.zeros((len(self.Vi), 3))
        np.add.at(s, self.pk, np.einsum("uab,ua->ub", self.Wu, xu))
        return -np.einsum("jab,jb->ja", self.Vi, self.gp + s)

    def pred(self, d):
        """-(g.d + 1/2 d^T H d) of the undamped H = J^T J"""
        xc, dX = d[:self.nc], d[self.nc:].reshape(-1, 3)
        xu = np.where(self.cam >= 0, np.asarray(xc, np.float64)[np.maximum(self.cam, 0)], 0.0)
        Jd = np.einsum("ura,ua->ur", self.Jc, xu) + np.einsum("ura,ua->ur", self.Jp, dX[self.pk])
        return -(self.gc @ xc + (self.gp * dX).sum() + 0.5 * (Jd * Jd).sum())


def schur_step(prob, poses, X, lam):
    """(d, pred) of Problem.schur_step, for lm(solve=...)"""
    return prob.schur_step(poses, X, lam)[:2]


def schur_solve(A, b, nc):
    """A x = b by the Schur complement onto the first nc unknowns, the rest 3 x 3 blocks"""
    U, W, V = A[:nc, :nc], A[:nc, nc:], A[nc:, nc:]
    Vi = np.zeros_like(V)
    for k in range(0, V.shape[0], 3):
        Vi[k:k + 3, k:k + 3] = np.linalg.inv(V[k:k + 3, k:k + 3])
    bc, bp = b[:nc], b[nc:]
    S = U - W @ Vi @ W.T
    xc = np.linalg.solve(S, bc - W @ Vi @ bp) if nc else np.zeros(0)
    xp = Vi @ (bp - W.T @ xc)
    return np.concatenate([xc, xp])


def lm(prob, poses, X, max_iters=50, function_tol=1e-6, initial_lambda=1e-4, solve=None):
    """the header's LM, each step by solve(prob, poses, X, lambda) -> (d, pred) (default the dense Problem.step; schur_step
    for large problems): (poses, X, report dict)"""
    solve = solve or (lambda p, po, x, lam: p.step(po, x, lam))
    X = np.asarray(X, np.float64).copy()
    rep = dict(iterations=0, accepted=0, termination=MAX_ITERS)
    if len(prob.set) == 0:
        rep.update(termination=NO_OBSERVATIONS, initial_cost=0.0, final_cost=0.0)
        return poses, X, rep
    cost = prob.cost(poses, X)
    rep.update(initial_cost=cost, final_cost=cost)
    if not math.isfinite(cost):
        rep["termination"] = NONFINITE_START
        return poses, X, rep
    lam, nu = float(initial_lambda), 2.0
    for _ in range(max_iters):
        d, pred = solve(prob, poses, X, lam)
        pn, Xn = prob.apply(poses, X, d)
        nc = prob.cost(pn, Xn)
        rep["iterations"] += 1
        if math.isfinite(nc) and nc < cost:
            rho = (cost - nc) / pred if pred != 0 else math.inf
            c = 2.0 * rho - 1.0
            f = max(1.0 / 3.0, 1.0 - c * c * c) if pred > 0 and math.isfinite(rho) else 1.0 / 3.0
            small = cost - nc < function_tol * cost
            lam *= f
            nu = 2.0
            cost, poses, X = nc, pn, Xn
            rep["accepted"] += 1
            if small:
                rep["termination"] = FUNCTION_TOL
                break
        else:
            lam *= nu
            nu *= 2.0
        if lam > 1e32:
            rep["termination"] = LAMBDA
            break
    rep["final_cost"] = cost
    return poses, X, rep


# ---- planted scenes --------------------------------------------------------------------------------------------------

def small_rotation(rng, deg):
    w = rng.normal(size=3)
    w *= math.radians(deg) / np.linalg.norm(w)
    return rodrigues(w)


def planted(rng, n_cams, lengths, noise=0.5, outliers=0.0, rot_deg=1.0, trans=0.2, point_sigma=0.02, **kw):
    """triangulate_oracle.planted_scene (cameras on a sphere of radius 10 around a cloud of spread 2; sets= gives every
    track's cameras) with every pose
    turned by rot_deg about a random axis and its t moved by `trans` (about 2 % of the scene scale) in a random direction,
    and every point moved by point_sigma per axis.  Adds poses_true, X0 (the perturbed points), status (all OK) and mask
    (all 1)."""
    sc = tro.planted_scene(rng, n_cams, lengths, noise=noise, outliers=outliers, **kw)
    sc["poses_true"] = [(R.copy(), t.copy()) for R, t in sc["poses"]]
    pert = []
    for R, t in sc["poses"]:
        dt = rng.normal(size=3)
        dt *= trans / np.linalg.norm(dt)
        pert.append((small_rotation(rng, rot_deg) @ R, t + dt))
    sc["poses"] = pert
    sc["X0"] = sc["Xtrue"] + rng.normal(scale=point_sigma, size=sc["Xtrue"].shape)
    sc["status"] = np.zeros(len(lengths), np.int32)
    sc["mask"] = np.ones(len(sc["members"]), np.uint8)
    return sc


def gauge_to_truth(sc, fixed_set=0, scale_set=1, scale_axis=0):
    """set the fixed set's pose and the held component of scale_set's t to their true values, so that the gauge the call
    holds is the truth's and the recovered poses can be compared with the truth directly"""
    sc["poses"][fixed_set] = sc["poses_true"][fixed_set]
    R, t = sc["poses"][scale_set]
    t = np.asarray(t, np.float64).copy()
    t[scale_axis] = sc["poses_true"][scale_set][1][scale_axis]
    sc["poses"][scale_set] = (R, t)


def problem(sc, fixed, **kw):
    return Problem(sc["feats"], sc["cams"], sc["start"], sc["members"], sc["status"], sc["mask"], fixed, **kw)


def pose_errors(poses, truth):
    """(rotation angle in degrees, centre distance) per pose"""
    rot, cen = [], []
    for (R, t), (Rt, tt) in zip(poses, truth):
        c = np.clip((np.trace(np.asarray(R) @ np.asarray(Rt).T) - 1.0) / 2.0, -1.0, 1.0)
        rot.append(math.degrees(math.acos(c)))
        cen.append(float(np.linalg.norm(-np.asarray(R).T @ t + np.asarray(Rt).T @ tt)))
    return np.array(rot), np.array(cen)
