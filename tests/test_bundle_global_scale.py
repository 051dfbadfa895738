"""ps_bundle_adjust, ps_global_positioning and ps_rotation_averaging on the GPU at the shapes where their kernels change how
they split the work (tests/scale_shapes.py: set and node loops past 256, per-set CTAs past 128 observations, more than one
per-track partial, more than 256 partials, two radix passes, more than one radix tile and scan block), against the
float64 oracles with the points eliminated (bundle_oracle.ReducedSystem, global_oracle.LaplacianSystem).

What is compared:
- exactly: the counts of the reports, the registered / positioned flags, termination, accepted steps and iterations, the
  guard bytes around every output (run_device / run_pos / run_rot);
- the starting cost within the summation bound n 2^-53 (relative) of n positive terms;
- one step (cg_tol = 1e-14): the device's step, read back from its outputs, in the oracle's reduced system (check_step);
- obs_error to float32 rounding of the float64 pixel error at the device's own output, +inf outside OK tracks;
- three iterations: the same steps accepted, costs within 1e-9;
- determinism on the largest scenes: two calls give the same bytes."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bundle_oracle as bo                # noqa: E402
import global_oracle as go                # noqa: E402
import scale_shapes as ss                 # noqa: E402
import triangulate_oracle as tro          # noqa: E402
from popsift_b200 import api              # noqa: E402
from test_bundle import run_device, _pts  # noqa: E402
from test_global import run_pos, run_rot  # noqa: E402

pytestmark = pytest.mark.gpu

U53 = 2.0 ** -53
CG_TOL, CG_MAX = 1e-14, 5000


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


@pytest.fixture(scope="module")
def scenes():
    """every scene and view graph of the table, built once and shared by the rows that use it"""
    cache = {}

    def get(row):
        kind, name = ss.ROWS[row][:2]
        key = (kind == "rotation", name)
        if key not in cache:
            cache[key] = (ss.GRAPHS if kind == "rotation" else ss.SCENES)[name]()
        return cache[key]
    return get


def check_step(S, b, x_dev, x_or, cg_iters, n_terms, scale, inflate=1.0):
    """The device's step x_dev against the oracle's x_or = S^-1 b; returns the bound on |x_dev - x_or|_2.

    CG stops once its recursive residual is at most cg_tol |b|.  The true residual |S x_dev - b| differs from it by the
    rounding of the cg_iters updates and of the n_terms-term sums that form S and b, each at most about n 2^-53 of
    scale |x| + |b|, where `scale` bounds the magnitude of the summed terms (|U + lambda D| for the bundle, the largest
    degree for a Laplacian; Higham's gamma_n, and the residual-gap bound of finite-precision CG).  So
        |r| <= cg_tol |b| + 4 (cg_iters + n_terms) 2^-53 (scale |x| + |b|)        (asserted)
    and, S being symmetric positive definite, the error e = x_dev - x_or has
        |e|_S = sqrt(r^T S^-1 r) <= |r| / sqrt(lambda_min)                            (asserted)
        |e|_inf <= |e|_2 <= |e|_S / sqrt(lambda_min)                                   (returned)
    `inflate` multiplies the residual bound where x_dev is not the solver's own iterate (see test_positioning_rows)."""
    x_dev, x_or, b = np.ravel(x_dev), np.ravel(x_or), np.ravel(b)
    n = len(x_dev)
    Sk = np.kron(S, np.eye(len(b) // len(S))) if len(b) != len(S) else S
    r = Sk @ x_dev - b
    lmin = float(np.linalg.eigvalsh(S)[0])
    bound = inflate * (CG_TOL * np.linalg.norm(b)) + inflate * 4 * (cg_iters + n_terms) * U53 * (scale * np.linalg.norm(x_dev) + np.linalg.norm(b))
    rn = float(np.linalg.norm(r))
    e = x_dev - x_or
    eS = math.sqrt(max(float(e @ (Sk @ e)), 0.0))
    print("step: %d unknowns, |r| %.3g (bound %.3g), |r|/|b| %.3g, |e|_S %.3g, lambda_min %.3g, cg %d" %
          (n, rn, bound, rn / np.linalg.norm(b), eS, lmin, cg_iters))
    assert rn <= bound, (rn, bound)
    assert eS <= rn / math.sqrt(lmin) * (1 + 1e-6) + 1e-300
    return eS / math.sqrt(lmin)


# ---- bundle adjustment ----

BUNDLE_ROWS = [r for r in ss.ROWS if ss.ROWS[r][0] == "bundle"]
BA_KW = dict(loss="huber", loss_scale=2.0, initial_lambda=1e-3)


def _held(sc):
    """the first free set with observations holds its t[2]"""
    return int(np.flatnonzero(sc["fixed"] == 0)[0]), 2


@pytest.mark.parametrize("row", BUNDLE_ROWS)
def test_bundle_rows(lib, scenes, row):
    sc = scenes(row)
    fixed = sc["fixed"]
    hs, ha = _held(sc)
    kw = dict(BA_KW, scale_set=hs, scale_axis=ha)
    prob = bo.problem(sc, fixed, loss_kind=kw["loss"], loss_scale=kw["loss_scale"], scale_set=hs, scale_axis=ha)
    M = len(sc["members"])
    # one step
    rc, poses, raw, err, rep = run_device(lib, sc, fixed, api._bundle_params(max_iters=1, cg_tol=CG_TOL, cg_max_iters=CG_MAX, **kw))
    assert rc == 0, api._last_error(lib)
    assert rep.n_obs == len(prob.set) == M and rep.n_points == len(prob.points) and rep.n_free_cams == len(prob.free)
    assert rep.cg_iterations < CG_MAX, "CG stopped on the count, not on cg_tol"
    c0 = prob.cost(sc["poses"], sc["X0"])
    assert abs(rep.initial_cost - c0) <= M * U53 * c0
    d, pred, sy = prob.schur_step(sc["poses"], sc["X0"], kw["initial_lambda"])
    pn, Xn = prob.apply(sc["poses"], sc["X0"], d)
    c1 = prob.cost(pn, Xn)
    assert c1 < c0                      # the planted perturbation: the first step is accepted, so the outputs carry it
    assert rep.iterations == 1 and rep.termination == bo.MAX_ITERS and rep.accepted == int(c1 < c0)
    # the device's step from its outputs: log(R_new R^T) and dt per free set, dX per point
    xc = np.zeros(prob.n_cam)
    tmax = 1.0
    for i, cols in prob.cam_cols.items():
        (R0, t0), (R1, t1) = sc["poses"][i], poses[i]
        v = np.r_[go.log(R1 @ np.asarray(R0).T), t1 - t0]
        tmax = max(tmax, float(np.abs(t0).max()))
        for k, c in enumerate(cols):
            if c >= 0:
                xc[c] = v[k]
            else:
                assert t1[k - 3] == sc["poses"][i][1][k - 3]        # the held component, bit for bit
    for i in range(len(poses)):
        if i not in prob.cam_cols:
            assert poses[i][0].tobytes() == np.asarray(sc["poses"][i][0]).tobytes()
            assert poses[i][1].tobytes() == np.asarray(sc["poses"][i][1]).tobytes()
    n_max = int(np.bincount(prob.set, minlength=prob.S).max())
    scale = float(np.abs(np.linalg.eigvalsh(sy.Ud)).max())
    e2 = check_step(sy.S, sy.b, xc, d[:prob.n_cam], rep.cg_iterations, n_max, scale)
    # poses: |e|_inf <= |e|_2, plus the rounding of reading the step back (a few 2^-53 of |R| = 1 and of |t|)
    assert np.abs(xc - d[:prob.n_cam]).max() <= e2 + 16 * U53 * tmax
    # points: dX_dev - dX_or = (back(xc_dev) - back(xc_or)), the camera error carried through the back-substitution
    # (computed exactly here), plus the rounding of a 3 x 3 solve of condition kappa_j on sums of a few hundred terms
    X0 = np.asarray(sc["X0"])[prob.points]
    dXd = _pts(raw)["X"][prob.points] - X0
    dXo = d[prob.n_cam:].reshape(-1, 3)
    prop = np.abs(sy.back(xc) - sy.back(d[:prob.n_cam])).max(1)
    kap = np.linalg.cond(sy.Vi)
    tol = prop + 1024 * U53 * kap * np.abs(dXo).max(1) + 4 * U53 * np.abs(X0).max(1)
    assert (np.abs(dXd - dXo).max(1) <= tol).all(), float((np.abs(dXd - dXo).max(1) / tol).max())
    # obs_error: the float64 pixel error at the device's output, rounded to float32
    off = np.cumsum([0] + [len(f) for f in sc["feats"]])
    mset = np.searchsorted(off, sc["members"], side="right") - 1
    xy = np.concatenate([np.asarray(f, np.float32).reshape(-1, 2) for f in sc["feats"]])[sc["members"]]
    track = np.repeat(np.arange(len(sc["start"]) - 1), np.diff(sc["start"]))
    Rs = np.stack([p[0] for p in poses])[mset]
    ts = np.stack([p[1] for p in poses])[mset]
    _, e2o = tro.error2(sc["cams"][mset], Rs, ts, _pts(raw)["X"][track], xy[:, 0], xy[:, 1])
    eo = np.sqrt(e2o)
    ed = err.view(np.float32).astype(np.float64)
    assert (np.abs(ed - eo) <= 2.0 ** -24 * eo + 1e-10).all()
    # three iterations: the same steps accepted, the same costs
    rc, poses3, raw3, _, rep3 = run_device(lib, sc, fixed, api._bundle_params(max_iters=3, cg_tol=1e-12, cg_max_iters=CG_MAX, **kw))
    _, _, orep = bo.lm(prob, sc["poses"], sc["X0"], max_iters=3, function_tol=kw.get("function_tol", 1e-6),
                       initial_lambda=kw["initial_lambda"], solve=bo.schur_step)
    print(row, "device", rep3.initial_cost, rep3.final_cost, rep3.iterations, rep3.accepted, rep3.cg_iterations, "oracle", orep)
    assert rc == 0 and (rep3.iterations, rep3.accepted, rep3.termination) == (orep["iterations"], orep["accepted"], orep["termination"])
    assert abs(rep3.final_cost - orep["final_cost"]) <= 1e-9 * orep["final_cost"]


def test_bundle_large_masked_and_deterministic(lib, scenes):
    """the large scene with masked members and non-OK tracks: the counts, +inf outside OK tracks, and two calls give the
    same bytes"""
    sc = dict(scenes("ba_large"))
    sc["mask"] = sc["mask"].copy()
    sc["mask"][::89] = 0
    sc["status"] = sc["status"].copy()
    sc["status"][::97] = tro.TOO_FEW_INLIERS
    hs, ha = _held(sc)
    prm = api._bundle_params(max_iters=3, cg_tol=1e-10, cg_max_iters=500, scale_set=hs, scale_axis=ha, **BA_KW)
    a = run_device(lib, sc, sc["fixed"], prm)
    b = run_device(lib, sc, sc["fixed"], prm)
    assert a[0] == 0
    prob = bo.problem(sc, sc["fixed"], loss_kind="huber", loss_scale=2.0, scale_set=hs, scale_axis=ha)
    rep = a[4]
    assert rep.n_obs == len(prob.set) and rep.n_points == len(prob.points) and rep.n_free_cams == len(prob.free)
    c0 = prob.cost(sc["poses"], sc["X0"])
    assert abs(rep.initial_cost - c0) <= len(prob.set) * U53 * c0
    track = np.repeat(np.arange(len(sc["start"]) - 1), np.diff(sc["start"]))
    bad = sc["status"][track] != tro.OK
    e = a[3].view(np.float32)
    assert np.isinf(e[bad]).all() and np.isfinite(e[~bad]).all()
    assert a[2].tobytes() == b[2].tobytes() and a[3].tobytes() == b[3].tobytes() and bytes(a[4]) == bytes(b[4])
    assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(a[1], b[1]))


# ---- global positioning ----

POSITION_ROWS = [r for r in ss.ROWS if ss.ROWS[r][0] == "position"]
GP_KW = dict(loss="huber", loss_scale=0.1)


@pytest.mark.parametrize("row", POSITION_ROWS)
def test_positioning_rows(lib, scenes, row):
    sc = scenes(row)
    S = len(sc["feats"])
    P = go.Positioning(sc["feats"], sc["cams"], sc["R"], np.ones(S, bool), sc["start"], sc["members"], solve=go.laplacian_solve_reduced, **GP_KW)
    # the first solve (d = 1, unit weights) with cg_tol = 1e-14
    rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(max_iters=0, cg_tol=CG_TOL, cg_max_iters=CG_MAX, function_tol=0.0, **GP_KW))
    assert rc == 0, api._last_error(lib)
    assert (rep.n_obs, rep.n_points, rep.n_cams) == (int(P.used.sum()), int(P.tpart.sum()), int(P.positioned.sum()))
    assert np.array_equal(pos.astype(bool), P.positioned) and rep.iterations == 0
    assert rep.cg_iterations < CG_MAX, "CG stopped on the count, not on cg_tol"
    W, g, _ = P.lin(np.zeros((P.S + P.T, 3)), init=True)
    sy = go.LaplacianSystem(P.S + P.T, P.ends, W, g, P.root, n_cam=P.S)
    xo = sy.solve()
    _, Xo = P.outputs(xo)
    # the outputs are scaled to RMS centre distance 1; rescaled to the oracle's RMS, the device's centres c differ from
    # the unscaled ones by at most |e|, so their residual is at most (1 + kappa) times the device's own
    C = np.stack([-R.T @ t for R, t in poses])
    rms = math.sqrt(float((xo[:S][P.positioned] ** 2).sum(1).mean()))
    xc = C[sy.cams] * rms
    lam = np.linalg.eigvalsh(sy.S)
    kappa = lam[-1] / lam[0]
    # the device's residual is of the whole Laplacian; eliminating the points multiplies it by at most 1 + sqrt(degree)
    deg = float(np.bincount(P.set[P.used], minlength=S).max())
    e2 = check_step(sy.S, sy.b, xc, xo[sy.cams], rep.cg_iterations, int(deg), float(sy.D.max()),
                    inflate=(1 + kappa) * (1 + math.sqrt(deg)))
    assert np.abs(xc - xo[sy.cams]).max() <= e2 + 1e-14 * rms
    # points: x_j = (b_j + sum w x_c) / D_j, a weighted mean of the camera error: within the same bound, scaled by 1 / rms
    assert np.abs(X - Xo).max() <= (e2 + 1e-13 * rms) / rms
    # three iterations
    rc, _, _, _, rep3 = run_pos(lib, sc, api._position_params(max_iters=3, cg_tol=1e-12, cg_max_iters=CG_MAX, function_tol=0.0, **GP_KW))
    _, orep = P.run(max_iters=3, function_tol=0.0)
    print(row, "device", rep3.initial_cost, rep3.final_cost, rep3.iterations, rep3.cg_iterations, "oracle", orep)
    assert rc == 0 and (rep3.iterations, rep3.termination) == (orep["iterations"], orep["termination"])
    assert abs(rep3.initial_cost - orep["initial_cost"]) <= 1e-9 * orep["initial_cost"]
    assert abs(rep3.final_cost - orep["final_cost"]) <= 1e-9 * orep["final_cost"]


def test_positioning_large_deterministic(lib, scenes):
    sc = scenes("gp_large")
    prm = api._position_params(max_iters=3, **GP_KW)
    a, b = run_pos(lib, sc, prm), run_pos(lib, sc, prm)
    assert a[0] == 0 and a[3].tobytes() == b[3].tobytes() and bytes(a[4]) == bytes(b[4])
    assert all(x[1].tobytes() == y[1].tobytes() for x, y in zip(a[1], b[1]))


# ---- rotation averaging ----

ROTATION_ROWS = [r for r in ss.ROWS if ss.ROWS[r][0] == "rotation"]
RA_KW = dict(loss="cauchy", loss_scale=2.0, min_inliers=0)


@pytest.mark.parametrize("row", ROTATION_ROWS)
def test_rotation_rows(lib, scenes, row):
    Rt, pairs, Rp, nf, _ = scenes(row)
    S = int(np.asarray(pairs).max()) + 1
    rc, R, reg, err, rep = run_rot(lib, S, pairs, Rp, nf, api._rotation_params(max_iters=1, cg_tol=CG_TOL, cg_max_iters=CG_MAX, **RA_KW))
    assert rc == 0, api._last_error(lib)
    Rpo = np.stack([go.orthonormal(m) for m in Rp])
    used, rego, root, R0 = go.start(S, pairs, Rpo, nf, 0)
    assert np.array_equal(reg.astype(bool), rego) and rep.n_pairs == int(used.sum()) and rep.n_registered == int(rego.sum())
    assert rep.iterations == 1 and rep.cg_iterations < CG_MAX, "CG stopped on the count, not on cg_tol"
    # the oracle's first linear system at the start
    s2 = (RA_KW["loss_scale"] * go.DEG) ** 2
    ends = np.asarray(pairs)
    res = go.log_batch(np.matmul(np.swapaxes(R0[ends[:, 1]], 1, 2), np.matmul(Rpo, R0[ends[:, 0]])))
    r2 = (res * res).sum(1)
    rho, w = bo.loss(RA_KW["loss"], r2 / s2)
    c0 = float(np.sum(0.5 * (s2 * rho)))
    assert abs(rep.initial_cost - c0) <= len(pairs) * U53 * c0
    sy = go.LaplacianSystem(S, ends, w, -w[:, None] * res, root)
    xo = sy.solve()
    xd = np.stack([go.log(R0[i].T @ R[i]) for i in range(S)])
    assert (xd[~rego] == 0).all() and (xd[root] == 0).all()
    e2 = check_step(sy.S, sy.b, xd[sy.cams], xo[sy.cams], rep.cg_iterations, int(np.bincount(ends.reshape(-1)).max()), float(sy.D.max()))
    assert np.abs(xd - xo).max() <= e2 + 16 * U53
    # three iterations
    rc, R3, _, err3, rep3 = run_rot(lib, S, pairs, Rp, nf, api._rotation_params(max_iters=3, step_tol=0.0, cg_tol=1e-12, cg_max_iters=CG_MAX, **RA_KW))
    Ro, _, erro, orep = go.rotation_averaging(S, pairs, Rp, nf, max_iters=3, step_tol=0.0, solve=go.laplacian_solve_reduced, **RA_KW)
    print(row, "device", rep3.initial_cost, rep3.final_cost, rep3.iterations, rep3.cg_iterations, "oracle", orep)
    assert rc == 0 and (rep3.iterations, rep3.termination) == (orep["iterations"], orep["termination"])
    assert abs(rep3.final_cost - orep["final_cost"]) <= 1e-9 * orep["final_cost"]
    if row == "ra_large":
        b = run_rot(lib, S, pairs, Rp, nf, api._rotation_params(max_iters=3, step_tol=0.0, cg_tol=1e-12, cg_max_iters=CG_MAX, **RA_KW))
        assert R3.tobytes() == b[1].tobytes() and err3.tobytes() == b[3].tobytes() and bytes(rep3) == bytes(b[4])
