"""ps_bundle_adjust on the GPU against tests/bundle_oracle.py on planted scenes (one step, convergence under each loss,
robust losses, structure only, untouched records, a non-finite start), determinism, argument errors with the outputs
untouched, and the chain extraction -> tracks -> triangulate -> bundle adjustment on rendered views with known poses.

How results are compared.  The device solves the reduced camera system by preconditioned CG and the oracle the whole
damped system densely, so they agree to the CG tolerance, not bit for bit: one step with cg_tol = 1e-14 within a relative
1e-7, converged costs within a relative 1e-6."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bundle_oracle as bo                # noqa: E402
import triangulate_oracle as tro          # noqa: E402
from popsift_b200 import api              # noqa: E402

pytestmark = pytest.mark.gpu

PS_ERR_ARG = -1
SENTINEL = 0x5A
GUARD = 256


def _features(xy):
    f = np.zeros(len(xy), api.FEATURE_DTYPE)
    f["x"], f["y"], f["sigma"], f["num_ori"] = xy[:, 0], xy[:, 1], 2.0, 1
    return f


def _records(sc, X=None):
    T = len(sc["start"]) - 1
    rec = np.zeros(T, api.TRACK_POINT_DTYPE)
    rec["X"] = sc["X0"] if X is None else X
    rec["status"] = sc["status"]
    rec["n_inliers"] = np.diff(sc["start"])
    rec["error"], rec["angle"] = 0.25, 7.5
    return rec


def run_device(lib, sc, fixed, prm, rec=None, start=None, members=None, errors=True, feats=None):
    """ps_bundle_adjust on a planted scene.  d_points holds the records between GUARD sentinel bytes on both sides and
    d_obs_error is prefilled with the sentinel and fenced the same way; the fences must come back untouched.  Returns
    (rc, poses_out, points (bytes), obs_error (bytes or None), report)"""
    start = np.ascontiguousarray(sc["start"] if start is None else start, np.int32)
    members = np.ascontiguousarray(sc["members"] if members is None else members, np.int32)
    rec = _records(sc) if rec is None else rec
    feats = sc["feats"] if feats is None else feats
    T, M = len(start) - 1, len(members)
    raw = np.full(rec.nbytes + 2 * GUARD, SENTINEL, np.uint8)
    raw[GUARD:GUARD + rec.nbytes] = rec.view(np.uint8)
    n = len(feats)
    out = (api.PsRigid * n)()
    for i in range(n):
        out[i].R[:] = [-7.0] * 9
        out[i].t[:] = [-7.0] * 3
    rep = api.PsBundleReport(-7.0, -7.0, -7, -7, -7, -7, -7, -7, -7, 0)
    bufs = api._DevBuffers(lib)
    try:
        ptrs = [bufs.upload(_features(np.asarray(f, np.float32).reshape(-1, 2))) for f in feats]
        d_raw = bufs.upload(raw)
        d_err = bufs.upload(np.full(4 * max(M, 1) + 2 * GUARD, SENTINEL, np.uint8))
        rc = lib.ps_bundle_adjust(0, n, (C.c_int32 * n)(*[len(f) for f in feats]), (C.c_void_p * n)(*ptrs),
                                  api._c_cameras(sc["cams"]).ctypes.data, api._c_rigids(sc["poses"]), T, bufs.upload(start),
                                  bufs.upload(members), M, d_raw + GUARD, bufs.upload(np.ascontiguousarray(sc["mask"], np.uint8)),
                                  (C.c_uint8 * n)(*[int(v) for v in fixed]), C.byref(prm), out, d_err + GUARD if errors else None,
                                  C.byref(rep))
        got = bufs.download(d_raw, len(raw), np.uint8)
        err = bufs.download(d_err, 4 * max(M, 1) + 2 * GUARD, np.uint8)
    finally:
        bufs.free()
    assert (got[:GUARD] == SENTINEL).all() and (got[GUARD + rec.nbytes:] == SENTINEL).all(), "a write outside d_points"
    assert (err[:GUARD] == SENTINEL).all() and (err[GUARD + 4 * max(M, 1):] == SENTINEL).all(), "a write outside d_obs_error"
    err = err[GUARD:GUARD + 4 * M]
    if not errors:
        assert (err == SENTINEL).all()
        err = None
    poses = [(np.array(out[i].R[:]).reshape(3, 3), np.array(out[i].t[:])) for i in range(n)]
    return rc, poses, got[GUARD:GUARD + rec.nbytes], err, rep


def _pts(raw):
    return raw.view(api.TRACK_POINT_DTYPE)


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


def _scene(seed, n_cams=6, n_tracks=60, **kw):
    rng = np.random.default_rng(seed)
    return bo.planted(rng, n_cams, list(rng.integers(3, n_cams + 1, size=n_tracks)), **kw)


def _fixed(n, *idx):
    f = np.zeros(n, np.uint8)
    f[list(idx)] = 1
    return f


@pytest.mark.parametrize("loss", ["squared", "cauchy"])
def test_one_iteration(lib, loss):
    """max_iters = 1 with CG run to 1e-14: the device's step is the oracle's dense damped step"""
    for seed in (1, 2):
        sc = _scene(seed)
        fixed = _fixed(6, 0)
        kw = dict(loss=loss, loss_scale=2.0, initial_lambda=1e-3, scale_set=1, scale_axis=2)
        prm = api._bundle_params(max_iters=1, cg_tol=1e-14, cg_max_iters=6 * 6 + 10, **kw)
        rc, poses, raw, _, rep = run_device(lib, sc, fixed, prm)
        assert rc == 0, api._last_error(lib)
        prob = bo.problem(sc, fixed, loss_kind=loss, loss_scale=2.0, scale_set=1, scale_axis=2)
        d, pred = prob.step(sc["poses"], sc["X0"], 1e-3)
        pn, Xn = prob.apply(sc["poses"], sc["X0"], d)
        assert prob.cost(pn, Xn) < prob.cost(sc["poses"], sc["X0"])
        assert rep.iterations == 1 and rep.accepted == 1 and rep.termination == bo.MAX_ITERS
        assert abs(rep.initial_cost - prob.cost(sc["poses"], sc["X0"])) <= 1e-12 * rep.initial_cost
        assert abs(rep.final_cost - prob.cost(pn, Xn)) <= 1e-7 * rep.final_cost
        for (R, t), (Ro, to) in zip(poses, pn):
            assert np.abs(R - Ro).max() <= 1e-7 and np.abs(t - to).max() <= 1e-7 * max(1.0, np.abs(to).max())
        X = _pts(raw)["X"]
        assert np.abs(X - Xn).max() <= 1e-7 * max(1.0, np.abs(Xn).max())
        assert rep.n_obs == len(sc["members"]) and rep.n_points == 60 and rep.n_free_cams == 5
        assert poses[0][0].tobytes() == np.asarray(sc["poses"][0][0]).tobytes()
        assert poses[1][1][2] == sc["poses"][1][1][2]                      # the held component


@pytest.mark.parametrize("loss", ["squared", "huber", "cauchy"])
def test_convergence(lib, loss):
    """0.5 px noise, poses turned by 1 degree and moved by 2 % of the scene: the device's converged cost is the dense LM's
    within 1e-6, the oracle's gradient there is below 1e-4 of its starting value, and every free pose gets closer to the
    truth (by at least half its rotation error and half its centre error)"""
    sc = _scene(3, n_cams=8, n_tracks=120)
    fixed = _fixed(8, 0)
    bo.gauge_to_truth(sc, 0, 1, 2)
    kw = dict(loss=loss, loss_scale=2.0, scale_set=1, scale_axis=2)
    prm = api._bundle_params(max_iters=100, function_tol=1e-12, cg_tol=1e-10, cg_max_iters=200, **kw)
    rc, poses, raw, err, rep = run_device(lib, sc, fixed, prm)
    assert rc == 0, api._last_error(lib)
    prob = bo.problem(sc, fixed, loss_kind=loss, loss_scale=2.0, scale_set=1, scale_axis=2)
    _, _, orep = bo.lm(prob, sc["poses"], sc["X0"], max_iters=100, function_tol=1e-12)
    print(loss, "device", rep.final_cost, rep.iterations, rep.accepted, rep.cg_iterations, rep.termination,
          "oracle", orep)
    assert rep.termination == bo.FUNCTION_TOL
    assert abs(rep.final_cost - orep["final_cost"]) <= 1e-6 * orep["final_cost"]
    X = _pts(raw)["X"]
    g0 = np.abs(prob.gradient(sc["poses"], sc["X0"])).max()
    g1 = np.abs(prob.gradient(poses, X)).max()
    assert g1 <= 1e-4 * g0, (g1, g0)
    r0, c0 = bo.pose_errors(sc["poses"], sc["poses_true"])
    r1, c1 = bo.pose_errors(poses, sc["poses_true"])
    print("rotation before", r0[1:], "after", r1[1:], "centre before", c0[1:], "after", c1[1:])
    assert (r1[1:] < 0.5 * r0[1:]).all() and (c1[1:] < 0.5 * c0[1:]).all()
    # outputs: error is the mean pixel error over the used observations, obs_error every member's
    e = err.view(np.float32)
    pts = _pts(raw)
    for k in (0, 7, 50):
        s0, s1 = sc["start"][k], sc["start"][k + 1]
        assert abs(pts["error"][k] - e[s0:s1].astype(np.float64).mean()) <= 1e-5 * max(1.0, float(pts["error"][k]))
    assert np.median(e) < 1.0


def test_robust_losses_downweight_outliers(lib):
    """15 % outliers kept in the mask: Huber and Cauchy recover the poses better than the squared loss"""
    rng = np.random.default_rng(4)
    sc = bo.planted(rng, 8, list(rng.integers(4, 9, size=200)), noise=0.5, outliers=0.15)
    bo.gauge_to_truth(sc, 0, 1, 2)
    fixed = _fixed(8, 0)
    res = {}
    for loss in ("squared", "huber", "cauchy"):
        prm = api._bundle_params(loss=loss, loss_scale=2.0, max_iters=100, function_tol=1e-10, cg_tol=1e-8, cg_max_iters=200,
                                 scale_set=1, scale_axis=2)
        rc, poses, raw, _, rep = run_device(lib, sc, fixed, prm)
        assert rc == 0
        r, c = bo.pose_errors(poses, sc["poses_true"])
        res[loss] = (r[1:].max(), c[1:].max())
    print(res)
    for loss in ("huber", "cauchy"):
        assert res[loss][0] < 0.7 * res["squared"][0] and res[loss][1] < 0.7 * res["squared"][1]


def test_structure_only(lib):
    """all poses fixed: the poses come back bit for bit and the points are the dense LM's"""
    sc = _scene(5)
    fixed = np.ones(6, np.uint8)
    prm = api._bundle_params(max_iters=30, function_tol=1e-12, cg_tol=1e-10)
    rc, poses, raw, _, rep = run_device(lib, sc, fixed, prm)
    assert rc == 0 and rep.n_free_cams == 0 and rep.cg_iterations == 0
    for (R, t), (R0, t0) in zip(poses, sc["poses"]):
        assert R.tobytes() == np.asarray(R0).tobytes() and t.tobytes() == np.asarray(t0).tobytes()
    prob = bo.problem(sc, fixed)
    _, Xo, orep = bo.lm(prob, sc["poses"], sc["X0"], max_iters=30, function_tol=1e-12)
    assert abs(rep.final_cost - orep["final_cost"]) <= 1e-6 * orep["final_cost"]
    assert np.abs(_pts(raw)["X"] - Xo).max() < 1e-6


def test_untouched_records_and_sets(lib):
    """non-OK tracks keep their bytes, masked members are not used, a free set without observations keeps its pose"""
    sc = _scene(6, n_cams=6, n_tracks=80)
    # set 6: free, no features at all; set 5: free, every observation masked out
    sc["feats"] = list(sc["feats"]) + [np.zeros((0, 2), np.float32)]
    sc["cams"] = np.concatenate([sc["cams"], sc["cams"][:1]])
    sc["poses"] = list(sc["poses"]) + [sc["poses"][2]]
    off = np.concatenate([[0], np.cumsum([len(f) for f in sc["feats"]])])
    sets = np.searchsorted(off, sc["members"], side="right") - 1
    sc["mask"] = (sets != 5).astype(np.uint8)
    sc["mask"][::7] = 0
    bad = np.arange(0, 80, 9)
    sc["status"][bad] = tro.TOO_FEW_INLIERS
    fixed = _fixed(7, 0)
    rec = _records(sc)
    prm = api._bundle_params(max_iters=10)
    rc, poses, raw, err, rep = run_device(lib, sc, fixed, prm, rec=rec)
    assert rc == 0
    pts = _pts(raw)
    assert pts[bad].tobytes() == rec[bad].tobytes()
    for i in (5, 6):
        assert poses[i][0].tobytes() == np.asarray(sc["poses"][i][0]).tobytes()
        assert poses[i][1].tobytes() == np.asarray(sc["poses"][i][1]).tobytes()
    assert rep.n_free_cams == 4 and rep.accepted > 0
    e = err.view(np.float32)
    track = np.repeat(np.arange(80), np.diff(sc["start"]))
    assert np.isinf(e[np.isin(track, bad)]).all() and np.isfinite(e[~np.isin(track, bad)]).all()
    # the oracle with the same mask and statuses
    prob = bo.problem(sc, fixed)
    assert rep.n_obs == len(prob.set)
    _, _, orep = bo.lm(prob, sc["poses"], sc["X0"], max_iters=10)
    assert abs(rep.initial_cost - orep["initial_cost"]) <= 1e-12 * orep["initial_cost"]


def test_nonfinite_start(lib):
    sc = _scene(7)
    R, t = sc["poses"][3]
    flip = np.diag([-1.0, 1.0, -1.0])
    sc["poses"][3] = (flip @ R, flip @ t)
    rec = _records(sc)
    rc, poses, raw, err, rep = run_device(lib, sc, _fixed(6, 0), api._bundle_params(), rec=rec)
    assert rc == 0 and rep.termination == bo.NONFINITE_START and rep.iterations == 0
    assert raw.tobytes() == rec.tobytes()
    for (R, t), (R0, t0) in zip(poses, sc["poses"]):
        assert R.tobytes() == np.asarray(R0).tobytes() and t.tobytes() == np.asarray(t0).tobytes()
    assert np.isinf(err.view(np.float32)).any()


def test_no_observations(lib):
    sc = _scene(8)
    sc["mask"] = np.zeros_like(sc["mask"])
    rec = _records(sc)
    rc, poses, raw, _, rep = run_device(lib, sc, _fixed(6, 0), api._bundle_params(), rec=rec)
    assert rc == 0 and rep.termination == bo.NO_OBSERVATIONS and rep.n_obs == 0 and raw.tobytes() == rec.tobytes()


def test_determinism(lib):
    rng = np.random.default_rng(9)
    sc = bo.planted(rng, 12, list(rng.integers(2, 12, size=400)), noise=0.5, outliers=0.05)
    prm = api._bundle_params(loss="huber", loss_scale=2.0, max_iters=8, scale_set=2, scale_axis=1)
    a = run_device(lib, sc, _fixed(12, 0, 5), prm)
    b = run_device(lib, sc, _fixed(12, 0, 5), prm)
    assert a[0] == 0 and a[2].tobytes() == b[2].tobytes() and a[3].tobytes() == b[3].tobytes()
    assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(a[1], b[1]))
    assert bytes(a[4]) == bytes(b[4])


def test_argument_errors(lib):
    sc = _scene(10, n_tracks=5)
    fixed = _fixed(6, 0)
    prm = api._bundle_params(max_iters=3)
    assert run_device(lib, sc, fixed, prm)[0] == 0
    assert run_device(lib, sc, fixed, prm, errors=False)[0] == 0
    rec = _records(sc)

    def untouched(r):
        rc, poses, raw, err, rep = r
        assert rc == PS_ERR_ARG
        assert raw.tobytes() == rec.tobytes() and (err is None or (err == SENTINEL).all())
        assert all((p[0] == -7.0).all() and (p[1] == -7.0).all() for p in poses) and rep.termination == -7

    N = sum(len(f) for f in sc["feats"])
    st = np.asarray(sc["start"])
    M = len(sc["members"])
    # found on the device
    for start, members in ((st, np.r_[sc["members"][:-1], N]), (st, np.r_[sc["members"][:-1], -1]), (np.r_[1, st[1:]], None),
                           (np.r_[st[:-1], M - 1], None), (np.r_[st[0], st[2], st[1], st[3:]], None)):
        untouched(run_device(lib, sc, fixed, prm, start=start, members=members))
    # refused on the host
    for kw in (dict(max_iters=-1), dict(max_iters=10001), dict(cg_max_iters=0), dict(cg_max_iters=10001), dict(loss_scale=0.0),
               dict(loss_scale=float("nan")), dict(function_tol=-1.0), dict(cg_tol=1.0), dict(cg_tol=-0.1), dict(initial_lambda=0.0),
               dict(initial_lambda=1e33), dict(scale_set=6), dict(scale_set=-2), dict(scale_axis=3), dict(scale_axis=-1)):
        untouched(run_device(lib, sc, fixed, api._bundle_params(**kw)))
    bad_loss = api._bundle_params()
    bad_loss.loss = 3
    untouched(run_device(lib, sc, fixed, bad_loss))
    untouched(run_device(lib, sc, np.zeros(6, np.uint8), prm))           # no fixed set
    untouched(run_device(lib, sc, np.r_[1, 2, 0, 0, 0, 0].astype(np.uint8), prm))
    bad_cam = dict(sc, cams=sc["cams"].copy())
    bad_cam["cams"][2, 1] = -1.0
    untouched(run_device(lib, bad_cam, fixed, prm))
    bad_pose = dict(sc, poses=list(sc["poses"]))
    bad_pose["poses"][1] = (np.eye(3) * 1.001, np.zeros(3))
    untouched(run_device(lib, bad_pose, fixed, prm))


def test_api_round_trip(lib):
    """api.bundle_adjust on host Feature records gives what the C ABI gives"""
    sc = _scene(11)
    fixed = _fixed(6, 0)
    prm_kw = dict(loss="huber", loss_scale=1.5, max_iters=5, scale_set=1, scale_axis=1)
    rc, poses, raw, err, rep = run_device(lib, sc, fixed, api._bundle_params(**prm_kw))
    off = np.cumsum([0] + [len(f) for f in sc["feats"]])
    sets_of = np.searchsorted(off, sc["members"], side="right") - 1
    tr = api.Tracks(sc["start"], sets_of, sc["members"] - off[sets_of], None, 0, 0, 0)
    r = _records(sc)
    tp = api.TrackPoints(r["X"], r["error"], r["angle"], r["n_inliers"], r["status"], sc["mask"], None, None)
    feats = [_features(np.asarray(f, np.float32)) for f in sc["feats"]]
    p2, tp2, rep2 = api.bundle_adjust(feats, tr, tp, sc["cams"], sc["poses"], fixed.astype(bool), **prm_kw)
    assert all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() for a, b in zip(poses, p2))
    assert np.array_equal(_pts(raw)["X"], tp2.X) and np.array_equal(err.view(np.float32), tp2.obs_error)
    assert rep2.final_cost == rep.final_cost and rep2.termination == api.BA_TERMINATION[rep.termination]


# ---- end to end: test_triangulate's rendered views ----

from test_triangulate import VIEWS, _view_pose, rendered_views   # noqa: E402,F401  (rendered_views: the module fixture)
from test_pose import CAMS, W, H, _cast                         # noqa: E402,F401


def _perturbed(poses, rng):
    out = [poses[0]]
    for R, t in poses[1:]:
        out.append((bo.small_rotation(rng, 1.0) @ R, t + rng.normal(scale=0.01, size=3)))
    out[1][1][0] = poses[1][1][0]          # the held component keeps the true scale
    return out


def test_end_to_end_rendered(rendered_views, tmp_path):
    """extraction -> tracks -> triangulate with views 1..5 perturbed -> bundle_adjust with view 0 fixed and the x
    component of view 1's t held: every view gets closer to the truth"""
    imgs, cams, poses, sets = rendered_views
    rng = np.random.default_rng(21)
    pert = _perturbed(poses, rng)
    pairs = [(i, j) for i in range(len(sets)) for j in range(i + 1, len(sets))]
    tr = api.tracks(sets, pairs, model="fundamental", threshold=2.0, seed=1)
    tp = api.triangulate(sets, tr, cams, pert, max_error=8.0, min_angle=1.5, seed=2)
    fixed = [True] + [False] * (len(sets) - 1)
    # view 1's t[0] keeps its true value (the baseline's scale), so the gauge is the truth's
    out, tp2, rep = api.bundle_adjust(sets, tr, tp, cams, pert, fixed, loss="cauchy", loss_scale=2.0, max_iters=100,
                                      function_tol=1e-10, cg_tol=1e-8, scale_set=1, scale_axis=0)
    r0, c0 = bo.pose_errors(pert, poses)
    r1, c1 = bo.pose_errors(out, poses)
    ok = tp2.status == 0
    med = float(np.median(tp2.error[ok]))
    print("rendered BA:", rep, "rotation err before", r0, "after", r1, "centre err before", c0, "after", c1,
          "median reprojection before", float(np.median(tp.error[ok])), "after", med)
    assert rep.accepted > 0 and rep.final_cost < rep.initial_cost
    assert (r1[1:] < r0[1:]).all() and (c1[1:] < c0[1:]).all()
    # measured on an NVIDIA H100 80GB HBM3 at 700 W (DESIGN 4.14): 10 490 used observations of 4 117 points, 36 LM
    # iterations, all accepted (959 CG iterations); rotation errors of views 1..5 from 1 degree to 0.005 .. 0.028 degrees,
    # centre errors from 0.011 .. 0.027 to 0.0003 .. 0.0037, median reprojection error of the OK tracks from 5.2 px to
    # 0.074 px.  The floors keep a margin of about 3x.
    assert r1[1:].max() < 0.1 and c1[1:].max() < 0.01 and med < 0.3
    # the C++ API on the same frames against the C ABI
    from popsift_b200 import build as B
    files = []
    for k, im in enumerate(imgs):
        f = tmp_path / ("v%d.raw" % k)
        im.tofile(f)
        files.append(str(f))
    args = [B.BUNDLE_CHECK, str(W), str(H), str(len(imgs))] + files
    for cam, (R, t) in zip(cams, pert):
        args += ["%.9g" % v for v in cam] + ["%.17g" % v for v in np.r_[R.ravel(), t]]
    res = subprocess.run(args, capture_output=True, text=True, timeout=600)
    print(res.stdout)
    assert res.returncode == 0 and res.stdout.startswith("OK"), res.stdout + res.stderr      # H100, same run: "OK 10503 14 263.867"
