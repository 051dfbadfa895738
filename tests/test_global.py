"""ps_rotation_averaging and ps_global_positioning on the GPU against tests/global_oracle.py (the spanning-tree start, one
step, converged costs under each loss, a cost that never increases, edge cases), determinism, argument errors with the
outputs untouched, and the chain global_poses -> triangulate -> bundle_adjust on rendered views with intrinsics only.

How results are compared.  The device solves each linear system by preconditioned CG and the oracle densely, so they
agree to the CG tolerance, not bit for bit: one step with cg_tol = 1e-14 within a relative 1e-9."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bundle_oracle as bo                # noqa: E402
import global_oracle as go                # noqa: E402
from popsift_b200 import api              # noqa: E402

pytestmark = pytest.mark.gpu

PS_ERR_ARG = -1
SENTINEL = 0x5A
GUARD = 256


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


def _records(Rp, nf):
    rec = np.zeros(len(Rp), api.TWO_VIEW_DTYPE)
    rec["R"] = np.asarray(Rp, np.float32).reshape(-1, 3, 3)
    rec["n_front"] = nf
    rec["n_inliers"] = nf
    return rec


def run_rot(lib, n_sets, pairs, Rp, nf, prm):
    """ps_rotation_averaging with every host output prefilled with the sentinel: (rc, R, registered, pair_error, report)"""
    P = len(pairs)
    R = np.full(n_sets * 9 + GUARD, -7.0)
    reg = np.full(n_sets + GUARD, SENTINEL, np.uint8)
    err = np.full(P + GUARD, -7.0, np.float32)
    rep = api.PsRotationReport(-7.0, -7.0, -7, -7, -7, -7, -7, 0)
    bufs = api._DevBuffers(lib)
    try:
        d = bufs.upload(_records(Rp, nf)) if P else None
        rc = lib.ps_rotation_averaging(0, n_sets, P, api._c_pairs(pairs), d, C.byref(prm), R.ctypes.data, reg.ctypes.data, err.ctypes.data,
                                       C.byref(rep))
    finally:
        bufs.free()
    assert (R[9 * n_sets:] == -7.0).all() and (reg[n_sets:] == SENTINEL).all() and (err[P:] == -7.0).all(), "a write past an output"
    return rc, R[:9 * n_sets].reshape(-1, 3, 3), reg[:n_sets], err[:P], rep


def _graph(seed, n=20, p=80, **kw):
    return go.view_graph(np.random.default_rng(seed), n, p, **kw)


def test_rotation_start(lib):
    Rt, pairs, Rp, nf, _ = _graph(1)
    rc, R, reg, err, rep = run_rot(lib, 20, pairs, Rp, nf, api._rotation_params(max_iters=0, min_inliers=0))
    assert rc == 0, api._last_error(lib)
    _, _, err_o, orep = go.rotation_averaging(20, pairs, Rp, nf, max_iters=0, min_inliers=0)
    Ro = go.start(20, pairs, np.stack([go.orthonormal(m) for m in Rp]), nf, 0)[3]
    assert np.abs(R - Ro).max() <= 1e-12 and reg.all() and rep.iterations == 0
    assert abs(rep.initial_cost - orep["initial_cost"]) <= 1e-12 * orep["initial_cost"]
    assert np.abs(err - err_o).max() <= 1e-5


@pytest.mark.parametrize("loss", ["squared", "huber", "cauchy"])
def test_rotation_one_step_and_converged(lib, loss):
    Rt, pairs, Rp, nf, _ = _graph(2, noise_deg=0.5, outliers=0.2)
    kw = dict(loss=loss, loss_scale=2.0, min_inliers=0)
    rc, R, reg, err, rep = run_rot(lib, 20, pairs, Rp, nf, api._rotation_params(max_iters=1, cg_tol=1e-14, cg_max_iters=200, **kw))
    assert rc == 0
    Ro, _, _, orep = go.rotation_averaging(20, pairs, Rp, nf, max_iters=1, **kw)
    assert np.abs(R - Ro).max() <= 1e-9 and abs(rep.final_cost - orep["final_cost"]) <= 1e-9 * orep["final_cost"]
    rc, R, reg, err, rep = run_rot(lib, 20, pairs, Rp, nf, api._rotation_params(max_iters=100, step_tol=1e-9, cg_tol=1e-12,
                                                                                cg_max_iters=200, **kw))
    Ro, _, _, orep = go.rotation_averaging(20, pairs, Rp, nf, max_iters=100, step_tol=1e-9, **kw)
    print(loss, "device", rep.final_cost, rep.iterations, rep.cg_iterations, "oracle", orep)
    assert abs(rep.final_cost - orep["final_cost"]) <= 1e-6 * orep["final_cost"]


def test_rotation_edge_cases(lib):
    I = np.eye(3)
    # disconnected: {2, 3, 4} registered; the self pair and the pair below min_inliers are not used
    pairs = [(0, 1), (2, 3), (3, 4), (5, 5), (1, 5)]
    Rp = np.stack([I] * 5)
    rc, R, reg, err, rep = run_rot(lib, 6, pairs, Rp, [50, 50, 50, 50, 5], api._rotation_params(min_inliers=15))
    assert rc == 0 and list(reg) == [0, 0, 1, 1, 1, 0] and rep.n_pairs == 2 and rep.n_registered == 3
    assert np.isinf(err[[0, 3, 4]]).all() and np.isfinite(err[[1, 2]]).all()
    assert all(np.array_equal(R[i], I) for i in (0, 1, 5))
    # a tie: the component of set 0
    rc, R, reg, err, rep = run_rot(lib, 4, [(0, 1), (2, 3)], Rp[:2], [50, 50], api._rotation_params())
    assert rc == 0 and list(reg) == [1, 1, 0, 0]
    # no pairs, no sets
    rc, R, reg, err, rep = run_rot(lib, 3, [], Rp[:0], [], api._rotation_params())
    assert rc == 0 and list(reg) == [1, 0, 0] and rep.termination == go.RA_NO_PAIRS
    assert run_rot(lib, 0, [], Rp[:0], [], api._rotation_params())[0] == 0
    # argument errors leave the outputs untouched
    for kw in (dict(max_iters=-1), dict(cg_max_iters=0), dict(loss_scale=0.0), dict(step_tol=-1.0), dict(cg_tol=1.0), dict(min_inliers=-1)):
        rc, R, reg, err, rep = run_rot(lib, 6, pairs, Rp, [50] * 5, api._rotation_params(**kw))
        assert rc == PS_ERR_ARG and (R == -7.0).all() and (reg == SENTINEL).all() and (err == -7.0).all() and rep.termination == -7
    rc, R, reg, err, rep = run_rot(lib, 6, pairs + [(0, 6)], np.stack([I] * 6), [50] * 6, api._rotation_params())
    assert rc == PS_ERR_ARG and (R == -7.0).all()


def test_rotation_determinism(lib):
    Rt, pairs, Rp, nf, _ = _graph(3, n=40, p=300, outliers=0.1)
    a = run_rot(lib, 40, pairs, Rp, nf, api._rotation_params(max_iters=10, min_inliers=0))
    b = run_rot(lib, 40, pairs, Rp, nf, api._rotation_params(max_iters=10, min_inliers=0))
    assert a[1].tobytes() == b[1].tobytes() and a[3].tobytes() == b[3].tobytes() and bytes(a[4]) == bytes(b[4])


# ---- positioning

def _features(xy):
    f = np.zeros(len(xy), api.FEATURE_DTYPE)
    f["x"], f["y"], f["sigma"], f["num_ori"] = xy[:, 0], xy[:, 1], 2.0, 1
    return f


def _scene(seed, n_cams=6, n_tracks=80, **kw):
    rng = np.random.default_rng(seed)
    sc = bo.planted(rng, n_cams, list(rng.integers(2, n_cams + 1, size=n_tracks)), **kw)
    sc["R"] = np.stack([np.asarray(R) for R, _ in sc["poses_true"]])
    return sc


def run_pos(lib, sc, prm, reg=None, start=None, members=None, X=True):
    """ps_global_positioning; d_X is fenced by GUARD sentinel bytes on both sides and every host output prefilled.
    Returns (rc, poses, positioned, X or None, report)"""
    start = np.ascontiguousarray(sc["start"] if start is None else start, np.int32)
    members = np.ascontiguousarray(sc["members"] if members is None else members, np.int32)
    feats = sc["feats"]
    n, T, M = len(feats), len(start) - 1, len(members)
    reg = np.ones(n, np.uint8) if reg is None else np.asarray(reg, np.uint8)
    out = (api.PsRigid * (n + 3))()         # 3 guard records (288 bytes) past the end
    for i in range(n + 3):
        out[i].R[:] = [-7.0] * 9
        out[i].t[:] = [-7.0] * 3
    pos = np.full(n + GUARD, SENTINEL, np.uint8)
    rep = api.PsPositionReport(-7.0, -7.0, -7, -7, -7, -7, -7, -7)
    nb = 24 * T + 2 * GUARD
    bufs = api._DevBuffers(lib)
    try:
        ptrs = [bufs.upload(_features(np.asarray(f, np.float32).reshape(-1, 2))) for f in feats]
        d_x = bufs.upload(np.full(nb, SENTINEL, np.uint8))
        Rs = np.ascontiguousarray(sc["R"], np.float64)
        rc = lib.ps_global_positioning(0, n, (C.c_int32 * n)(*[len(f) for f in feats]), (C.c_void_p * n)(*ptrs),
                                       api._c_cameras(sc["cams"]).ctypes.data, Rs.ctypes.data, reg.ctypes.data, T, bufs.upload(start),
                                       bufs.upload(members) if M else None, M, C.byref(prm), out, pos.ctypes.data,
                                       d_x + GUARD if X else None, C.byref(rep))
        got = bufs.download(d_x, nb, np.uint8)
    finally:
        bufs.free()
    assert (got[:GUARD] == SENTINEL).all() and (got[GUARD + 24 * T:] == SENTINEL).all(), "a write outside d_X"
    assert (pos[n:] == SENTINEL).all() and all((np.array(out[i].R[:]) == -7.0).all() for i in range(n, n + 3)), "a write past an output"
    body = got[GUARD:GUARD + 24 * T]
    if not X:
        assert (body == SENTINEL).all()
    poses = [(np.array(out[i].R[:]).reshape(3, 3), np.array(out[i].t[:])) for i in range(n)]
    return rc, poses, pos[:n], body.view(np.float64).reshape(-1, 3) if X else None, rep


def _oracle(sc, reg=None, **kw):
    reg = np.ones(len(sc["feats"]), bool) if reg is None else np.asarray(reg, bool)
    return go.Positioning(sc["feats"], sc["cams"], sc["R"], reg, sc["start"], sc["members"], **kw)


@pytest.mark.parametrize("loss", ["squared", "huber", "cauchy"])
def test_positioning_against_oracle(lib, loss):
    """one iteration with cg_tol = 1e-14 is the oracle's dense solve; after 40 iterations the costs agree to 1e-6"""
    sc = _scene(1, noise=0.3)
    kw = dict(loss=loss, loss_scale=0.1)
    P = _oracle(sc, **kw)
    for iters in (0, 1):
        rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(max_iters=iters, cg_tol=1e-14, cg_max_iters=500, function_tol=0.0, **kw))
        assert rc == 0, api._last_error(lib)
        p, orep = P.run(max_iters=iters, function_tol=0.0)
        po, Xo = P.outputs(p)
        assert abs(rep.final_cost - orep["final_cost"]) <= 1e-9 * orep["final_cost"]
        assert np.abs(X - Xo).max() <= 1e-9 * max(1.0, np.abs(Xo).max())
        assert max(np.abs(t - to).max() for (_, t), (_, to) in zip(poses, po)) <= 1e-9
        assert rep.n_obs == int(P.used.sum()) and rep.n_points == int(P.tpart.sum()) and rep.n_cams == 6 and pos.all()
    rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(max_iters=40, cg_tol=1e-12, cg_max_iters=500, function_tol=0.0, **kw))
    p, orep = P.run(max_iters=40, function_tol=0.0)
    print(loss, "device", rep.final_cost, rep.iterations, rep.cg_iterations, "oracle", orep)
    assert abs(rep.final_cost - orep["final_cost"]) <= 1e-6 * orep["final_cost"]


def test_positioning_cost_never_increases(lib):
    sc = _scene(2, noise=0.5, outliers=0.1)
    costs = []
    for k in range(1, 7):
        rc, _, _, _, rep = run_pos(lib, sc, api._position_params(max_iters=k, cg_tol=1e-14, cg_max_iters=500, function_tol=0.0))
        assert rc == 0 and rep.iterations == k
        costs.append(rep.final_cost)
    assert all(b <= a * (1 + 1e-12) for a, b in zip(costs, costs[1:])), costs


def test_positioning_edge_cases(lib):
    sc = _scene(3)
    reg = np.ones(6, np.uint8)
    reg[4] = 0
    rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(max_iters=5), reg=reg)
    P = _oracle(sc, reg)
    assert rc == 0 and list(pos) == [1, 1, 1, 1, 0, 1] and (poses[4][1] == 0).all()
    assert np.array_equal(poses[4][0], sc["R"][4])
    assert (X[~P.tpart] == 0).all() and rep.n_points == int(P.tpart.sum()) and (~P.tpart).any()
    # no tracks
    rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(), start=[0], members=np.zeros(0, np.int32))
    assert rc == 0 and rep.termination == go.GP_NO_OBSERVATIONS and not pos.any() and all((t == 0).all() for _, t in poses)
    # nothing registered
    rc, poses, pos, X, rep = run_pos(lib, sc, api._position_params(), reg=np.zeros(6, np.uint8))
    assert rc == 0 and rep.termination == go.GP_NO_OBSERVATIONS and rep.n_obs == 0 and (X == 0).all()


def test_positioning_determinism_and_errors(lib):
    sc = _scene(4, n_cams=8, n_tracks=300, noise=0.5, outliers=0.05)
    prm = api._position_params(max_iters=6)
    a = run_pos(lib, sc, prm)
    b = run_pos(lib, sc, prm)
    assert a[0] == 0 and a[3].tobytes() == b[3].tobytes() and bytes(a[4]) == bytes(b[4])
    assert all(x[1].tobytes() == y[1].tobytes() for x, y in zip(a[1], b[1]))
    assert run_pos(lib, sc, prm, X=False)[0] == 0

    def untouched(r):
        rc, poses, pos, X, rep = r
        assert rc == PS_ERR_ARG and (X is None or (X.view(np.uint8) == SENTINEL).all())
        assert all((p[0] == -7.0).all() and (p[1] == -7.0).all() for p in poses) and (pos == SENTINEL).all() and rep.termination == -7

    N = sum(len(f) for f in sc["feats"])
    st = np.asarray(sc["start"])
    M = len(sc["members"])
    for start, members in ((st, np.r_[sc["members"][:-1], N]), (st, np.r_[sc["members"][:-1], -1]), (np.r_[1, st[1:]], None),
                           (np.r_[st[:-1], M - 1], None), (np.r_[st[0], st[2], st[1], st[3:]], None)):
        untouched(run_pos(lib, sc, prm, start=start, members=members))
    for kw in (dict(max_iters=-1), dict(cg_max_iters=0), dict(loss_scale=0.0), dict(function_tol=-1.0), dict(cg_tol=1.0)):
        untouched(run_pos(lib, sc, api._position_params(**kw)))
    untouched(run_pos(lib, sc, prm, reg=np.r_[1, 2, 1, 1, 1, 1, 1, 1]))
    bad = dict(sc, R=sc["R"].copy())
    bad["R"][2] *= 1.001
    untouched(run_pos(lib, bad, prm))


# ---- end to end: test_pose's six rendered views, intrinsics only ----

from test_triangulate import VIEWS, _view_pose, rendered_views   # noqa: E402,F401  (rendered_views: the module fixture)
from test_pose import W, H                                       # noqa: E402


def test_end_to_end_rendered(rendered_views, tmp_path):
    """global_poses -> triangulate -> bundle_adjust with view 0 fixed and one translation component of view 1 held"""
    imgs, cams, poses, sets = rendered_views
    pairs = [(i, j) for i in range(len(sets)) for j in range(i + 1, len(sets))]
    gp = api.global_poses(sets, pairs, cams, pose=dict(threshold=1.0, seed=1), rotation=dict(loss_scale=2.0),
                          position=dict(max_iters=1500, function_tol=1e-12))
    print("rotation", gp.rotation_report, "positioning", gp.position_report, "pair errors", gp.pair_error)
    assert gp.registered.all() and gp.positioned.all()

    def errors(est):
        C = np.stack([-R.T @ t for R, t in est])
        Ct = np.stack([-R.T @ t for R, t in poses])
        # the gauge: view 0 at the origin with the truth's rotation frame, scale by least squares
        s = float((C * Ct).sum() / (C * C).sum())
        rot = go.rotation_errors([R for R, _ in est], [R for R, _ in poses])
        cen = np.linalg.norm(s * C - Ct, axis=1) / np.linalg.norm(Ct, axis=1).max()
        return rot, cen, s

    r0, c0, s0 = errors(gp.poses)
    # bundle adjustment in the truth's scale: the held component of view 1 keeps the scaled global estimate
    scaled = [(R, s0 * t) for R, t in gp.poses]
    tp = api.triangulate(sets, gp.tracks, cams, scaled, max_error=4.0, min_angle=1.0, seed=2)
    out, tp2, rep = api.bundle_adjust(sets, gp.tracks, tp, cams, scaled, [True] + [False] * 5, loss="cauchy", loss_scale=2.0,
                                      max_iters=100, function_tol=1e-10, cg_tol=1e-8, scale_set=1, scale_axis=0)
    r1, c1, _ = errors(out)
    print("global: rotation errors", r0, "centre errors", c0, "after bundle adjustment", r1, c1, rep)
    assert r0.max() < 0.1 and c0.max() < 0.01
    assert r1.max() < 0.1 and c1.max() < 0.01
    # the C++ API on the same frames against the C ABI
    from popsift_b200 import build as B
    files = []
    for k, im in enumerate(imgs):
        f = tmp_path / ("v%d.raw" % k)
        im.tofile(f)
        files.append(str(f))
    args = [B.GLOBAL_CHECK, str(W), str(H), str(len(imgs))] + files
    for cam in cams:
        args += ["%.9g" % v for v in cam]
    res = subprocess.run(args, capture_output=True, text=True, timeout=600)
    print(res.stdout)
    assert res.returncode == 0 and res.stdout.startswith("OK"), res.stdout + res.stderr
