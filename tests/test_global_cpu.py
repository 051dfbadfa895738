"""tests/global_oracle.py against independent statements (scipy's rotations, planted view graphs and scenes, central
differences) and against k_global.h built for the host (tests/cpp/global_math_check.cpp); no GPU."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bundle_oracle as bo                # noqa: E402
import global_oracle as go                # noqa: E402


def _rotations(rng):
    """random rotations, plus ones near 0, near pi and exactly pi"""
    out = [go.random_rotation(rng) for _ in range(20)]
    for ang in (1e-10, 1e-5, 0.3, math.pi - 1e-3, math.pi - 1e-7, math.pi):
        w = rng.normal(size=3)
        out.append(bo.rodrigues(ang * w / np.linalg.norm(w)))
    return out


def test_log_exp_against_scipy():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(1)
    for R in _rotations(rng):
        w = go.log(R)
        ref = Rotation.from_matrix(R).as_rotvec()
        if np.linalg.norm(ref) > math.pi - 1e-6:       # at pi the sign of the axis is a convention
            assert abs(np.linalg.norm(w) - np.linalg.norm(ref)) < 1e-9
            assert np.abs(go.exp(w) - R).max() < 1e-9
        else:
            assert np.abs(w - ref).max() <= 1e-9 * max(1.0, np.linalg.norm(ref)), (w, ref)
    for s in (1e-9, 1e-3, 0.5, 3.0):
        w = rng.normal(size=3)
        w *= s / np.linalg.norm(w)
        assert np.abs(go.exp(w) - Rotation.from_rotvec(w).as_matrix()).max() < 1e-14


def _graph(seed, **kw):
    return go.view_graph(np.random.default_rng(seed), 50, 400, **kw)


def test_rotation_averaging_planted():
    """50 cameras, 400 pairs, 0.5 degree noise, 20 % outlier pairs: Cauchy IRLS has a median error below 0.3 degrees and
    beats the squared loss"""
    Rt, pairs, Rp, nf, out = _graph(2, noise_deg=0.5, outliers=0.2)
    med = {}
    for loss in ("cauchy", "squared"):
        R, reg, err, rep = go.rotation_averaging(50, pairs, Rp, nf, loss=loss, loss_scale=2.0, max_iters=50, min_inliers=0)
        assert reg.all() and rep["n_registered"] == 50
        e = go.rotation_errors(R, Rt)
        med[loss] = float(np.median(e))
        print(loss, rep, "median", med[loss], "max", e.max())
    assert med["cauchy"] < 0.3 and med["cauchy"] < med["squared"]


def test_rotation_start_is_spanning_tree():
    """with no noise and no outliers the spanning-tree start is the truth (up to the gauge), and IRLS stays there"""
    Rt, pairs, Rp, nf, _ = _graph(3, noise_deg=0.0, outliers=0.0)
    used, reg, root, R = go.start(50, pairs, Rp, nf, 0)
    assert root == 0 and reg.all() and used.all()
    assert go.rotation_errors(R, Rt).max() < 1e-10
    # the records hold float32 rotations (about 1e-5 degrees); their projections stay rotations along the chains
    R2, _, err, rep = go.rotation_averaging(50, pairs, Rp, nf, max_iters=5, min_inliers=0)
    assert go.rotation_errors(R2, Rt).max() < 1e-4 and err.max() < 1e-4
    assert max(np.abs(r.T @ r - np.eye(3)).max() for r in R2) < 1e-13


def test_rotation_components():
    """two components: the larger is registered; a tie goes to the component with the smallest set"""
    I = np.eye(3)
    pairs = [(0, 1), (2, 3), (3, 4), (5, 5)]
    Rp = np.stack([I, I, I, I])
    _, reg, root, _ = go.start(6, pairs, Rp, np.array([50, 50, 50, 50]), 15)
    assert list(reg) == [0, 0, 1, 1, 1, 0] and root == 2
    _, reg, root, _ = go.start(6, pairs[:3], Rp[:3], np.array([50, 50, 10]), 15)
    assert list(reg) == [1, 1, 0, 0, 0, 0] and root == 0


def _scene(seed, n_cams=6, n_tracks=80, **kw):
    rng = np.random.default_rng(seed)
    return bo.planted(rng, n_cams, list(rng.integers(2, n_cams + 1, size=n_tracks)), **kw)


def _positioning(sc, **kw):
    R = np.stack([np.asarray(R) for R, _ in sc["poses_true"]])
    return go.Positioning(sc["feats"], sc["cams"], R, np.ones(len(R), bool), sc["start"], sc["members"], **kw)


@pytest.mark.parametrize("loss", ["squared", "huber", "cauchy"])
def test_positioning_stationary_and_monotone(loss):
    """the cost never increases, and the converged point is a stationary point of the reduced cost"""
    sc = _scene(4, noise=0.3)
    P = _positioning(sc, loss=loss)
    pos = P.step(np.zeros((P.S + P.T, 3)), init=True)
    g0 = np.abs(P.free_gradient(pos)).max()
    costs = [P.cost(pos)]
    for _ in range(1500):           # majorise-minimise converges linearly: about 1 000 steps to 1e-6 here
        pos = P.step(pos)
        costs.append(P.cost(pos))
    assert all(b <= a * (1 + 1e-12) for a, b in zip(costs, costs[1:]))
    g1 = np.abs(P.free_gradient(pos)).max()
    print(loss, len(costs), costs[0], costs[-1], g0, g1)
    assert g1 <= 1e-6 * g0


def test_positioning_recovers_centres():
    """true rotations, 0.5 px noise: after similarity alignment the centres are within 1 % of the scene scale"""
    for seed in (5, 6):
        sc = _scene(seed, n_cams=8, n_tracks=200, noise=0.5)
        P = _positioning(sc)
        pos, rep = P.run(max_iters=200, function_tol=1e-12)
        poses, X = P.outputs(pos)
        C = np.stack([-R.T @ t for R, t in poses])
        Ct = np.stack([-np.asarray(R).T @ np.asarray(t) for R, t in sc["poses_true"]])
        A = go.align_centres(C, Ct)
        scale = np.linalg.norm(Ct - Ct.mean(0), axis=1).max()
        err = np.linalg.norm(A - Ct, axis=1).max() / scale
        print(rep, "max centre error / scene scale", err)
        assert err < 0.01
        assert abs(np.sqrt((C[P.positioned] ** 2).sum(1).mean()) - 1.0) < 1e-12


def test_positioning_participation():
    """a track with one registered member takes no part; an unregistered set is not positioned"""
    sc = _scene(7)
    R = np.stack([np.asarray(R) for R, _ in sc["poses_true"]])
    reg = np.ones(6, bool)
    reg[3] = False
    P = go.Positioning(sc["feats"], sc["cams"], R, reg, sc["start"], sc["members"])
    assert not P.positioned[3] and P.positioned[[0, 1, 2, 4, 5]].all()
    sets = [P.set[a:b] for a, b in zip(sc["start"][:-1], sc["start"][1:])]
    for t, s in enumerate(sets):
        assert P.tpart[t] == ((s != 3).sum() >= 2)


def _math_check(lines):
    from popsift_b200 import build as B
    if not os.path.exists(B.GLOBAL_MATH_CHECK):
        pytest.skip("global_math_check is not built")
    out = subprocess.run([B.GLOBAL_MATH_CHECK], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [[float(v) for v in ln.split()[1:]] for ln in out.stdout.splitlines()]


def _f(v):
    return " ".join("%.17g" % x for x in np.ravel(v))


def test_host_math_against_oracle():
    rng = np.random.default_rng(8)
    Rs = _rotations(rng)
    got = _math_check(["g " + _f(R) for R in Rs])
    for R, g in zip(Rs, got):
        assert np.abs(np.array(g) - go.log(R)).max() <= 1e-15 * max(1.0, np.linalg.norm(go.log(R))) + 1e-15
    got = _math_check(["q " + _f(R) for R in Rs])
    for R, g in zip(Rs, got):
        assert np.abs(np.array(g) - go.orthonormal(R).ravel()).max() <= 1e-15
        assert np.abs(go.orthonormal(R) - R).max() < 1e-6
    trip = [(Rs[k], Rs[k + 1], Rs[k + 2]) for k in range(10)]
    got = _math_check(["r " + _f(np.r_[a.ravel(), b.ravel(), c.ravel()]) for a, b, c in trip])
    for (a, b, c), g in zip(trip, got):
        assert np.abs(np.array(g) - go.pair_residual(a, b, c)).max() <= 1e-12
    xs = [rng.normal(scale=s, size=3) for s in (1e-9, 1e-3, 0.5)]
    got = _math_check(["u " + _f(np.r_[Rs[0].ravel(), x]) for x in xs])
    for x, g in zip(xs, got):
        assert np.abs(np.array(g) - (Rs[0] @ go.exp(x)).ravel()).max() <= 1e-15
    rows = [(rng.normal(size=3), rng.normal(size=3), rng.normal(size=3)) for _ in range(10)] + [(np.ones(3), np.zeros(3), np.zeros(3))]
    got = _math_check(["o " + _f(np.r_[v, X, c]) for v, X, c in rows])
    for (v, X, c), g in zip(rows, got):
        d, e = go.obs(v[None], X[None], c[None])
        assert abs(g[0] - d[0]) <= 1e-12 * max(1.0, abs(d[0])) and np.abs(np.array(g[1:4]) - e[0]).max() <= 1e-12
        assert abs(g[4] - float((e[0] * e[0]).sum())) <= 1e-12


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_global.h is exported and listed in api.GLOBAL_EXPORTS, apart from the others; the
    ctypes structures match the header"""
    import ctypes as C
    import re
    from popsift_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    body = open(os.path.join(root, "include", "popsift_b200_global.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.GLOBAL_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS,
                  api.BUNDLE_EXPORTS):
        assert not set(api.GLOBAL_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.GLOBAL_EXPORTS:
        assert hasattr(lib, name)
    structs = (("ps_rotation_params", api.PsRotationParams), ("ps_rotation_report", api.PsRotationReport),
               ("ps_position_params", api.PsPositionParams), ("ps_position_report", api.PsPositionReport))
    for struct, cls in structs:
        assert C.sizeof(cls) == 40
        block = body[body.index("typedef struct %s" % struct):]
        block = block[:block.index("} %s;" % struct)]
        names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct, names)
    for k, name in enumerate(api.RA_TERMINATION):
        assert "PS_RA_%s = %d" % (name.upper(), k) in body
    for k, name in enumerate(api.GP_TERMINATION):
        assert "PS_GP_%s = %d" % (name.upper(), k) in body


# ---- the Laplacian with the point nodes eliminated against the dense one ----

@pytest.mark.parametrize("loss", ["squared", "huber", "cauchy"])
def test_reduced_laplacian_equals_dense(loss):
    """positioning with an unregistered set, a track left with one member and a set without features; rotations with a
    set outside the registered component and a pair below min_inliers"""
    sc = _scene(9, n_cams=7, n_tracks=60, noise=0.3)
    sc["feats"] = list(sc["feats"][:4]) + [np.zeros((0, 2), np.float32)] + list(sc["feats"][4:])
    sc["cams"] = np.concatenate([sc["cams"][:4], sc["cams"][:1], sc["cams"][4:]])
    sc["poses_true"] = list(sc["poses_true"][:4]) + [sc["poses_true"][0]] + list(sc["poses_true"][4:])
    R = np.stack([np.asarray(r) for r, _ in sc["poses_true"]])
    reg = np.ones(8, bool)
    reg[2] = False
    kw = dict(loss=loss, loss_scale=0.1)
    a = go.Positioning(sc["feats"], sc["cams"], R, reg, sc["start"], sc["members"], **kw)
    b = go.Positioning(sc["feats"], sc["cams"], R, reg, sc["start"], sc["members"], solve=go.laplacian_solve_reduced, **kw)
    assert not a.positioned[[2, 4]].any() and (~a.tpart).any()
    pa, ra = a.run(max_iters=4, function_tol=0.0)
    pb, rb = b.run(max_iters=4, function_tol=0.0)
    assert np.abs(pa - pb).max() <= 1e-10 * np.abs(pa).max() and abs(ra["final_cost"] - rb["final_cost"]) <= 1e-10 * ra["final_cost"]
    W, g, _ = a.lin(pa)
    assert np.abs(go.laplacian_solve(a.S + a.T, a.ends, W, g, a.root) -
                  go.laplacian_solve_reduced(a.S + a.T, a.ends, W, g, a.root, n_cam=a.S)).max() <= 1e-10 * np.abs(pa).max()
    Rt, pairs, Rp, nf, _ = go.view_graph(np.random.default_rng(10), 30, 120, hub=(3, 20))
    pairs = pairs + [(30, 31)]
    Rp = np.concatenate([Rp, Rp[:1]])
    nf = np.r_[nf, 400]
    nf[5] = 3
    ra = go.rotation_averaging(32, pairs, Rp, nf, loss=loss, loss_scale=2.0, max_iters=3)
    rb = go.rotation_averaging(32, pairs, Rp, nf, loss=loss, loss_scale=2.0, max_iters=3, solve=go.laplacian_solve_reduced)
    assert not ra[1][30:].any() and ra[3]["n_pairs"] < len(pairs)
    assert np.abs(ra[0] - rb[0]).max() <= 1e-10 and abs(ra[3]["final_cost"] - rb[3]["final_cost"]) <= 1e-10 * ra[3]["final_cost"]
    fin = np.isfinite(ra[2])
    assert np.array_equal(fin, np.isfinite(rb[2])) and np.abs(ra[2][fin] - rb[2][fin]).max() <= 1e-9


def test_view_graph_hub():
    _, pairs, _, _, _ = go.view_graph(np.random.default_rng(11), 300, 600, hub=(7, 150))
    deg = np.bincount(np.asarray(pairs).reshape(-1), minlength=300)
    assert deg[7] >= 150 and len(set(map(tuple, pairs))) == 600


def test_large_oracles_runtime():
    """the largest positioning scene's first solve and the largest view graph's IRLS stay inside the GPU tests' budget"""
    import time
    import scale_shapes as ss
    t0 = time.perf_counter()
    sc = ss.SCENES["large"]()
    P = go.Positioning(sc["feats"], sc["cams"], sc["R"], np.ones(len(sc["R"]), bool), sc["start"], sc["members"],
                       solve=go.laplacian_solve_reduced)
    pos, rep = P.run(max_iters=1, function_tol=0.0)
    t1 = time.perf_counter()
    g = ss.GRAPHS["large"]()
    go.rotation_averaging(600, g[1], g[2], g[3], max_iters=1, min_inliers=0, solve=go.laplacian_solve_reduced)
    t2 = time.perf_counter()
    print("positioning %.1f s, rotations %.1f s" % (t1 - t0, t2 - t1), rep)
    assert rep["final_cost"] < rep["initial_cost"] and t2 - t0 < 40.0
