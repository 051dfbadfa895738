"""tests/bundle_oracle.py against independent statements (central differences, a dense solve, scipy's least squares) and
against k_bundle.h built for the host (tests/cpp/bundle_math_check.cpp); no GPU."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import bundle_oracle as bo                # noqa: E402


def _scene(seed, n_cams=5, n_tracks=30):
    rng = np.random.default_rng(seed)
    sc = bo.planted(rng, n_cams, list(rng.integers(3, n_cams + 1, size=n_tracks)))
    bo.gauge_to_truth(sc, 0, 1, 2)
    return sc


def _fixed(n):
    f = np.zeros(n, np.uint8)
    f[0] = 1
    return f


@pytest.mark.parametrize("loss", bo.LOSSES)
def test_jacobians_central_differences(loss):
    sc = _scene(1)
    p = bo.problem(sc, _fixed(5), loss_kind=loss, loss_scale=2.0, scale_set=1, scale_axis=2)
    front, e, Jc, Jp = p.residuals(sc["poses"], sc["X0"])
    assert front.all()
    # unweighted Jacobian of the residuals over every free parameter
    _, _, Jc, Jp = p.residuals(sc["poses"], sc["X0"])
    h = 1e-6
    for c in range(p.n):
        d = np.zeros(p.n)
        d[c] = h
        _, ea, _, _ = p.residuals(*p.apply(sc["poses"], sc["X0"], d))
        _, eb, _, _ = p.residuals(*p.apply(sc["poses"], sc["X0"], -d))
        num = (ea - eb) / (2 * h)
        ana = np.zeros_like(num)
        for i, cols in p.cam_cols.items():
            if c in cols:
                k = cols.index(c)
                ana[p.set == i] = Jc[p.set == i, :, k]
        for j, c0 in p.pt_col.items():
            if c0 <= c < c0 + 3:
                ana[p.track == j] = Jp[p.track == j, :, c - c0]
        assert np.abs(num - ana).max() <= 1e-6 * max(1.0, np.abs(ana).max()), c
    # the IRLS gradient J^T W e is the gradient of the cost
    g = p.gradient(sc["poses"], sc["X0"])
    for c in range(0, p.n, 7):
        d = np.zeros(p.n)
        d[c] = 1e-6
        num = (p.cost(*p.apply(sc["poses"], sc["X0"], d)) - p.cost(*p.apply(sc["poses"], sc["X0"], -d))) / 2e-6
        assert abs(num - g[c]) <= 1e-5 * max(1.0, abs(g[c])), (c, num, g[c])


def test_schur_equals_dense():
    sc = _scene(2)
    p = bo.problem(sc, _fixed(5), loss_kind="huber", loss_scale=1.0, scale_set=1, scale_axis=2)
    for lam in (1e-6, 1e-3, 10.0):
        d1, pr1 = p.step(sc["poses"], sc["X0"], lam)
        d2, pr2 = p.step(sc["poses"], sc["X0"], lam, schur=True)
        assert np.abs(d1 - d2).max() <= 1e-9 * np.abs(d1).max()
        assert abs(pr1 - pr2) <= 1e-9 * abs(pr1) and pr1 > 0


def test_squared_loss_against_scipy():
    """the oracle's converged cost for the squared loss is scipy's least squares' on the same residuals and gauge"""
    from scipy.optimize import least_squares
    sc = _scene(3, n_cams=5, n_tracks=40)
    p = bo.problem(sc, _fixed(5), scale_set=1, scale_axis=2)
    _, _, rep = bo.lm(p, sc["poses"], sc["X0"], max_iters=100, function_tol=1e-14)

    def fun(x):
        _, e, _, _ = p.residuals(*p.apply(sc["poses"], sc["X0"], x))
        return e.reshape(-1)

    # scipy's own finite-difference Jacobian and trust-region solver: nothing of the oracle's solve is shared
    r = least_squares(fun, np.zeros(p.n), jac="2-point", method="trf", ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
    print("oracle", rep["final_cost"], "scipy", r.cost)
    assert abs(rep["final_cost"] - r.cost) <= 1e-8 * r.cost


def _math_check(lines):
    from popsift_b200 import build as B
    if not os.path.exists(B.BUNDLE_MATH_CHECK):
        pytest.skip("bundle_math_check is not built")
    out = subprocess.run([B.BUNDLE_MATH_CHECK], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [[float(v) for v in ln.split()[1:]] for ln in out.stdout.splitlines()]


def _f(v):
    return " ".join("%.17g" % x for x in np.ravel(v))


def test_host_math_against_oracle():
    sc = _scene(4)
    p = bo.problem(sc, _fixed(5))
    R = np.stack([np.asarray(sc["poses"][i][0]) for i in p.set])
    t = np.stack([np.asarray(sc["poses"][i][1]) for i in p.set])
    X = sc["X0"][p.track]
    front, e, Jc, Jp = bo.jacobian(p.cams[p.set], R, t, X, p.xy[:, 0], p.xy[:, 1])
    cam = p.cams[p.set].astype(np.float64)
    lines = ["j " + _f(np.r_[cam[u], R[u].ravel(), t[u], X[u], float(p.xy[u, 0]), float(p.xy[u, 1])]) for u in range(40)]
    got = _math_check(lines)
    for u, g in enumerate(got):
        assert g[0] == 1
        want = np.r_[e[u], Jc[u].ravel(), Jp[u].ravel()]
        assert np.abs(np.array(g[1:]) - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), u
    # losses
    zs = [0.0, 0.3, 1.0, 1.0000001, 7.5, 1e6]
    lines = ["l %d %.17g" % (k, z) for k in range(3) for z in zs]
    got = _math_check(lines)
    for (k, z), g in zip([(k, z) for k in range(3) for z in zs], got):
        rho, w = bo.loss(bo.LOSSES[k], z)
        assert g[0] == pytest.approx(float(rho), rel=1e-15, abs=0) and g[1] == pytest.approx(float(w), rel=1e-15, abs=0)
    # Rodrigues updates, including one below the series threshold and one of 90 degrees
    rng = np.random.default_rng(5)
    ds = [np.r_[rng.normal(scale=s, size=3), rng.normal(size=3)] for s in (1e-9, 1e-3, 0.1, 1.0)] + [np.r_[math.pi / 2, 0, 0, 0, 0, 0]]
    Rs, ts = sc["poses"][1]
    got = _math_check(["u " + _f(np.r_[np.ravel(Rs), ts, d]) for d in ds])
    for d, g in zip(ds, got):
        Rn, tn = bo.pose_update(np.asarray(Rs), ts, d)
        assert np.abs(np.array(g[:9]) - Rn.ravel()).max() <= 1e-15 and np.abs(np.array(g[9:]) - tn).max() <= 1e-14
        assert np.abs(Rn @ Rn.T - np.eye(3)).max() < 1e-14
    # the 6 x 6 Cholesky and solve, on an SPD matrix and on a singular one
    A = rng.normal(size=(6, 6))
    A = A @ A.T + 0.1 * np.eye(6)
    got = _math_check(["c " + _f(A), "c " + _f(np.zeros((6, 6)))])
    L = np.array(got[0][1:37]).reshape(6, 6)
    assert got[0][0] == 1 and np.abs(L - np.linalg.cholesky(A)).max() <= 1e-12 * np.abs(A).max()
    assert np.abs(np.array(got[0][37:]) - np.linalg.solve(A, np.arange(1.0, 7.0))).max() <= 1e-9 * np.abs(np.linalg.solve(A, np.arange(1.0, 7.0))).max()
    assert got[1][0] == 0
    # the 3 x 3 inverse
    V = rng.normal(size=(3, 3))
    V = V @ V.T + 0.5 * np.eye(3)
    got = _math_check(["i " + _f(V[np.triu_indices(3)])])
    Vi = np.linalg.inv(V)
    assert got[0][0] == 1 and np.abs(np.array(got[0][1:]) - Vi[np.triu_indices(3)]).max() <= 1e-12 * np.abs(Vi).max()


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_bundle.h is exported and listed in api.BUNDLE_EXPORTS, apart from the others; the
    ctypes structures match the header"""
    import ctypes as C
    import re
    from popsift_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "popsift_b200_bundle.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.BUNDLE_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS):
        assert not set(api.BUNDLE_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.BUNDLE_EXPORTS:
        assert hasattr(lib, name)
    assert C.sizeof(api.PsBundleParams) == 56 and C.sizeof(api.PsBundleReport) == 48
    body = open(os.path.join(root, "include", "popsift_b200_bundle.h")).read()
    for struct, cls in (("ps_bundle_params", api.PsBundleParams), ("ps_bundle_report", api.PsBundleReport)):
        block = body[body.index("typedef struct %s" % struct):]
        block = block[:block.index("} %s;" % struct)]
        names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct, names)
    for k, name in enumerate(api.BA_TERMINATION):
        assert "PS_BA_%s = %d" % (name.upper(), k) in body
    for k, name in enumerate(api.BA_LOSS):
        assert "PS_LOSS_%s = %d" % (name.upper(), k) in body
    assert bo.LOSSES == api.BA_LOSS


# ---- the vectorised Schur-complement step against the dense one ----

def _edge_scene(seed):
    """fixed sets 0 and 3, an empty set in the middle (4) and at the end (7), masked members, non-OK tracks"""
    import scale_shapes as ss
    import triangulate_oracle as tro
    rng = np.random.default_rng(seed)
    sc = ss.bundle_scene(seed, 8, lengths=list(rng.integers(2, 7, size=50)), empty=(4, 7), fixed=(0, 3))
    sc["mask"][::6] = 0
    sc["status"][::9] = tro.TOO_FEW_INLIERS
    return sc


@pytest.mark.parametrize("loss", bo.LOSSES)
def test_schur_step_equals_dense(loss):
    for seed, held in ((21, (1, 2)), (22, (5, 0)), (23, (-1, 0))):
        sc = _edge_scene(seed)
        p = bo.problem(sc, sc["fixed"], loss_kind=loss, loss_scale=2.0, scale_set=held[0], scale_axis=held[1])
        assert len(p.free) == 4 and (held[0] < 0 or p.held)
        for lam in (1e-4, 1e-3, 10.0):
            d1, pr1 = p.step(sc["poses"], sc["X0"], lam)
            d2, pr2, sy = p.schur_step(sc["poses"], sc["X0"], lam)
            assert np.abs(d1 - d2).max() <= 1e-10 * np.abs(d1).max(), (seed, lam)
            assert abs(pr1 - pr2) <= 1e-10 * abs(pr1) and pr1 > 0
            # the reduced system is the dense one's Schur complement
            J, e = p.system(sc["poses"], sc["X0"])
            H = J.T @ J
            H[np.diag_indices(p.n)] = bo.damp(np.diag(H), lam)
            A, B, C = H[:p.n_cam, :p.n_cam], H[:p.n_cam, p.n_cam:], H[p.n_cam:, p.n_cam:]
            g = J.T @ e
            Ci = np.linalg.inv(C)
            S = A - B @ Ci @ B.T
            assert np.abs(sy.S - S).max() <= 1e-10 * np.abs(S).max()
            assert np.abs(sy.b - (-g[:p.n_cam] + B @ Ci @ g[p.n_cam:])).max() <= 1e-10 * np.abs(sy.b).max()


def test_lm_with_schur_steps_equals_dense():
    sc = _edge_scene(24)
    p = bo.problem(sc, sc["fixed"], loss_kind="cauchy", loss_scale=2.0, scale_set=1, scale_axis=0)
    a = bo.lm(p, sc["poses"], sc["X0"], max_iters=4, initial_lambda=1e-3)
    b = bo.lm(p, sc["poses"], sc["X0"], max_iters=4, initial_lambda=1e-3, solve=bo.schur_step)
    assert a[2]["accepted"] == b[2]["accepted"] and a[2]["iterations"] == b[2]["iterations"] == 4
    assert abs(a[2]["final_cost"] - b[2]["final_cost"]) <= 1e-10 * a[2]["final_cost"]
    assert np.abs(a[1] - b[1]).max() <= 1e-9


# ---- the boundary table against the kernel sources ----

def kernel_constants():
    """kCamT, kT, kCgT (k_bundle.cu), kNodeT, kRedT (k_global.cu), kScanChunk and kRadixTile (k_scan.h)"""
    import re
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "popsift_b200", "csrc")

    def ints(name):
        return {m.group(1): m.group(2) for m in re.finditer(r"constexpr\s+(?:long long|int)\s+(\w+)\s*=\s*([^;]+);",
                                                             open(os.path.join(src, name)).read())}
    b, g, s = ints("k_bundle.cu"), ints("k_global.cu"), ints("k_scan.h")
    assert b["kT"] == g["kT"]
    k = {n: int(b[n]) for n in ("kCamT", "kT", "kCgT")}
    k.update({n: int(g[n]) for n in ("kNodeT", "kRedT")})
    env = {n: int(s[n]) for n in ("kScanT", "kScanPer", "kRadixT", "kRadixRounds")}
    k["kScanChunk"] = eval(s["kScanChunk"].replace("(long long)", ""), {}, env)
    k["kRadixTile"] = eval(s["kRadixTile"].replace("(long long)", ""), {}, env)
    assert int(s["kRadixT"]) == 256          # one digit per thread: the histogram has 256 entries per tile
    return k


def test_boundary_rows_sit_on_their_boundaries():
    """every row of tests/scale_shapes.py still straddles the boundary it names, so that a changed constant cannot leave
    a scale test running on the easy side"""
    import scale_shapes as ss
    k = kernel_constants()
    assert k == dict(kCamT=128, kT=256, kCgT=256, kNodeT=128, kRedT=256, kScanChunk=4096, kRadixTile=4096), k
    cache = {}
    for row, (kind, scene, doc, claims) in ss.ROWS.items():
        key = (kind == "rotation", scene)
        if key not in cache:
            cache[key] = (ss.GRAPHS if kind == "rotation" else ss.SCENES)[scene]()
        q = ss.quantities(kind, ss.stats(row, cache[key]), k)
        for name, want in claims.items():
            got = q[name][:len(want)] if isinstance(want, list) else q[name]
            assert got == want, (row, doc, name, got, want)
    # the rows come in pairs on each side of a boundary
    st = {r: ss.stats(r, cache[(ss.ROWS[r][0] == "rotation", ss.ROWS[r][1])]) for r in ss.ROWS}
    assert (st["ba_sets_256"]["S"], st["ba_sets_257"]["S"]) == (256, 257) and (st["gp_sets_255"]["S"], st["gp_sets_256"]["S"]) == (255, 256)
    assert list(st["ba_counts"]["counts"][:6]) == list(ss.COUNTS) + [ss.FIXED_COUNT] and st["ba_counts"]["counts"][[8, 21]].sum() == 0
    assert (st["ba_tracks_256"]["T"], st["ba_tracks_257"]["T"]) == (256, 257)
    assert [st["ba_members_%d" % m]["M"] for m in (4095, 4096, 4097)] == [4095, 4096, 4097]
    assert st["ba_large"]["T"] > 65536 and st["ba_large"]["S"] + st["ba_large"]["T"] > 256 * 256
    assert (st["ra_pairs_256"]["P"], st["ra_pairs_257"]["P"]) == (256, 257) and st["ra_large"]["P"] > 65536
    assert st["ra_sets_257_hub"]["S"] == 257 and st["ra_sets_257_hub"]["degree"].max() >= 129


def test_large_oracle_runtime():
    """the largest bundle scene's scene, Schur step and costs stay well inside the GPU tests' budget"""
    import time
    import scale_shapes as ss
    t0 = time.perf_counter()
    sc = ss.SCENES["large"]()
    p = bo.problem(sc, sc["fixed"])
    d, pred, _ = p.schur_step(sc["poses"], sc["X0"], 1e-3)
    c0 = p.cost(sc["poses"], sc["X0"])
    c1 = p.cost(*p.apply(sc["poses"], sc["X0"], d))
    dt = time.perf_counter() - t0
    print("large: %d observations, %d camera columns, %.1f s" % (len(p.set), p.n_cam, dt))
    assert c1 < c0 and pred > 0 and dt < 30.0
