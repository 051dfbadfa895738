"""The triangulation oracle (tests/triangulate_oracle.py) without a GPU: its refinement against scipy's least squares, its
enumeration against a brute force, the exhaustive / sampled boundary, the host build of the kernels' math header, and the
header's exports and struct layouts."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import triangulate_oracle as tro      # noqa: E402
import verify_oracle as vo            # noqa: E402
from popsift_b200 import api          # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _track(rng, L, noise=0.5, outliers=0.0, shift=0.0):
    sc = tro.planted_scene(rng, max(L, 3) + 2, [L], noise=noise, outliers=outliers, shift=(shift, 0.0, 0.0))
    off = np.concatenate([[0], np.cumsum([len(f) for f in sc["feats"]])])
    sets = np.searchsorted(off, sc["members"], side="right") - 1
    xy = np.concatenate(sc["feats"])[sc["members"]]
    R = np.stack([sc["poses"][s][0] for s in sets])
    t = np.stack([sc["poses"][s][1] for s in sets])
    return xy[:, 0], xy[:, 1], sc["cams"][sets], R, t, sc


def test_refinement_against_least_squares():
    from scipy.optimize import least_squares
    rng = np.random.default_rng(0)
    n_ok = 0
    for k in range(40):
        L = int(rng.integers(3, 12))
        x, y, cam, R, t, sc = _track(rng, L, noise=0.7)
        rec, mask, err, inf = tro.triangulate_track(x, y, cam, R, t, k, 4.0, 1.0, 2, 256, 32, 1, info=True)
        if rec["status"] != tro.OK or inf["refit_count"] < inf["counts"][inf["win"]]:
            continue
        S0 = inf["e2"][inf["win"]] <= inf["thr2"]
        if not np.array_equal(S0, mask.astype(bool)):
            continue

        def res(X):
            _, ex, ey = tro.residual(cam[S0], R[S0], t[S0], X[None], x[S0], y[S0])
            return np.concatenate([ex, ey])
        ls = least_squares(res, rec["X"], xtol=1e-15, ftol=1e-15, gtol=1e-15)
        scale = np.linalg.norm(rec["X"] - tro.centre(R, t)[0])
        assert np.linalg.norm(ls.x - rec["X"]) <= 1e-7 * scale, (k, ls.x, rec["X"])
        # the kept steps decrease the cost, so the refined point's is the smallest of the trail
        assert abs(2 * ls.cost - min(inf["trail"])) <= 1e-6 * max(2 * ls.cost, 1e-9)
        n_ok += 1
    assert n_ok >= 30


def test_enumeration_brute_force():
    rng = np.random.default_rng(1)
    for k in range(25):
        L = int(rng.integers(2, 9))
        x, y, cam, R, t, sc = _track(rng, L, outliers=0.3)
        rec, mask, err, inf = tro.triangulate_track(x, y, cam, R, t, k, 3.0, 1.0, 2, 1000, 0, 0, info=True)
        C = tro.centre(R, t)
        _, d = tro.direction(cam, R, x, y)
        h = 0
        best, best_h = -1, -1
        for a in range(L):
            for b in range(a + 1, L):
                ok, X = tro.hypothesis(C[a], d[a], C[b], d[b], inf["cos_min"])
                cnt = -1
                if ok:
                    cnt = 0
                    for j in range(L):
                        fr, e2 = tro.error2(cam[j], R[j], t[j], X, x[j], y[j])
                        cnt += int(bool(fr) and float(e2) <= inf["thr2"])
                assert cnt == inf["counts"][h], (k, a, b)
                if cnt > best:
                    best, best_h = cnt, h
                h += 1
        assert h == L * (L - 1) // 2
        assert inf["win"] == best_h


def test_exhaustive_sampled_boundary():
    rng = np.random.default_rng(2)
    for L in (5, 8, 23):
        x, y, cam, R, t, _ = _track(rng, L)
        n = L * (L - 1) // 2
        _, _, _, inf = tro.triangulate_track(x, y, cam, R, t, 3, 4.0, 1.0, 2, n, 0, 9, info=True)
        assert len(inf["counts"]) == n                  # every pair at L (L - 1) / 2 == n_samples
        valid, a, b = tro.hypothesis_pairs(L, n, 9, 3)
        assert valid.all() and list(zip(a, b)) == [(i, j) for i in range(L) for j in range(i + 1, L)]
        _, _, _, inf = tro.triangulate_track(x, y, cam, R, t, 3, 4.0, 1.0, 2, n - 1, 0, 9, info=True)
        assert len(inf["counts"]) == n - 1             # drawn one below it
        valid, a, b = tro.hypothesis_pairs(L, n - 1, 9, 3)
        v2, idx = vo.samples(9, 3, np.arange(n - 1), L, 2)
        assert np.array_equal(valid, v2) and (a < b)[valid].all()
        assert np.array_equal(a, np.minimum(idx[:, 0], idx[:, 1])) and np.array_equal(b, np.maximum(idx[:, 0], idx[:, 1]))


def test_statuses():
    rng = np.random.default_rng(3)
    x, y, cam, R, t, _ = _track(rng, 6)
    assert tro.triangulate_track(x, y, cam, R, t, 0, 4.0, 1.0, 7, 256, 5, 0)[0]["status"] == tro.TOO_FEW_OBS
    assert tro.triangulate_track(x, y, cam, R, t, 0, 4.0, 1.0, 2, 256, 5, 0)[0]["status"] == tro.OK
    # every ray through one centre: parallel rays, no hypothesis
    R1, t1 = np.repeat(R[:1], 6, 0), np.repeat(t[:1], 6, 0)
    r = tro.triangulate_track(x, y, cam[:1].repeat(6, 0), R1, t1, 0, 4.0, 1.0, 2, 256, 5, 0)
    assert r[0]["status"] == tro.NO_HYPOTHESIS and not r[1].any() and np.isinf(r[2]).all()
    # a pair whose rays meet at less than min_angle is no hypothesis
    _, _, _, inf = tro.triangulate_track(x, y, cam, R, t, 0, 4.0, 60.0, 2, 256, 5, 0, info=True)
    _, d = tro.direction(cam, R, x, y)
    a, b = np.triu_indices(6, 1)
    narrow = tro.dot3(d[a], d[b]) > math.cos(math.radians(60.0))
    assert narrow.any() and (inf["counts"][narrow] == -1).all()


def _math_check(lines):
    from popsift_b200 import build as B
    if not os.path.exists(B.TRIANGULATE_MATH_CHECK):
        pytest.skip("triangulate_math_check is not built")
    out = subprocess.run([B.TRIANGULATE_MATH_CHECK], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [[float(v) for v in ln.split()[1:]] for ln in out.stdout.splitlines()]


def _fmt(vals):
    return " ".join("%.17g" % float(v) for v in vals)


def test_host_math_matches_oracle():
    """k_triangulate.h built for the host gives the oracle's bits: centres, rays, hypotheses, residuals and steps"""
    rng = np.random.default_rng(4)
    lines, want = [], []
    for k in range(300):
        x, y, cam, R, t, _ = _track(rng, 2, shift=float(rng.choice([0.0, 1e6])))
        c = cam.astype(np.float64)
        lines.append("c " + _fmt(np.r_[R[0].ravel(), t[0]]))
        want.append(list(tro.centre(R[0], t[0])))
        lines.append("d " + _fmt(np.r_[c[0], R[0].ravel(), t[0], x[0], y[0]]))
        ok, d = tro.direction(cam[0], R[0], x[0], y[0])
        want.append([float(ok)] + list(d))
        C = tro.centre(R, t)
        _, dd = tro.direction(cam, R, x, y)
        cm = math.cos(math.radians(float(rng.uniform(0, 5))))
        lines.append("h " + _fmt(np.r_[C[0], dd[0], C[1], dd[1], cm]))
        ok, X = tro.hypothesis(C[0], dd[0], C[1], dd[1], cm)
        want.append([float(ok)] + list(X if ok else np.zeros(3)))
        Xq = X if ok else C[0] + dd[0]
        lines.append("r " + _fmt(np.r_[c[1], R[1].ravel(), t[1], Xq, x[1], y[1]]))
        fr, ex, ey, Jx, Jy = tro.residual(cam[1], R[1], t[1], Xq, x[1], y[1], jac=True)
        want.append([float(fr)] + ([ex, ey] + list(Jx) + list(Jy) if fr else [0.0] * 8))
        S = np.r_[rng.normal(size=9), 0.0]
        A = rng.normal(size=(3, 3)); A = A @ A.T
        S[:6] = [A[0, 0], A[0, 1], A[0, 2], A[1, 1], A[1, 2], A[2, 2]]
        lines.append("s " + _fmt(S))
        ok, dX = tro.step(S)
        want.append([float(ok)] + list(dX))
    got = _math_check(lines)
    assert len(got) == len(want)
    for g, w, ln in zip(got, want, lines):
        assert np.array_equal(np.asarray(g), np.asarray(w, np.float64)), (ln[:1], g, w)


def test_header_exports():
    """every ps_*( of popsift_b200_triangulate.h is exported and listed in api.TRIANGULATE_EXPORTS, apart from the others"""
    hdr = open(os.path.join(ROOT, "include", "popsift_b200_triangulate.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    decl = sorted(set(re.findall(r"\b(ps_\w+)\(", hdr)))
    assert decl == sorted(api.TRIANGULATE_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS):
        assert not set(api.TRIANGULATE_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.TRIANGULATE_EXPORTS:
        assert hasattr(lib, name)


def test_struct_layouts():
    assert C.sizeof(api.PsRigid) == 96 and C.sizeof(api.PsTriangulateParams) == 32 and C.sizeof(api.PsTriangulateCounts) == 24
    assert api.TRACK_POINT_DTYPE.itemsize == 40 and tro.POINT_DTYPE == api.TRACK_POINT_DTYPE
    assert [f[0] for f in api.PsTriangulateParams._fields_] == ["max_error", "min_angle", "min_views", "n_samples", "refine_iters",
                                                                "pad_", "seed"]
    assert api.TRI_STATUS.index("ok") == tro.OK and api.TRI_STATUS.index("small_angle") == tro.SMALL_ANGLE
