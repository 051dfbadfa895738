"""The two-view configuration's contract in float64 (tests/twoview_oracle.py) against planted truth and, when it is
importable, OpenCV; the kernel's math built for the host (tests/cpp/twoview_math_check.cpp) against the oracle; the
classification rules on a table of counts; the header's exports and layouts.  No GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import pose_oracle as po                  # noqa: E402
import twoview_oracle as tvo              # noqa: E402


def _cv2():
    try:
        import cv2
        return cv2
    except Exception:
        return None


def _planted_h(rng, k):
    """(H_c as a caller would get it: scaled by a random factor of either sign, R, t / d, n, plane rows (calibrated)) for a
    random plane n . X = d in front of the left camera and a random pose"""
    R = tvo.random_rotation(rng, 1.0, 40.0)
    n = rng.normal(size=3) * np.array([0.4, 0.4, 1.0])
    n[2] = abs(n[2]) + 0.2
    n /= np.linalg.norm(n)
    d = rng.uniform(2.0, 10.0)
    t = rng.normal(size=3)
    t *= rng.uniform(0.2, 2.0) / np.linalg.norm(t)
    H = R + np.outer(t / d, n)
    xy = rng.uniform(-0.5, 0.5, (60, 2))
    ray = np.hstack([xy, np.ones((60, 1))])
    X = ray * (d / (ray @ n))[:, None]
    Xr = X @ R.T + t
    keep = (X[:, 2] > 0) & (Xr[:, 2] > 0)
    rows = np.hstack([X[keep, :2] / X[keep, 2:], Xr[keep, :2] / Xr[keep, 2:]])
    scale = rng.uniform(0.3, 3.0) * (1 if k % 2 else -1)
    return H * scale, R, t / d, n, rows


def _match(cands, R, td, n, tol):
    """index of the candidate equal to the truth"""
    for k, (Rc, tc, nc) in enumerate(cands):
        if np.abs(Rc - R).max() < tol and np.abs(tc - td).max() < tol and np.abs(nc - n).max() < tol:
            return k
    return None


def test_oracle_recovers_planted_planes():
    """the truth is one of the four candidates, in every position over the draws, and it survives the pruning and wins the
    cheirality count"""
    rng = np.random.default_rng(1)
    pos = set()
    n_unique = 0
    for k in range(400):
        Hs, R, td, n, rows = _planted_h(rng, k)
        Hn = tvo.h_signed(tvo.h_normalise(Hs), rows)
        cands = tvo.h_decompose(Hn)
        assert len(cands) == 4
        j = _match(cands, R, td, n, 1e-8)
        assert j is not None, k
        pos.add(j)
        keep = tvo.prune(cands)
        assert j in keep and len(keep) == 2
        w, tu, counts = tvo.choose([cands[i] for i in keep], rows)
        # every row is in front under the truth; the other kept candidate may explain them all too (the two-fold
        # ambiguity of a plane), and then the tie goes to the lower index
        assert counts[keep.index(j)] == len(rows), (k, counts)
        if counts[0] != counts[1]:
            assert keep[w] == j
            n_unique += 1
        for Rc, tc, nc in cands:
            assert np.abs(Rc @ Rc.T - np.eye(3)).max() < 1e-9 and abs(np.linalg.det(Rc) - 1) < 1e-9
            assert np.abs(Rc + np.outer(tc, nc) - Hn).max() < 1e-9
    assert pos == {0, 1, 2, 3}
    print("draws with a unique cheirality winner", n_unique, "of 400")
    assert n_unique > 100


def test_oracle_against_opencv():
    cv2 = _cv2()
    if cv2 is None:
        pytest.skip("cv2 is not importable")
    rng = np.random.default_rng(2)
    for k in range(100):
        Hs, R, td, n, rows = _planted_h(rng, k)
        Hn = tvo.h_signed(tvo.h_normalise(Hs), rows)
        ours = tvo.h_decompose(Hn)
        m, Rs, ts, ns = cv2.decomposeHomographyMat(Hn, np.eye(3))
        theirs = [(np.asarray(Rs[i]), np.asarray(ts[i]).ravel(), np.asarray(ns[i]).ravel()) for i in range(m)]
        for Rc, tc, nc in ours:
            assert any(np.abs(Rc - a).max() < 1e-6 and np.abs(tc - b).max() < 1e-6 and np.abs(nc - c).max() < 1e-6
                       for a, b, c in theirs), k


def test_oracle_no_parallax_and_rotation():
    rng = np.random.default_rng(3)
    for _ in range(50):
        R = tvo.random_rotation(rng, 0.5, 30.0)
        assert tvo.h_decompose(tvo.h_normalise(R * rng.uniform(0.5, 2))) == []
        a = tvo.rays(rng.uniform(-0.5, 0.5, (40, 2)))
        b = a @ R.T
        rows = np.hstack([a[:, :2] / a[:, 2:], b[:, :2] / b[:, 2:]])
        assert np.abs(tvo.kabsch(tvo.kabsch_sum(rows)) - R).max() < 1e-12


def _math_check(lines):
    from popsift_b200 import build as B
    if not os.path.exists(B.TWOVIEW_MATH_CHECK):
        pytest.skip("twoview_math_check is not built")
    out = subprocess.run([B.TWOVIEW_MATH_CHECK], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [[float(v) for v in ln.split()[1:]] for ln in out.stdout.splitlines()]


def _f(v):
    return " ".join("%.17g" % x for x in np.ravel(v))


def test_host_math_against_oracle():
    """k_twoview.h built for the host: Kabsch, the normalisation, sign count, decomposition, pruning, choice and angles
    within 1e-9 of the oracle"""
    rng = np.random.default_rng(4)
    lines, cases = [], []
    for k in range(200):
        Hs, R, td, n, rows = _planted_h(rng, k)
        lines.append("d " + _f(Hs))
        lines.append("c " + _f(Hs) + " " + _f(rows))
        B = tvo.kabsch_sum(rows + rng.normal(0, 1e-3, rows.shape))
        lines.append("k " + _f(B))
        cases.append((Hs, R, td, n, rows, B))
    got = _math_check(lines)
    n_chosen = 0
    for i, (Hs, R, td, n, rows, B) in enumerate(cases):
        d, c, kb = got[3 * i], got[3 * i + 1], got[3 * i + 2]
        Hn0 = tvo.h_normalise(Hs)
        xl = np.hstack([rows[:, :2], np.ones((len(rows), 1))]); xr = np.hstack([rows[:, 2:], np.ones((len(rows), 1))])
        assert int(c[0]) == int(((xr * (xl @ Hn0.T)).sum(1) > 0).sum())
        assert kb[0] == 1 and np.abs(np.array(kb[1:]).reshape(3, 3) - tvo.kabsch(B)).max() < 1e-9
        # the host decomposes the normalised H as given; the oracle the same, in the same order
        assert int(d[0]) == 4
        ours = tvo.h_decompose(Hn0)
        vals = np.array(d[1:61]).reshape(4, 15)
        for k in range(4):
            Rh, th, nh = vals[k, :9].reshape(3, 3), vals[k, 9:12], vals[k, 12:15]
            assert np.abs(Rh - ours[k][0]).max() < 1e-9 and np.abs(th - ours[k][1]).max() < 1e-9 and np.abs(nh - ours[k][2]).max() < 1e-9
        keep = [int(v) for v in d[61:65] if v >= 0]
        assert keep == tvo.prune(ours)
        # the choice between the kept candidates under the signed H
        Hn = tvo.h_signed(Hn0, rows)
        cands = tvo.h_decompose(Hn)
        kk = tvo.prune(cands)
        w, _, counts = tvo.choose([cands[j] for j in kk], rows)
        if counts[0] != counts[1]:
            assert _match([cands[kk[w]]], R, td, n, 1e-8) == 0
            n_chosen += 1
    assert n_chosen > 50
    # angles: pose_front's midpoint and the angle at it
    lines, ref = [], []
    for k in range(100):
        R = tvo.random_rotation(rng, 1.0, 20.0)
        t = rng.normal(size=3); t /= np.linalg.norm(t)
        X = rng.normal(size=3) * np.array([1, 1, 0.3]) + np.array([0, 0, 5.0])
        Xr = R @ X + t
        row = np.array([X[0] / X[2], X[1] / X[2], Xr[0] / Xr[2], Xr[1] / Xr[2]]) + rng.normal(0, 1e-4, 4)
        lines.append("f " + _f(R) + " " + _f(t) + " " + _f(row))
        ref.append((R, t, row))
    got = _math_check(lines)
    for (R, t, row), g in zip(ref, got):
        det, _, dl, dr, Xo = po.triangulate(R, t, row[None])
        assert g[0] == 1
        assert np.abs(np.array(g[1:4]) - Xo[0]).max() < 1e-9 * max(1.0, np.abs(Xo[0]).max())
        assert abs(g[4] - tvo.angle(Xo[0], R, t)[0]) < 1e-9


def test_classification_table():
    """step 2 on a table of counts, with each boundary on both sides (>= against >)"""
    C = tvo
    rows = [
        # n_e, n_f, n_h, min_inliers, ef, h, want
        (15, 15, 0, 15, 0.95, 0.8, C.GENERAL),
        (14, 15, 0, 15, 0.95, 0.8, C.UNCALIBRATED),      # n_e < min_inliers
        (14, 14, 0, 15, 0.95, 0.8, C.DEGENERATE),        # n_f < min_inliers
        (95, 100, 0, 15, 0.95, 0.8, C.GENERAL),          # n_e == ef * n_f
        (94, 100, 0, 15, 0.95, 0.8, C.UNCALIBRATED),     # just below
        (100, 100, 80, 15, 0.95, 0.8, C.GENERAL),        # n_h == h * n_e: not >
        (100, 100, 81, 15, 0.95, 0.8, C.PLANAR),         # just above
        (100, 100, 15, 15, 0.0, 0.1, C.PLANAR),          # n_h == min_inliers
        (100, 100, 14, 15, 0.0, 0.1, C.GENERAL),         # n_h < min_inliers
        (10, 100, 80, 15, 0.95, 0.8, C.UNCALIBRATED),    # m = n_f: 80 is not > 80
        (10, 100, 81, 15, 0.95, 0.8, C.PLANAR),
        (0, 0, 0, 0, 0.95, 0.8, C.GENERAL),              # every count 0 with min_inliers 0
        (0, 0, 0, 0, 0.95, 0.0, C.GENERAL),              # 0 > 0 is false
        (0, 10, 0, 1, 0.95, 0.8, C.UNCALIBRATED),
        (0, 0, 0, 1, 0.95, 0.8, C.DEGENERATE),
    ]
    for n_e, n_f, n_h, mi, ef, hr, want in rows:
        assert tvo.classify(n_e, n_f, n_h, mi, ef, hr) == want, (n_e, n_f, n_h, mi, ef, hr)
        assert tvo.classify(n_e, n_f, n_h, mi, ef, hr, allow_h=False) != tvo.PLANAR


def test_lower_median_rank():
    assert tvo.lower_median([]) == 0
    assert tvo.lower_median([3.0]) == 3.0
    assert tvo.lower_median([4.0, 1.0]) == 1.0
    assert tvo.lower_median([5.0, 1.0, 3.0]) == 3.0
    assert tvo.lower_median([5.0, 1.0, 3.0, 2.0]) == 2.0


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_twoview.h is exported and listed in api.TWOVIEW_EXPORTS, apart from the others; the
    ctypes structures and the info dtype match the header"""
    import ctypes as C
    import re
    from popsift_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    body = open(os.path.join(root, "include", "popsift_b200_twoview.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.TWOVIEW_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS,
                  api.BUNDLE_EXPORTS, api.GLOBAL_EXPORTS, api.VIEWGRAPH_EXPORTS):
        assert not set(api.TWOVIEW_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.TWOVIEW_EXPORTS:
        assert hasattr(lib, name)
    for struct, cls, size in (("ps_two_view_config_params", api.PsTwoViewConfigParams, 32), ("ps_two_view_info", api.PsTwoViewInfo, 40)):
        assert C.sizeof(cls) == size and "%d bytes" % size in body[body.index("typedef struct %s" % struct):][:80]
        block = body[body.index("typedef struct %s" % struct):]
        block = block[:block.index("} %s;" % struct)]
        names = re.findall(r"\b(\w+)\s*(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct, names)
    assert api.TWO_VIEW_INFO_DTYPE.names == tuple(f[0] for f in api.PsTwoViewInfo._fields_)
    enum = re.search(r"enum \{([^}]*PS_TV_[^}]*)\}", hdr).group(1)
    codes = dict((k.strip(), int(v)) for k, v in (e.split("=") for e in enum.split(",")))
    assert [codes["PS_TV_" + name.upper()] for name in api.TV_CONFIG] == list(range(5))
