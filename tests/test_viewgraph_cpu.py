"""tests/viewgraph_oracle.py against independent statements (brute-force triangles, exact and perturbed cycles, planted
outlier graphs with global_oracle's rotation averaging downstream) and against k_viewgraph.h built for the host
(tests/cpp/viewgraph_math_check.cpp); the header's exports and layouts; no GPU."""
import itertools
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import global_oracle as go                # noqa: E402
import viewgraph_oracle as vo             # noqa: E402


def _random_graph(rng, n, density):
    pairs = [(i, j) if rng.random() < 0.5 else (j, i) for i in range(n) for j in range(i + 1, n) if rng.random() < density]
    return pairs


def test_triangles_brute_force():
    """the oracle's triangles are exactly the triples of itertools.combinations whose three pairs are used"""
    rng = np.random.default_rng(1)
    for n, density in ((8, 0.6), (15, 0.3), (25, 0.2), (12, 1.0)):
        pairs = _random_graph(rng, n, density)
        used = rng.random(len(pairs)) < 0.85
        tri, tp = vo.triangles(n, pairs, used)
        edge = {}
        for p, (a, b) in enumerate(pairs):
            if used[p]:
                edge[(min(a, b), max(a, b))] = p
        want = [(a, b, c) for a, b, c in itertools.combinations(range(n), 3) if (a, b) in edge and (b, c) in edge and (a, c) in edge]
        assert [tuple(t) for t in tri] == want
        for (a, b, c), (pab, pbc, pca) in zip(tri, tp):
            assert (pab, pbc, pca) == (edge[(a, b)], edge[(b, c)], edge[(a, c)])


def test_cycle_error_exact_direction_and_planted_angle():
    rng = np.random.default_rng(2)
    Rt = np.stack([go.random_rotation(rng) for _ in range(12)])
    pairs = vo.complete(12)
    Rp = vo.exact_pairs(Rt, pairs)
    used = np.ones(len(pairs), bool)
    tri, tp = vo.triangles(12, pairs, used)
    assert len(tri) == 220
    e = vo.cycle_errors(pairs, Rp, tri, tp)
    assert e.max() < 1e-12
    # stored the other way round: the same errors (to rounding), on a noisy graph
    Rn = vo.exact_pairs(Rt, pairs, rng, noise_deg=2.0)
    flipped = [(b, a) for a, b in pairs]
    Rf = np.swapaxes(Rn, 1, 2)
    e1 = vo.cycle_errors(pairs, Rn, tri, tp)
    e2 = vo.cycle_errors(flipped, Rf, tri, tp)
    assert e1.max() > 0.5 and np.abs(e1 - e2).max() <= 1e-12
    # one edge turned by a planted angle about a random axis: its triangles have exactly that error
    for ang in (0.5, 7.0, 90.0, 179.0):
        Rq = Rp.copy()
        w = rng.normal(size=3)
        Rq[5] = go.exp(w / np.linalg.norm(w) * ang * vo.DEG) @ Rp[5]
        e = vo.cycle_errors(pairs, Rq, tri, tp)
        hit = (tp == 5).any(1)
        assert hit.sum() == 10 and np.abs(e[hit] - ang).max() < 1e-9 and e[~hit].max() < 1e-12


def test_filter_rules():
    """statistics and the one-pass decision on a small graph, against a direct count; unused pairs neither counted nor kept"""
    rng = np.random.default_rng(3)
    n = 10
    Rt = np.stack([go.random_rotation(rng) for _ in range(n)])
    pairs = vo.complete(n)[:30] + [(9, 9)]
    Rp = np.concatenate([vo.exact_pairs(Rt, pairs[:-1], rng, 1.0), np.eye(3)[None]])
    Rp[3] = go.random_rotation(rng)
    nf = np.full(len(pairs), 100)
    nf[7] = 4
    Rp[11, 0, 0] = np.nan
    out = vo.view_graph_filter(n, pairs, Rp, nf, max_cycle_error=3.0, min_consistent=2)
    used = out["used"]
    assert not used[[7, 11, 30]].any() and used.sum() == len(pairs) - 3
    assert (out["n_triangles"][~used] == 0).all() and np.isinf(out["min_error"][~used]).all() and not out["keep"][~used].any()
    tri = out["triangles"]
    for p, (a, b) in enumerate(pairs):
        if not used[p]:
            continue
        mine = [k for k, t in enumerate(tri) if a in t and b in t]
        assert out["n_triangles"][p] == len(mine)
        assert out["n_consistent"][p] == sum(out["errors"][k] <= 3.0 for k in mine)
        want = out["n_consistent"][p] >= 2 if mine else False
        assert out["keep"][p] == want
    assert not out["keep"][3]
    rep = out["report"]
    assert rep["n_used"] == used.sum() and rep["n_kept"] == out["keep"].sum() and rep["n_triangles"] == len(tri)


def test_doppelganger_rule():
    """the wrong pairs of set 0 close among the group: kept at min_consistent 1, dropped at min_fraction 0.5"""
    Rt, pairs, Rp, nf, bad = vo.doppelganger(np.random.default_rng(4))
    a = vo.view_graph_filter(len(Rt), pairs, Rp, nf)
    b = vo.view_graph_filter(len(Rt), pairs, Rp, nf, min_fraction=0.5)
    assert a["keep"][bad].all() and (a["n_consistent"][bad] == 2).all()
    assert not b["keep"][bad].any() and b["keep"].sum() == len(pairs) - len(bad)


def test_planted_outliers_and_rotation_averaging():
    """300 cameras, 17 700 pairs, 10 % outlier pairs with n_front drawn like the inliers': every outlier dropped, no inlier
    dropped, and
    rotation averaging on the kept pairs reaches a median error below 0.1 degree and a largest below 0.5"""
    Rt, pairs, Rp, nf, outl = vo.planted(np.random.default_rng(5), 300, 17700, noise_deg=0.5, outliers=0.1)
    out = vo.view_graph_filter(300, pairs, Rp, nf, max_cycle_error=3.0, min_inliers=0)
    keep = out["keep"]
    print(out["report"], "outliers", outl.sum())
    assert not keep[outl].any() and keep[~outl].all()
    kw = dict(loss="cauchy", loss_scale=2.0, max_iters=5, min_inliers=0, solve=go.laplacian_solve_reduced)
    k = np.flatnonzero(keep)
    R, reg, _, _ = go.rotation_averaging(300, [pairs[p] for p in k], Rp[k], nf[k], **kw)
    e = go.rotation_errors(R, Rt)
    R0, _, _, _ = go.rotation_averaging(300, pairs, Rp, nf, **kw)
    e0 = go.rotation_errors(R0, Rt)
    print("all pairs: median %.3f max %.3f; kept: median %.4f max %.4f" % (np.median(e0), e0.max(), np.median(e), e.max()))
    assert reg.all() and np.median(e) < 0.1 and e.max() < 0.5


def _math_check(lines):
    from popsift_b200 import build as B
    if not os.path.exists(B.VIEWGRAPH_MATH_CHECK):
        pytest.skip("viewgraph_math_check is not built")
    out = subprocess.run([B.VIEWGRAPH_MATH_CHECK], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return [float(ln.split()[1]) for ln in out.stdout.splitlines()]


def test_host_math_against_oracle():
    """vg_cycle_error built for the host against the oracle's, to 1e-12 degrees, every storage direction, near 0 and pi"""
    rng = np.random.default_rng(6)
    rows = []
    for k in range(40):
        Rs = [go.random_rotation(rng) for _ in range(3)]
        if k % 4 == 1:      # a nearly closed cycle
            Rs[2] = (Rs[1] @ Rs[0]).T @ go.exp(rng.normal(size=3) * 1e-6)
        if k % 4 == 2:      # a cycle near pi
            w = rng.normal(size=3)
            Rs[2] = (Rs[1] @ Rs[0]).T @ go.exp(w / np.linalg.norm(w) * (math.pi - 1e-4))
        ts = [int(v) for v in rng.integers(0, 2, size=3)]
        # the stored matrices: transposed where the pair is stored the other way round
        St = [R.T if t else R for R, t in zip(Rs, ts)]
        rows.append((St, ts))
    lines = ["c " + " ".join(" ".join("%.17g" % v for v in np.ravel(S)) + " %d" % t for S, t in zip(St, ts)) for St, ts in rows]
    got = _math_check(lines)
    for (St, ts), g in zip(rows, got):
        want = vo.cycle_error(St[0], ts[0], St[1], ts[1], St[2], ts[2])
        assert abs(g - want) <= 1e-12, (g, want)


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_viewgraph.h is exported and listed in api.VIEWGRAPH_EXPORTS, apart from the others; the
    ctypes structures match the header"""
    import ctypes as C
    import re
    from popsift_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    body = open(os.path.join(root, "include", "popsift_b200_viewgraph.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.VIEWGRAPH_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS,
                  api.BUNDLE_EXPORTS, api.GLOBAL_EXPORTS):
        assert not set(api.VIEWGRAPH_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.VIEWGRAPH_EXPORTS:
        assert hasattr(lib, name)
    structs = (("ps_view_graph_params", api.PsViewGraphParams, 32), ("ps_cycle_stats", api.PsCycleStats, 12),
               ("ps_view_graph_report", api.PsViewGraphReport, 32))
    for struct, cls, size in structs:
        assert C.sizeof(cls) == size and "%d bytes" % size in body[body.index("typedef struct %s" % struct):][:80]
        block = body[body.index("typedef struct %s" % struct):]
        block = block[:block.index("} %s;" % struct)]
        names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct, names)
    assert api.CYCLE_STATS_DTYPE.names == tuple(f[0] for f in api.PsCycleStats._fields_)
