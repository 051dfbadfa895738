"""ps_view_graph_filter on the GPU against tests/viewgraph_oracle.py: keep, n_triangles and n_consistent exactly, min_error
to float rounding of values that agree to 1e-9 degrees, on planted graphs, out-lists at the warp-split boundaries with a
hub, a complete graph, a tree and the doppelganger case; unused pairs, duplicates and argument errors with the outputs
untouched; d_kept and determinism; rotation averaging on the kept pairs, global_poses with the filter on the rendered
views, and the C++ API against the C ABI."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import global_oracle as go                # noqa: E402
import viewgraph_oracle as vo             # noqa: E402
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
    rec["t"] = np.arange(3 * len(Rp), dtype=np.float32).reshape(-1, 3)    # bytes d_kept must carry over
    return rec


def run_vg(lib, n_sets, pairs, Rp, nf, prm, stats=True, kept=True):
    """ps_view_graph_filter with every host output prefilled with the sentinel and d_kept fenced by GUARD sentinel bytes on
    both sides: (rc, keep, stats or None, d_kept bytes or None, report, records)"""
    P = len(pairs)
    rec = _records(Rp, nf)
    keep = np.full(P + GUARD, SENTINEL, np.uint8)
    st = np.full((P + GUARD) * 12, SENTINEL, np.uint8)
    rep = api.PsViewGraphReport(-7, -7, -7, -7, -7, -7)
    nb = P * 128 + 2 * GUARD
    bufs = api._DevBuffers(lib)
    try:
        d = bufs.upload(rec) if P else None
        d_k = bufs.upload(np.full(nb, SENTINEL, np.uint8))
        rc = lib.ps_view_graph_filter(0, n_sets, P, api._c_pairs(pairs), d, C.byref(prm), keep.ctypes.data,
                                      st.ctypes.data if stats else None, d_k + GUARD if kept else None, C.byref(rep))
        got = bufs.download(d_k, nb, np.uint8)
    finally:
        bufs.free()
    assert (keep[P:] == SENTINEL).all() and (st[12 * P:] == SENTINEL).all(), "a write past an output"
    assert (got[:GUARD] == SENTINEL).all(), "a write before d_kept"
    if not stats:
        assert (st == SENTINEL).all()
    body = got[GUARD:GUARD + 128 * P]
    return rc, keep[:P], st[:12 * P].view(api.CYCLE_STATS_DTYPE) if stats else None, body, rep, rec


def _check(lib, n_sets, pairs, Rp, nf, **kw):
    """the device against the oracle; returns (oracle dict, device keep)"""
    o = vo.view_graph_filter(n_sets, pairs, Rp, nf, **kw)
    rc, keep, st, body, rep, rec = run_vg(lib, n_sets, pairs, Rp, nf, api._view_graph_params(**kw))
    assert rc == 0, api._last_error(lib)
    assert np.array_equal(keep.astype(bool), o["keep"]) and set(np.unique(keep)) <= {0, 1}
    assert np.array_equal(st["n_triangles"], o["n_triangles"]) and np.array_equal(st["n_consistent"], o["n_consistent"])
    fin = np.isfinite(o["min_error"])
    assert np.array_equal(np.isfinite(st["min_error"]), fin)
    m = st["min_error"][fin].astype(np.float64)
    want = o["min_error"][fin]
    assert (np.abs(m - want) <= 1e-9 + np.spacing(np.float32(want)).astype(np.float64)).all()
    r = o["report"]
    assert (rep.n_triangles, rep.n_consistent_triangles, rep.n_used, rep.n_kept, rep.n_untested) == (
        r["n_triangles"], r["n_consistent_triangles"], r["n_used"], r["n_kept"], r["n_untested"])
    n_kept = int(keep.sum())
    assert body[:128 * n_kept].tobytes() == rec[keep.astype(bool)].tobytes()
    assert (body[128 * n_kept:] == SENTINEL).all(), "a write past the kept records"
    return o, keep


@pytest.mark.parametrize("seed,n,p", [(1, 40, 300), (2, 300, 17700)])
def test_planted_against_oracle(lib, seed, n, p):
    Rt, pairs, Rp, nf, outl = vo.planted(np.random.default_rng(seed), n, p, noise_deg=0.5, outliers=0.1)
    for kw in (dict(min_inliers=0), dict(min_inliers=200, min_consistent=3, min_fraction=0.4, keep_untested=True),
               dict(min_inliers=0, max_cycle_error=0.5)):
        o, keep = _check(lib, n, pairs, Rp, nf, **kw)
        print(kw, o["report"])
    o, keep = _check(lib, n, pairs, Rp, nf, min_inliers=0)
    assert not keep[outl].any() and keep[~outl].all()


def test_warp_boundaries_and_hub(lib):
    """a hub of degree 1 000 and a complete graph on 34 sets, whose out-lists are 0 .. 33 long (0, 1, 31, 32, 33 among them),
    joined to the rest by one pair; both lists of an edge at every length up to 33"""
    rng = np.random.default_rng(3)
    Rt, pairs, Rp, nf, _ = vo.planted(rng, 1100, 4000, noise_deg=0.5, outliers=0.1, hub=(5, 1000))
    Rc = np.stack([go.random_rotation(rng) for _ in range(34)])
    cpairs = [(1100 + a, 1100 + b) for a, b in vo.complete(34)] + [(0, 1100)]
    Rall = np.concatenate([Rt, Rc])
    Rq = vo.exact_pairs(Rall, cpairs, rng, noise_deg=1.0)
    Rq[7] = go.random_rotation(rng)
    pairs2 = pairs + cpairs
    deg = np.bincount(np.asarray(pairs2).reshape(-1), minlength=1134)
    assert deg[5] >= 1000
    _check(lib, 1134, pairs2, np.concatenate([Rp, Rq]), np.r_[nf, np.full(len(cpairs), 300)], min_inliers=0)


def test_complete_graph(lib):
    rng = np.random.default_rng(4)
    Rt = np.stack([go.random_rotation(rng) for _ in range(70)])
    pairs = vo.complete(70)
    pairs = [(b, a) if k % 3 == 0 else (a, b) for k, (a, b) in enumerate(pairs)]     # some stored the other way round
    Rp = vo.exact_pairs(Rt, pairs, rng, noise_deg=1.0)
    bad = rng.choice(len(pairs), 100, replace=False)
    for p in bad:
        Rp[p] = go.random_rotation(rng)
    o, keep = _check(lib, 70, pairs, Rp, np.full(len(pairs), 100), min_fraction=0.5)
    assert o["report"]["n_triangles"] == 70 * 69 * 68 // 6 and not keep[bad].any()


def test_tree_is_untested(lib):
    rng = np.random.default_rng(5)
    Rt = np.stack([go.random_rotation(rng) for _ in range(50)])
    pairs = vo.tree(rng, 50)
    Rp = vo.exact_pairs(Rt, pairs)
    for ku in (False, True):
        o, keep = _check(lib, 50, pairs, Rp, np.full(49, 100), keep_untested=ku)
        assert o["report"]["n_triangles"] == 0 and o["report"]["n_untested"] == 49 and keep.all() == ku and keep.any() == ku


def test_doppelganger(lib):
    Rt, pairs, Rp, nf, bad = vo.doppelganger(np.random.default_rng(6))
    o, keep = _check(lib, len(Rt), pairs, Rp, nf)
    assert keep[bad].all()
    o, keep = _check(lib, len(Rt), pairs, Rp, nf, min_fraction=0.5)
    assert not keep[bad].any() and keep.sum() == len(pairs) - len(bad)


def test_unused_duplicates_and_errors(lib):
    rng = np.random.default_rng(7)
    Rt = np.stack([go.random_rotation(rng) for _ in range(12)])
    pairs = vo.complete(12) + [(3, 3)]
    Rp = np.concatenate([vo.exact_pairs(Rt, pairs[:-1]), np.eye(3)[None]])
    nf = np.full(len(pairs), 100)
    nf[4] = 14
    Rp[9, 1, 2] = np.inf
    o, keep = _check(lib, 12, pairs, Rp, nf)
    assert not o["used"][[4, 9, len(pairs) - 1]].any() and not keep[[4, 9, len(pairs) - 1]].any()
    rc, keep, st, body, rep, _ = run_vg(lib, 12, pairs, Rp, nf, api._view_graph_params())
    assert (st["n_triangles"][[4, 9, len(pairs) - 1]] == 0).all() and np.isinf(st["min_error"][[4, 9, len(pairs) - 1]]).all()
    # no stats, no d_kept
    rc2, keep2, _, body2, rep2, _ = run_vg(lib, 12, pairs, Rp, nf, api._view_graph_params(), stats=False, kept=False)
    assert rc2 == 0 and np.array_equal(keep, keep2) and bytes(rep) == bytes(rep2) and (body2 == SENTINEL).all()

    def untouched(r):
        rc, keep, st, body, rep, _ = r
        assert rc == PS_ERR_ARG and (keep == SENTINEL).all() and (st.view(np.uint8) == SENTINEL).all() and (body == SENTINEL).all()
        assert rep.n_used == -7 and rep.n_triangles == -7

    ok = vo.complete(12)
    Rok = vo.exact_pairs(Rt, ok)
    nok = np.full(len(ok), 100)
    for dup in ((0, 1), (1, 0)):       # a duplicate in either order
        untouched(run_vg(lib, 12, ok + [dup], np.concatenate([Rok, Rok[:1]]), np.r_[nok, 100], api._view_graph_params()))
    for kw in (dict(min_inliers=-1), dict(min_consistent=-1), dict(max_cycle_error=-1.0), dict(max_cycle_error=np.inf),
               dict(max_cycle_error=np.nan), dict(min_fraction=-0.1), dict(min_fraction=1.5)):
        untouched(run_vg(lib, 12, ok, Rok, nok, api._view_graph_params(**kw)))
    prm = api._view_graph_params()
    prm.keep_untested = 2
    untouched(run_vg(lib, 12, ok, Rok, nok, prm))
    untouched(run_vg(lib, 11, ok, Rok, nok, api._view_graph_params()))       # an index outside [0, n_sets)
    untouched(run_vg(lib, -1, [], Rok[:0], nok[:0], api._view_graph_params()))
    # NULL keep / report / prm, and d_two_view or d_kept on the host
    rep = api.PsViewGraphReport()
    keep = np.zeros(len(ok), np.uint8)
    host_rec = _records(Rok, nok)
    bufs = api._DevBuffers(lib)
    try:
        d = bufs.upload(host_rec)
        cp = api._c_pairs(ok)
        assert lib.ps_view_graph_filter(0, 12, len(ok), cp, d, C.byref(prm), None, None, None, C.byref(rep)) == PS_ERR_ARG
        assert lib.ps_view_graph_filter(0, 12, len(ok), cp, d, C.byref(api._view_graph_params()), keep.ctypes.data, None, None, None) == PS_ERR_ARG
        assert lib.ps_view_graph_filter(0, 12, len(ok), cp, d, None, keep.ctypes.data, None, None, C.byref(rep)) == PS_ERR_ARG
        assert lib.ps_view_graph_filter(0, 12, len(ok), None, d, C.byref(api._view_graph_params()), keep.ctypes.data, None, None,
                                        C.byref(rep)) == PS_ERR_ARG
        assert lib.ps_view_graph_filter(0, 12, len(ok), cp, host_rec.ctypes.data, C.byref(api._view_graph_params()), keep.ctypes.data,
                                        None, None, C.byref(rep)) == PS_ERR_ARG
        assert lib.ps_view_graph_filter(0, 12, len(ok), cp, d, C.byref(api._view_graph_params()), keep.ctypes.data, None,
                                        host_rec.ctypes.data, C.byref(rep)) == PS_ERR_ARG
        assert (keep == 0).all()
    finally:
        bufs.free()
    # empty calls
    rc, keep, st, body, rep, _ = run_vg(lib, 0, [], Rok[:0], nok[:0], api._view_graph_params())
    assert rc == 0 and rep.n_used == 0 and rep.n_triangles == 0
    rc, keep, st, body, rep, _ = run_vg(lib, 5, [], Rok[:0], nok[:0], api._view_graph_params())
    assert rc == 0 and rep.n_kept == 0


def test_determinism(lib):
    Rt, pairs, Rp, nf, _ = vo.planted(np.random.default_rng(8), 200, 8000, noise_deg=1.0, outliers=0.1)
    prm = api._view_graph_params(min_inliers=0, min_fraction=0.3)
    a = run_vg(lib, 200, pairs, Rp, nf, prm)
    b = run_vg(lib, 200, pairs, Rp, nf, prm)
    assert a[0] == 0 and a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes() and a[3].tobytes() == b[3].tobytes()
    assert bytes(a[4]) == bytes(b[4])


def test_rotation_averaging_on_kept_pairs(lib):
    """ps_rotation_averaging on the kept subset of the planted outlier graph: median below 0.1 degree, largest below 0.5;
    filter_view_graph (Python) agrees with the C call"""
    Rt, pairs, Rp, nf, outl = vo.planted(np.random.default_rng(5), 300, 17700, noise_deg=0.5, outliers=0.1)
    vg = api.filter_view_graph(300, pairs, [(R, n) for R, n in zip(Rp, nf)], min_inliers=0)
    o = vo.view_graph_filter(300, pairs, Rp, nf, min_inliers=0)
    assert np.array_equal(vg.keep, o["keep"]) and np.array_equal(vg.n_triangles, o["n_triangles"]) and vg.report.n_kept == o["report"]["n_kept"]
    k = np.flatnonzero(vg.keep)
    R, reg, err, rep = api.rotation_averaging(300, [pairs[p] for p in k], [(Rp[p], nf[p]) for p in k], loss="cauchy", loss_scale=2.0,
                                              max_iters=5, step_tol=0.0, cg_max_iters=50, cg_tol=1e-10, min_inliers=0)
    e = go.rotation_errors(R, Rt)
    print("kept", len(k), "median", np.median(e), "max", e.max(), rep)
    assert reg.all() and np.median(e) < 0.1 and e.max() < 0.5


# ---- the chain on test_pose's six rendered views ----

from test_triangulate import rendered_views   # noqa: E402,F401  (the module fixture)


def test_global_poses_with_filter(rendered_views):
    """every pair of the six views closes its triangles: the filter keeps all 15 and global_poses returns the same bytes"""
    imgs, cams, poses, sets = rendered_views
    pairs = [(i, j) for i in range(len(sets)) for j in range(i + 1, len(sets))]
    kw = dict(pose=dict(threshold=1.0, seed=1), rotation=dict(loss_scale=2.0), position=dict(max_iters=300, function_tol=1e-12))
    a = api.global_poses(sets, pairs, cams, **kw)
    b = api.global_poses(sets, pairs, cams, view_graph=dict(max_cycle_error=3.0), **kw)
    print("pair errors", a.pair_error)
    assert np.isfinite(b.pair_error).all() and a.pair_error.tobytes() == b.pair_error.tobytes()
    assert a.registered.tobytes() == b.registered.tobytes() and a.positioned.tobytes() == b.positioned.tobytes()
    assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(a.poses, b.poses))
    assert a.rotation_report == b.rotation_report and a.position_report == b.position_report
    def raw(v):
        return b"".join(np.asarray(x).tobytes() for x in v) if isinstance(v, list) else np.asarray(v).tobytes()

    for f in a.tracks._fields:
        assert raw(getattr(a.tracks, f)) == raw(getattr(b.tracks, f)), f
    with pytest.raises(api.PopSiftError):
        api.global_poses(sets, pairs, cams, view_graph=dict(min_inliers=3), **kw)


def test_cpp_api_against_c_abi():
    from popsift_b200 import build as B
    res = subprocess.run([B.VIEWGRAPH_CHECK], capture_output=True, text=True, timeout=300)
    print(res.stdout)
    assert res.returncode == 0 and res.stdout.startswith("OK"), res.stdout + res.stderr
