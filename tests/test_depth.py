"""ps_depth_maps and ps_depth_filter on the GPU against tests/depth_oracle.py and against the ray-cast truth of test_pose's
rendered scene, the chain from global poses to dense points, determinism, image layouts and argument errors."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import depth_oracle as do                                   # noqa: E402
from popsift_b200 import api                                # noqa: E402
from test_pose import CAMS, W, H, _cast                      # noqa: E402
from test_triangulate import VIEWS, _view_pose, rendered_views   # noqa: E402,F401  (rendered_views: the module fixture)

pytestmark = pytest.mark.gpu

PS_ERR_ARG = -1


def _truth_depth(cam, R, t, w, h):
    """camera-frame depth of every pixel by ray casting (the renderer's Z is the world z of the hit)"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    Z, v = _cast(cam, R, t, x.ravel(), y.ravel())
    d = R.T @ np.linalg.solve(do.K(cam), np.stack([x.ravel(), y.ravel(), np.ones(h * w)]))
    o = -R.T @ t
    lam = (Z - o[2]) / d[2]
    return lam.reshape(h, w), np.clip(np.rint(v), 0, 255).astype(np.uint8).reshape(h, w)


def _rendered(scale):
    """the six views of test_triangulate at 1280 x 960 times scale: images, cameras, poses, true depths"""
    w, h = int(W * scale), int(H * scale)
    imgs, cams, poses, truth = [], [], [], []
    for k, (Rv, Cv) in enumerate(VIEWS):
        cam = np.asarray(CAMS[k % 2], np.float64) * scale
        R, t = _view_pose(Rv, Cv)
        D, im = _truth_depth(cam, R, t, w, h)
        imgs.append(im); cams.append(cam.astype(np.float32)); poses.append((R, t)); truth.append(D)
    return imgs, cams, poses, truth


def _true_range(D):
    return float(np.percentile(D, 0.5) * 0.8), float(np.percentile(D, 99.5) * 1.25)


def _random_scene(seed, h=120, w=160, n=4):
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(seed)
    imgs = []
    for _ in range(n):
        a = gaussian_filter(rng.normal(size=(h, w)), 1.0)
        imgs.append(np.clip(np.rint((a - a.mean()) / a.std() * 50 + 128), 0, 255).astype(np.uint8))
    cams = [np.array([140.0, 145.0, 80.0, 60.0], np.float32)] * n
    poses = [(np.eye(3), np.zeros(3))]
    for k in range(1, n):
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        th = np.radians(rng.uniform(0, 3))
        S = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.cos(th) * np.eye(3) + np.sin(th) * S + (1 - np.cos(th)) * np.outer(a, a)
        poses.append((R, rng.normal(size=3) * 0.15))
    return imgs, cams, poses


PRM = dict(radius=3, top_k=3, min_sources=1, max_cost=2.0, min_var=1.0)


def _oracle_maps(imgs, cams, poses, refs, sources, ranges, n_depths, **prm):
    return [do.depth_map(imgs[r], cams[r], poses[r], [(imgs[s], cams[s], poses[s]) for s in sources[j]], ranges[j][0], ranges[j][1],
                         n_depths=n_depths, **prm) for j, r in enumerate(refs)]


def _compare(dev, ora, tag):
    stats = []
    for j, o in enumerate(ora):
        d, c, ns = dev.depth[j], dev.cost[j], dev.n_src[j]
        h, w = d.shape
        cand = do.candidates(h, w, PRM["radius"])
        # non-candidates: no winner
        assert (d[~cand] == 0).all() and np.isinf(c[~cand]).all() and (ns[~cand] == 0).all()
        has = np.isfinite(o["cost"])
        assert np.array_equal(np.isfinite(c), has), tag
        sel = has & (o["margin"] >= 1e-3) & o["var_ok"]
        iota = o["iota"]
        di = iota[1] - iota[0]
        # the winner: within half a plane step everywhere, so k* is the oracle's
        pos = (1.0 / d[has] - iota[0]) / di
        near = np.abs(pos - (1.0 / o["depth"][has] - iota[0]) / di) <= 0.5 + 1e-3
        assert near.mean() >= 0.999, (tag, near.mean())
        assert (np.abs((1.0 / d[sel] - iota[0]) / di - o["k"][sel]) <= 0.5 + 1e-4).all(), tag
        ce = np.abs(c[sel] - o["cost"][sel])
        de = np.abs(d[sel] / o["depth"][sel] - 1)
        fc, fd, fn = (ce <= 1e-4).mean(), (de <= 1e-4).mean(), (ns[sel] == o["n_src"][sel]).mean()
        stats.append((int(sel.sum()), fc, fd, fn, float(ce.max()), float(de.max())))
        assert fc >= 0.999 and fd >= 0.999 and fn >= 0.999, (tag, stats[-1])
        assert dev.report["candidates"] == sum(int(do.candidates(*x.shape, PRM["radius"]).sum()) for x in dev.depth)
        assert dev.report["depths"] == sum(int((x > 0).sum()) for x in dev.depth)
    print(tag, "compared pixels, cost / depth / n_src agreement, largest cost and relative depth error", stats)


def _compare_filter(dev, imgs, cams, poses, refs, sources, fprm):
    nc, pts = do.depth_filter(dev.depth, imgs, cams, poses, refs, sources, **fprm)
    mism = sum(int((a != b).sum()) for a, b in zip(nc, dev.n_consistent))
    total = sum(a.size for a in nc)
    assert mism <= max(2, 1e-4 * total), mism
    key = {(p[1], p[3], p[2]): p for p in pts}
    got = dev.points
    order = list(zip(got["ref"], got["y"], got["x"]))
    assert order == sorted(order)
    assert dev.filter_report["points"] == len(got)
    match = 0
    for rec in got:
        p = key.get((int(rec["ref"]), int(rec["y"]), int(rec["x"])))
        if p is None:
            continue
        match += 1
        assert np.allclose(rec["X"], p[0], rtol=1e-6, atol=1e-6) and rec["n_consistent"] == p[4] and rec["grey"] == p[5]
    assert match >= len(pts) - max(2, 1e-4 * total) and len(got) - match <= max(2, 1e-4 * total)


@pytest.mark.parametrize("scene", ["random", "rendered160", "rendered320"])
def test_against_oracle(scene):
    if scene == "random":
        imgs, cams, poses = _random_scene(1)
        refs, sources = [0, 1], [[1, 2, 3], [0, 2, 3]]
        ranges = [(2.0, 12.0), (1.5, 20.0)]
        n = 48
    else:
        scale = 0.125 if scene == "rendered160" else 0.25
        imgs, cams, poses, truth = _rendered(scale)
        refs, sources = ([0, 3], [[1, 2, 3, 4, 5], [0, 1, 2]]) if scene == "rendered160" else ([0], [[1, 2, 3, 4, 5]])
        ranges = [_true_range(truth[r]) for r in refs]
        n = 32 if scene == "rendered160" else 64
    fprm = dict(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=1)
    dev = api.depth_maps(imgs, cams, poses, refs, sources, ranges, n_depths=n, filter=fprm, **PRM)
    ora = _oracle_maps(imgs, cams, poses, refs, sources, ranges, n, **PRM)
    # measured on the H100: cost and n_src agree on 100 % of the compared pixels, depth on >= 99.994 %; the largest cost
    # difference 2.4e-5, the largest relative depth difference 1.0e-4
    _compare(dev, ora, scene)
    _compare_filter(dev, imgs, cams, poses, refs, sources, fprm)


def _errors(depth, truth):
    ok = depth > 0
    rel = np.abs(depth[ok] / truth[ok] - 1)
    return ok.mean(), float(np.median(rel)), float(np.percentile(rel, 90)), float((rel > 0.05).mean())


def test_against_truth_640():
    imgs, cams, poses, truth = _rendered(0.5)
    refs = list(range(6))
    sources = [[s for s in range(6) if s != r] for r in refs]
    ranges = [_true_range(truth[r]) for r in refs]
    fprm = dict(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2)
    dev = api.depth_maps(imgs, cams, poses, refs, sources, ranges, n_depths=128, radius=3, top_k=3, max_cost=0.5, filter=fprm)
    rows = [_errors(dev.depth[j], truth[r]) for j, r in enumerate(refs)]
    frac = np.mean([r[0] for r in rows])
    allrel = np.concatenate([np.abs(dev.depth[j][dev.depth[j] > 0] / truth[r][dev.depth[j] > 0] - 1) for j, r in enumerate(refs)])
    med, p90, above = float(np.median(allrel)), float(np.percentile(allrel, 90)), float((allrel > 0.05).mean())
    # the kept points against the truth at their pixels
    pts = dev.points
    dd = np.stack(dev.depth)[pts["ref"], pts["y"], pts["x"]]
    kept = np.abs(dd / np.stack(truth)[np.asarray(refs)[pts["ref"]], pts["y"], pts["x"]] - 1)
    above_f = float((kept > 0.05).mean())
    print("640 x 480, six references: per reference (with depth, median, p90, > 5 %)", rows, "overall with depth", frac, "median",
          med, "p90", p90, "> 5 %", above, "filtered points", len(pts), "> 5 %", above_f, "report", dev.report, dev.filter_report)
    # measured on the H100: 93.1 % of the pixels with a depth (view 0 alone 96.6 %, views 2 and 4, which see the most
    # occlusion, 84-86 %), median relative error 0.22 %, p90 1.02 %, 2.9 % above 5 %; after the filter 1 487 137 points,
    # 0.001 % of them above 5 %
    assert frac >= 0.93 and med < 0.003 and p90 < 0.012
    assert above_f < above


def test_chain_from_global_poses(rendered_views):
    """global_poses -> triangulate -> bundle_adjust -> depth_ranges / select_sources -> depth_maps(filter) at full size,
    against the true depth after the similarity that aligns the estimated centres to the true ones"""
    imgs, cams, poses, sets = rendered_views
    pairs = [(i, j) for i in range(len(sets)) for j in range(i + 1, len(sets))]
    gp = api.global_poses(sets, pairs, cams, pose=dict(threshold=1.0, seed=1), rotation=dict(loss_scale=2.0),
                          position=dict(max_iters=1500, function_tol=1e-12))
    tp = api.triangulate(sets, gp.tracks, cams, gp.poses, max_error=4.0, min_angle=1.0, seed=2)
    est, tp2, rep = api.bundle_adjust(sets, gp.tracks, tp, cams, gp.poses, [True] + [False] * 5, loss="cauchy", loss_scale=2.0,
                                      max_iters=100, function_tol=1e-10, cg_tol=1e-8, scale_set=1, scale_axis=0)
    n = len(sets)
    ranges = api.depth_ranges(gp.tracks, tp2, est, n)
    srcs = api.select_sources(gp.tracks, tp2, est, n_sources=5, min_angle=1.0)
    refs = [i for i in range(n) if ranges[i, 1] > 0 and srcs[i]]
    dev = api.depth_maps(imgs, cams, est, refs, [srcs[r] for r in refs], [ranges[r] for r in refs], n_depths=128, radius=3, top_k=3,
                         max_cost=0.5, filter=dict(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2))
    # the similarity: the true centres from the estimated ones (scale; view 0 is the gauge origin in both)
    Ce = np.stack([-R.T @ t for R, t in est])
    Ct = np.stack([-R.T @ t for R, t in poses])
    s = float(((Ce - Ce[0]) * (Ct - Ct[0])).sum() / ((Ce - Ce[0]) ** 2).sum())
    truth = [_truth_depth(np.asarray(cams[r], np.float64), poses[r][0], poses[r][1], W, H)[0] for r in refs]
    rows = [_errors(dev.depth[j] * s, truth[j]) for j in range(len(refs))]
    allrel = np.concatenate([np.abs(dev.depth[j][dev.depth[j] > 0] * s / truth[j][dev.depth[j] > 0] - 1) for j in range(len(refs))])
    print("chain: refs", refs, "sources", srcs, "ranges", ranges.tolist(), "scale", s, "per reference (with depth, median, p90, > 5 %)",
          rows, "median", np.median(allrel), "points", dev.filter_report)
    # measured on the H100: every view a reference with five sources, median relative error 0.16 % (per view 0.11-0.22 %),
    # 86-99 % of the pixels with a depth, 6.1 M points after the filter
    assert len(refs) == n
    assert np.median(allrel) < 0.005


def test_determinism_and_layouts():
    import torch
    imgs, cams, poses = _random_scene(2)
    refs, sources, ranges = [0, 2], [[1, 2, 3], [0, 1]], [(2.0, 12.0), (2.0, 12.0)]
    fprm = dict(max_reproj_error=2.0, max_depth_diff=0.05, min_consistent=1)
    a = api.depth_maps(imgs, cams, poses, refs, sources, ranges, n_depths=40, filter=fprm, **PRM)
    b = api.depth_maps(imgs, cams, poses, refs, sources, ranges, n_depths=40, filter=fprm, **PRM)
    for f in ("depth", "cost", "n_src", "n_consistent"):
        for x, y in zip(getattr(a, f), getattr(b, f)):
            assert x.tobytes() == y.tobytes(), f
    assert a.points.tobytes() == b.points.tobytes() and a.report == b.report and a.filter_report == b.filter_report
    # torch CUDA tensors in place, one of them a view with pitch > width
    big = [torch.zeros((im.shape[0], im.shape[1] + 37), dtype=torch.uint8, device="cuda") for im in imgs]
    for t, im in zip(big, imgs):
        t[:, 5:5 + im.shape[1]] = torch.from_numpy(im).cuda()
    views = [t[:, 5:5 + im.shape[1]] for t, im in zip(big, imgs)]
    assert views[0].stride(0) > views[0].shape[1]
    c = api.depth_maps(views, cams, poses, refs, sources, ranges, n_depths=40, filter=fprm, **PRM)
    dense = [torch.from_numpy(im).cuda() for im in imgs]
    d = api.depth_maps(dense, cams, poses, refs, sources, ranges, n_depths=40, filter=fprm, **PRM)
    for r in (c, d):
        for f in ("depth", "cost", "n_src", "n_consistent"):
            for x, y in zip(getattr(a, f), getattr(r, f)):
                assert x.tobytes() == y.tobytes(), f
        assert a.points.tobytes() == r.points.tobytes()
    # independence: a reference alone gives the same bytes as within a larger call
    e = api.depth_maps(imgs, cams, poses, refs[1:], sources[1:], ranges[1:], n_depths=40, **PRM)
    assert e.depth[0].tobytes() == a.depth[1].tobytes() and e.cost[0].tobytes() == a.cost[1].tobytes()


def test_no_refs_and_no_valid_source():
    imgs, cams, poses = _random_scene(3, n=3)
    z = api.depth_maps(imgs, cams, poses, [], [], [], filter=dict())
    assert z.depth == [] and z.report == {"candidates": 0, "depths": 0} and len(z.points) == 0
    # a source that sees nothing of the reference: every depth 0, every cost +inf
    far = list(poses)
    far[1] = (np.eye(3), np.array([0.0, 0.0, -100.0]))
    r = api.depth_maps(imgs, cams, far, [0], [[1]], [(2.0, 12.0)], n_depths=16, **PRM)
    assert (r.depth[0] == 0).all() and np.isinf(r.cost[0]).all() and (r.n_src[0] == 0).all() and r.report["depths"] == 0
    assert r.report["candidates"] == int(do.candidates(120, 160, 3).sum())
    # no source at all
    r = api.depth_maps(imgs, cams, poses, [0], [[]], [(2.0, 12.0)], n_depths=16, **PRM)
    assert (r.depth[0] == 0).all() and np.isinf(r.cost[0]).all()


SENT = 0xA5


def test_argument_errors():
    lib = api.load_library()
    imgs, cams, poses = _random_scene(4, h=40, w=50, n=3)
    bufs = api._DevBuffers(lib)
    try:
        c_img = (api.PsImage * 3)(*[api.PsImage(bufs.upload(im), 50, 50, 40) for im in imgs])
        cam = api._c_cameras(cams)
        rig = api._c_rigids(poses)
        outs = [bufs.alloc(2000 * 4) for _ in range(6)]
        nsrc = [bufs.alloc(2000) for _ in range(2)]
        pts = bufs.alloc(4000 * 24)
        fill = np.full(4000 * 24, SENT, np.uint8)

        def reset():
            for p in outs + nsrc + [pts]:
                lib.ps_host_to_dev(p, fill.ctypes.data, 2000 if p in nsrc else (4000 * 24 if p == pts else 8000))

        def untouched():
            for p in outs + nsrc:
                n = 2000 if p in nsrc else 8000
                assert (bufs.download(p, n, np.uint8) == SENT).all()
            assert (bufs.download(pts, 4000 * 24, np.uint8) == SENT).all()

        host = np.zeros(8000, np.uint8)

        def call(refs=(0, 1), start=(0, 2, 3), src=(1, 2, 0), rng=(2.0, 12.0, 2.0, 12.0), prm=None, img=c_img, cm=cam, rg=rig,
                 dep=None, cst=None, ns=None, nsets=3, nrefs=None):
            nrefs = len(refs) if nrefs is None else nrefs
            prm = prm or api._depth_params(n_depths=8, **PRM)
            r = np.asarray(list(refs) or [0], np.int32); s = np.asarray(start, np.int32); q = np.asarray(list(src) or [0], np.int32)
            g = np.asarray(rng, np.float32)
            dep = dep or outs[:2]; cst = cst or outs[2:4]; ns = ns or nsrc
            rep = api.PsDepthReport(-7, -7)
            rc = lib.ps_depth_maps(0, nsets, img, cm.ctypes.data if cm is not None else None, rg, nrefs, r.ctypes.data, g.ctypes.data,
                                   s.ctypes.data, q.ctypes.data, C.byref(prm), (C.c_void_p * 2)(*dep), (C.c_void_p * 2)(*cst),
                                   (C.c_void_p * 2)(*ns), C.byref(rep))
            return rc, rep

        def fcall(fprm=None, dep=None, nc=None, p=pts, refs=(0, 1), start=(0, 2, 3), src=(1, 2, 0), img=c_img, rg=rig):
            fprm = fprm or api._depth_filter_params()
            r = np.asarray(refs, np.int32); s = np.asarray(start, np.int32); q = np.asarray(src, np.int32)
            rep = api.PsDepthFilterReport(-7, -7)
            rc = lib.ps_depth_filter(0, 3, img, cam.ctypes.data, rg, len(refs), r.ctypes.data, s.ctypes.data, q.ctypes.data,
                                     (C.c_void_p * 2)(*(dep or outs[:2])), C.byref(fprm), (C.c_void_p * 2)(*(nc or nsrc)), p, C.byref(rep))
            return rc, rep

        reset()
        rc, rep = call()
        assert rc == 0 and rep.n_candidates == 2 * 44 * 34
        rc, rep = fcall(nc=[outs[4], outs[5]])
        assert rc == 0 and rep.n_tested >= 0
        bad_img = (api.PsImage * 3)(*c_img)
        bad_img[1] = api.PsImage(host.ctypes.data, 50, 50, 40)
        small = (api.PsImage * 3)(*c_img)
        small[2] = api.PsImage(c_img[2].data, 50, 6, 40)
        narrow = (api.PsImage * 3)(*c_img)
        narrow[0] = api.PsImage(c_img[0].data, 40, 50, 40)
        bad_cam = cam.copy(); bad_cam[1][0] = 0.0
        bad_rig = api._c_rigids([poses[0], (poses[1][0] * 1.001, poses[1][1]), poses[2]])
        cases = [dict(nsets=-1), dict(nrefs=-1), dict(refs=(0, 0)), dict(refs=(0, 3)), dict(src=(1, 0, 0)), dict(src=(1, 3, 0)),
                 dict(start=(1, 2, 3)), dict(start=(0, 3, 2)), dict(img=bad_img), dict(img=small), dict(img=narrow),
                 dict(rng=(2.0, 1.0, 2.0, 12.0)), dict(rng=(0.0, 12.0, 2.0, 12.0)), dict(rng=(2.0, float("inf"), 2.0, 12.0)),
                 dict(rng=(float("nan"), 12.0, 2.0, 12.0)), dict(cm=bad_cam), dict(rg=bad_rig),
                 dict(dep=[outs[0], host.ctypes.data]), dict(cst=[host.ctypes.data, outs[3]]), dict(ns=[nsrc[0], host.ctypes.data])]
        for kw in (dict(n_depths=1), dict(n_depths=1025), dict(radius=0), dict(radius=8), dict(top_k=0), dict(top_k=33),
                   dict(min_sources=0), dict(min_sources=33), dict(max_cost=0.0), dict(max_cost=2.5), dict(min_var=-1.0),
                   dict(min_var=float("nan"))):
            p = dict(n_depths=8, **PRM)
            p.update(kw)
            cases.append(dict(prm=api._depth_params(**p)))
        for kw in cases:
            reset()
            rc, rep = call(**kw)
            assert rc == PS_ERR_ARG and rep.n_candidates == -7 and rep.n_depths == -7, kw
            untouched()
        for kw in (dict(fprm=api._depth_filter_params(max_reproj_error=0.0)), dict(fprm=api._depth_filter_params(max_depth_diff=-1.0)),
                   dict(fprm=api._depth_filter_params(min_consistent=0)), dict(fprm=api._depth_filter_params(min_consistent=256)),
                   dict(fprm=api._depth_filter_params(max_reproj_error=float("inf"))), dict(dep=[outs[0], host.ctypes.data]),
                   dict(nc=[nsrc[0], host.ctypes.data]), dict(p=host.ctypes.data), dict(refs=(1, 1)), dict(src=(0, 2, 0)),
                   dict(img=bad_img), dict(rg=bad_rig)):
            reset()
            rc, rep = fcall(**kw)
            assert rc == PS_ERR_ARG and rep.n_tested == -7 and rep.n_points == -7, kw
            untouched()
        # n_refs = 0: valid, the report zero, nothing read
        rc, rep = call(refs=(), start=(0,), src=(), rng=(0.0, 0.0))
        assert rc == 0 and rep.n_candidates == 0 and rep.n_depths == 0
    finally:
        bufs.free()


def test_cpp_api_against_c_abi(rendered_views, tmp_path):
    """depth_check: popsift::depthMaps / filterDepthMaps against ps_depth_maps / ps_depth_filter on the six rendered views,
    identical bytes"""
    from popsift_b200 import build as B
    imgs, cams, poses, _ = rendered_views
    args = [B.DEPTH_CHECK, str(W), str(H), str(len(imgs))]
    for k, im in enumerate(imgs):
        f = tmp_path / ("v%d.raw" % k)
        im.tofile(f)
        args.append(str(f))
    for cam, (R, t) in zip(cams, poses):
        # the scene's depths lie within 2.2 .. 11 in every view (test_pose's planes)
        args += ["%.9g" % v for v in cam] + ["%.17g" % v for v in np.r_[R.ravel(), t]] + ["2.0", "12.0"]
    out = subprocess.run(args, capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    assert int(out.stdout.split()[1]) > 0.5 * 6 * (W - 6) * (H - 6)
