"""ps_tsdf_integrate and ps_tsdf_mesh on the GPU against tests/mesh_oracle.py (identical bytes), at every work-split
boundary of the kernels, against the planes of test_pose's rendered scene, and the API's edges: determinism, split
calls, overflow and count-only calls, argument errors with fenced outputs, empty calls, and the C++ API against the C
ABI."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import mesh_oracle as mo                                   # noqa: E402
from popsift_b200 import api                               # noqa: E402
from test_depth import _rendered                           # noqa: E402
from test_pose import PLANES                               # noqa: E402

pytestmark = pytest.mark.gpu

F32 = np.float32
PS_ERR_ARG, PS_ERR_OVERFLOW = -1, -5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _const(path, name):
    """an integer constant of a kernel source: `name = <int expression of earlier constants>`"""
    src = open(os.path.join(ROOT, "popsift_b200", "csrc", path)).read()
    env = {}
    for m in re.finditer(r"constexpr\s+(?:long long|int)\s+(.*?);", src):
        for part in re.split(r",\s*(?=k\w+\s*=)", m.group(1)):
            k, v = part.split("=", 1)
            env[k.strip()] = eval(re.sub(r"\(long long\)", "", v).replace("/", "//"), {}, dict(env))
    return env[name]


K_SCAN_CHUNK = _const("k_scan.h", "kScanChunk")
K_RADIX_TILE = _const("k_scan.h", "kRadixTile")
K_CELL_BLOCK = _const("k_mesh.cu", "kCellBlock")
K_VIEW_CHUNK = _const("k_mesh.cu", "kViewChunk")


def _rot(rng, deg):
    a = rng.normal(size=3)
    a /= np.linalg.norm(a)
    th = np.radians(deg)
    S = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.cos(th) * np.eye(3) + np.sin(th) * S + (1 - np.cos(th)) * np.outer(a, a)


def _random_views(seed, n, w=64, h=48, centre=(0.0, 0.0, 0.0), dist=2.0):
    """n cameras on a sphere around `centre` looking at it, with smooth random depth maps around the centre's depth,
    10 % unknown pixels, random grey levels and random consistency masks"""
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(seed)
    imgs, cams, poses, depths, masks = [], [], [], [], []
    c = np.asarray(centre, np.float64)
    for _ in range(n):
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        C0 = c - dist * d                                   # camera centre, looking along d
        z = d
        x = np.cross([0.0, 1.0, 0.0] if abs(d[1]) < 0.9 else [1.0, 0.0, 0.0], z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = _rot(rng, 2.0) @ np.stack([x, y, z])
        t = -R @ C0
        cam = np.array([rng.uniform(0.8, 1.2) * w, rng.uniform(0.8, 1.2) * w, w / 2 + rng.normal(), h / 2 + rng.normal()], F32)
        D = (dist + gaussian_filter(rng.normal(size=(h, w)), 3.0) * 2.0).astype(F32)
        D[rng.random((h, w)) < 0.1] = 0.0
        imgs.append(rng.integers(0, 256, (h, w)).astype(np.uint8))
        cams.append(cam)
        poses.append((R, t))
        depths.append(D)
        masks.append(rng.integers(0, 4, (h, w)).astype(np.uint8))
    return imgs, cams, poses, depths, masks


def _compare_volumes(got, ref, tag):
    """identical bytes; a differing voxel is printed (it would be a rounding-boundary case of the projection)"""
    for name, a, b in zip(("tsdf", "weight", "grey"), got, ref):
        bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
        for g in bad[:10]:
            print(tag, name, "voxel", np.unravel_index(g, a.shape), "device", a.ravel()[g], "oracle", b.ravel()[g])
        assert len(bad) == 0, (tag, name, len(bad))


def _integrate_both(views, origin, voxel, shape, trunc, min_consistent=0, masks=True):
    imgs, cams, poses, depths, mk = views
    vol = api.TsdfVolume(origin, voxel, shape)
    rep = vol.integrate(imgs, cams, poses, depths, masks=mk if masks else None, trunc=trunc, min_consistent=min_consistent)
    got = vol.download()
    vol.free()
    nx, ny, nz = shape
    zero = np.zeros((nz, ny, nx), F32)
    ref, (n_upd, touched) = mo.integrate((zero, zero, zero), origin, voxel, imgs, cams, poses, depths, mk if masks else None, trunc=trunc,
                                         min_consistent=min_consistent)
    assert rep == {"updates": n_upd, "touched": touched}
    return got, ref, rep


@pytest.mark.parametrize("scene", ["random", "random_masked", "many_views", "rendered160"])
def test_integration_against_oracle(scene):
    if scene == "rendered160":
        imgs, cams, poses, truth = _rendered(0.125)
        views = (imgs, cams, poses, [D.astype(F32) for D in truth], None)
        origin, voxel, shape, trunc, mc = (-3.0, -2.2, 1.5), 0.1, (64, 48, 100), 0.3, 0
    elif scene == "many_views":
        # more views than one shared-memory chunk, each seeing part of the volume
        views = _random_views(7, K_VIEW_CHUNK + 6, w=24, h=18, dist=1.2)
        origin, voxel, shape, trunc, mc = (-0.6, -0.5, -0.55), 0.02, (61, 50, 55), 0.05, 0
    else:
        views = _random_views(1 if scene == "random" else 2, 5)
        origin, voxel, shape, trunc, mc = (-0.8, -0.7, -0.75), 0.025, (67, 57, 61), 0.08, (2 if scene == "random_masked" else 0)
    got, ref, rep = _integrate_both(views, origin, voxel, shape, trunc, min_consistent=mc, masks=views[4] is not None)
    print(scene, rep, "touched fraction", rep["touched"] / np.prod(shape))
    assert rep["touched"] > 0.05 * np.prod(shape)
    _compare_volumes(got, ref, scene)


@pytest.mark.parametrize("shape", [(2, 2, 2), (32, 4, 4), (64, 8, 12), (33, 5, 7), (97, 13, 6)])
def test_integration_and_extraction_at_block_shapes(shape):
    """whole and partial integration blocks (32 x 4 x 4), one classification block and several"""
    views = _random_views(11, 3, dist=1.5)
    nx, ny, nz = shape
    voxel = 1.2 / max(shape)
    origin = (-voxel * (nx - 1) / 2, -voxel * (ny - 1) / 2, -voxel * (nz - 1) / 2)
    got, ref, _ = _integrate_both(views, origin, voxel, shape, 4 * voxel)
    _compare_volumes(got, ref, shape)
    _compare_mesh(got, origin, voxel, 1.0, str(shape))


def _upload(vol, arrays):
    lib = vol._lib
    for p, a in zip(vol._ptrs, arrays):
        a = np.ascontiguousarray(a, F32)
        assert lib.ps_host_to_dev(p, a.ctypes.data, a.nbytes) == 0


def _compare_mesh(arrays, origin, voxel, min_weight, tag):
    T = arrays[0]
    nz, ny, nx = T.shape
    vol = api.TsdfVolume(origin, voxel, (nx, ny, nz))
    _upload(vol, arrays)
    m = vol.mesh(min_weight=min_weight)
    vol.free()
    V, tris, rep, _ = mo.mesh(arrays, origin, voxel, min_weight)
    assert m.report == {"cells": rep[0], "vertices": rep[1], "triangles": rep[2]}, tag
    got = np.stack([m.vertices["X"][:, 0], m.vertices["X"][:, 1], m.vertices["X"][:, 2], m.vertices["grey"]], 1).astype(F32)
    assert got.tobytes() == V.tobytes(), tag
    assert np.array_equal(m.triangles, tris), tag
    return m


def _sphere_volume(n, seed):
    rng = np.random.default_rng(seed)
    o, h = (-1.1, -1.0, -1.2), 2.3 / (n - 1)
    X, Y, Z = mo.grid_points(o, h, (n, n - 3, n + 2))
    T = (np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.85 + 0.05 * np.sin(5 * X)).astype(F32)
    W = rng.choice(np.array([0.0, 1.0, 2.0, 5.0], F32), T.shape, p=[0.02, 0.1, 0.3, 0.58])
    G = rng.uniform(0, 255, T.shape).astype(F32)
    return (T, W, G), o, h


def test_extraction_against_oracle():
    arrays, o, h = _sphere_volume(70, 1)
    m = _compare_mesh(arrays, o, h, 1.5, "sphere")
    assert m.report["triangles"] > 10000
    # the same volume with full weights: closed, genus 0
    full = (arrays[0], np.ones_like(arrays[1]), arrays[2])
    m = _compare_mesh(full, o, h, 1.0, "sphere full")
    boundary, dup, chi = mo.topology(m.triangles, len(m.vertices))
    assert len(boundary) == 0 and dup == 0 and chi == 2


def _line_volume(target, seed):
    """a volume of nx x 2 x 2 grid points whose active cells list exactly `target` edge entries (searched over seeds)"""
    for s in range(seed, seed + 200):
        rng = np.random.default_rng(s)
        T = rng.choice(np.array([-1.0, 1.0], F32), (2, 2, 2048)) * rng.uniform(0.1, 1.0, (2, 2, 2048)).astype(F32)
        g, mask = mo.active_cells(T, np.ones_like(T), 1.0)
        nk, _ = mo.cell_counts(mask)
        cum = np.cumsum(nk)
        hit = np.flatnonzero(cum == target)
        if len(hit):
            nx = int(g[hit[0]]) + 2                         # keeps the cells up to and including that one
            T = np.ascontiguousarray(T[:, :, :nx])
            return T, np.ones_like(T), np.full(T.shape, 7.0, F32)
    raise AssertionError("no volume found")


@pytest.mark.parametrize("target", [K_SCAN_CHUNK - 1, K_SCAN_CHUNK, K_SCAN_CHUNK + 1, K_RADIX_TILE - 1, K_RADIX_TILE + 1])
def test_extraction_edge_entries_at_boundaries(target):
    arrays = _line_volume(target, 3)
    g, mask = mo.active_cells(arrays[0], arrays[1], 1.0)
    assert mo.cell_counts(mask)[0].sum() == target
    _compare_mesh(arrays, (0.1, 0.2, 0.3), 0.01, 1.0, "entries %d" % target)


@pytest.mark.parametrize("cells", [K_SCAN_CHUNK - 1, K_SCAN_CHUNK, K_SCAN_CHUNK + 1, K_CELL_BLOCK + 1])
def test_extraction_active_cells_at_boundaries(cells):
    """a plane through a nx x ny x 2 volume: every cell active"""
    a, b = {4095: (63, 65), 4096: (64, 64), 4097: (17, 241), 2049: (3, 683)}[cells]
    T = np.empty((2, b + 1, a + 1), F32)
    T[0], T[1] = -0.3, 0.6
    arrays = (T, np.ones_like(T), np.full(T.shape, 3.0, F32))
    assert len(mo.active_cells(T, arrays[1], 1.0)[0]) == cells
    _compare_mesh(arrays, (0.0, 0.0, 0.0), 0.1, 1.0, "cells %d" % cells)


def test_split_calls_determinism_and_device_arrays():
    import torch
    imgs, cams, poses, depths, masks = _random_views(5, 6)
    origin, voxel, shape = (-0.8, -0.7, -0.75), 0.03, (56, 48, 50)
    a = api.TsdfVolume(origin, voxel, shape)
    ra = a.integrate(imgs, cams, poses, depths, masks, trunc=0.1, min_consistent=1)
    b = api.TsdfVolume(origin, voxel, shape)
    rb1 = b.integrate(imgs[:2], cams[:2], poses[:2], depths[:2], masks[:2], trunc=0.1, min_consistent=1)
    # the rest from torch CUDA tensors, in place
    dev = lambda xs: [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in xs]     # noqa: E731
    rb2 = b.integrate(dev(imgs[2:]), cams[2:], poses[2:], dev(depths[2:]), dev(masks[2:]), trunc=0.1, min_consistent=1)
    for x, y in zip(a.download(), b.download()):
        assert x.tobytes() == y.tobytes()
    assert ra["updates"] == rb1["updates"] + rb2["updates"]
    m1, m2 = a.mesh(), a.mesh()
    assert m1.vertices.tobytes() == m2.vertices.tobytes() and m1.triangles.tobytes() == m2.triangles.tobytes() and m1.report == m2.report
    assert m1.report["triangles"] > 0
    # a second identical integration gives identical bytes too
    c = api.TsdfVolume(origin, voxel, shape)
    c.integrate(imgs, cams, poses, depths, masks, trunc=0.1, min_consistent=1)
    for x, y in zip(a.download(), c.download()):
        assert x.tobytes() == y.tobytes()
    # clear resets
    c.clear()
    assert all((x == 0).all() for x in c.download())
    for v in (a, b, c):
        v.free()


SENT = 0xA5


def test_overflow_count_only_and_guards():
    lib = api.load_library()
    arrays, o, h = _sphere_volume(30, 2)
    nz, ny, nx = arrays[0].shape
    vol = api.TsdfVolume(o, h, (nx, ny, nz))
    _upload(vol, arrays)
    cv = vol.c_volume()
    prm = api.PsMeshParams(1.0, 0)
    rep = api.PsMeshReport(-7, -7, -7)
    assert lib.ps_tsdf_mesh(0, C.byref(cv), C.byref(prm), 0, 0, None, None, C.byref(rep)) == PS_ERR_OVERFLOW
    nv, nt = int(rep.n_vertices), int(rep.n_triangles)
    assert nv > 0 and nt > 0 and rep.n_cells > 0
    bufs = api._DevBuffers(lib)
    try:
        G = 256
        pv, pt = bufs.alloc(nv * 16 + 2 * G), bufs.alloc(nt * 12 + 2 * G)
        fill_v, fill_t = np.full(nv * 16 + 2 * G, SENT, np.uint8), np.full(nt * 12 + 2 * G, SENT, np.uint8)

        def reset():
            lib.ps_host_to_dev(pv, fill_v.ctypes.data, fill_v.nbytes)
            lib.ps_host_to_dev(pt, fill_t.ctypes.data, fill_t.nbytes)

        def untouched():
            assert (bufs.download(pv, fill_v.nbytes, np.uint8) == SENT).all() and (bufs.download(pt, fill_t.nbytes, np.uint8) == SENT).all()

        for cap in ((nv - 1, nt), (nv, nt - 1), (0, nt)):
            reset()
            r = api.PsMeshReport(-7, -7, -7)
            rc = lib.ps_tsdf_mesh(0, C.byref(cv), C.byref(prm), cap[0], cap[1], pv + G, pt + G, C.byref(r))
            assert rc == PS_ERR_OVERFLOW and (r.n_cells, r.n_vertices, r.n_triangles) == (rep.n_cells, nv, nt), cap
            untouched()
        reset()
        r = api.PsMeshReport(-7, -7, -7)
        assert lib.ps_tsdf_mesh(0, C.byref(cv), C.byref(prm), nv, nt, pv + G, pt + G, C.byref(r)) == 0
        bv, bt = bufs.download(pv, fill_v.nbytes, np.uint8), bufs.download(pt, fill_t.nbytes, np.uint8)
        assert (bv[:G] == SENT).all() and (bv[G + nv * 16:] == SENT).all() and (bt[:G] == SENT).all() and (bt[G + nt * 12:] == SENT).all()
        m = vol.mesh()
        assert bv[G:G + nv * 16].tobytes() == m.vertices.tobytes() and bt[G:G + nt * 12].tobytes() == m.triangles.tobytes()
    finally:
        bufs.free()
        vol.free()


def test_empty_calls():
    vol = api.TsdfVolume((0.0, 0.0, 0.0), 0.1, (20, 10, 5))
    assert vol.integrate([], [], [], []) == {"updates": 0, "touched": 0}
    assert all((x == 0).all() for x in vol.download())
    # weights 0 everywhere: no cell is meshed
    m = vol.mesh()
    assert len(m.vertices) == 0 and m.triangles.shape == (0, 3) and m.report == {"cells": 0, "vertices": 0, "triangles": 0}
    # weights 1 and T = 0 everywhere: every corner outside, nothing to mesh
    _upload(vol, (np.zeros((5, 10, 20), F32), np.ones((5, 10, 20), F32), np.zeros((5, 10, 20), F32)))
    assert vol.mesh().report == {"cells": 0, "vertices": 0, "triangles": 0}
    # a view that sees nothing of the volume
    imgs, cams, poses, depths, _ = _random_views(3, 1)
    far = [(poses[0][0], poses[0][1] + np.array([0.0, 0.0, -100.0]))]
    before = vol.download()
    assert vol.integrate(imgs, cams, far, depths, trunc=0.1)["updates"] == 0
    for x, y in zip(before, vol.download()):
        assert x.tobytes() == y.tobytes()
    vol.free()


def test_argument_errors():
    lib = api.load_library()
    imgs, cams, poses, depths, masks = _random_views(4, 2)
    vol = api.TsdfVolume((0.0, 0.0, 0.0), 0.05, (16, 12, 10))
    n = 16 * 12 * 10
    fence = np.full(n * 4, SENT, np.uint8)
    bufs = api._DevBuffers(lib)
    try:
        c_img = (api.PsImage * 2)(*[api.PsImage(bufs.upload(im), 64, 64, 48) for im in imgs])
        d_dep = [bufs.upload(d) for d in depths]
        d_msk = [bufs.upload(m) for m in masks]
        cam = api._c_cameras(cams)
        rig = api._c_rigids(poses)
        host = np.zeros(64 * 48 * 4, np.uint8)

        def reset():
            for p in vol._ptrs:
                lib.ps_host_to_dev(p, fence.ctypes.data, fence.nbytes)

        def untouched():
            for p in vol._ptrs:
                assert (bufs.download(p, fence.nbytes, np.uint8) == SENT).all()

        def call(nv=2, img=c_img, cm=cam, rg=rig, dep=None, msk=None, prm=None, cv=None, null_msk=False):
            dep = dep or d_dep
            msk = msk or d_msk
            prm = prm or api.PsTsdfParams(0.1, 1)
            cv = cv or vol.c_volume()
            rep = api.PsTsdfReport(-7, -7)
            rc = lib.ps_tsdf_integrate(0, nv, img, cm.ctypes.data, rg, (C.c_void_p * 2)(*dep), None if null_msk else (C.c_void_p * 2)(*msk),
                                       C.byref(prm), C.byref(cv), C.byref(rep))
            return rc, rep

        def vol_with(**kw):
            cv = vol.c_volume()
            for k, v in kw.items():
                if k == "origin":
                    cv.origin = (C.c_double * 3)(*v)
                else:
                    setattr(cv, k, v)
            return cv

        reset()
        rc, rep = call()
        assert rc == 0 and rep.n_updates >= 0
        bad_img = (api.PsImage * 2)(*c_img)
        bad_img[1] = api.PsImage(host.ctypes.data, 64, 64, 48)
        narrow = (api.PsImage * 2)(*c_img)
        narrow[0] = api.PsImage(c_img[0].data, 40, 64, 48)
        bad_cam = cam.copy(); bad_cam[1][0] = 0.0
        bad_rig = api._c_rigids([poses[0], (poses[1][0] * 1.001, poses[1][1])])
        cases = [dict(nv=-1), dict(img=bad_img), dict(img=narrow), dict(cm=bad_cam), dict(rg=bad_rig), dict(dep=[d_dep[0], host.ctypes.data]),
                 dict(msk=[d_msk[0], host.ctypes.data]), dict(null_msk=True), dict(prm=api.PsTsdfParams(0.0, 0)),
                 dict(prm=api.PsTsdfParams(float("inf"), 0)), dict(prm=api.PsTsdfParams(0.1, -1)), dict(prm=api.PsTsdfParams(0.1, 256)),
                 dict(cv=vol_with(voxel=0.0)), dict(cv=vol_with(voxel=float("nan"))), dict(cv=vol_with(origin=(0.0, float("inf"), 0.0))),
                 dict(cv=vol_with(nx=1)), dict(cv=vol_with(nz=2049)), dict(cv=vol_with(nx=2048, ny=2048, nz=512)),
                 dict(cv=vol_with(tsdf=host.ctypes.data)), dict(cv=vol_with(grey=vol._ptrs[1]))]
        for kw in cases:
            reset()
            rc, rep = call(**kw)
            assert rc == PS_ERR_ARG and rep.n_updates == -7 and rep.n_voxels_touched == -7, kw
            untouched()
        # n_views = 0: valid, the volume untouched
        reset()
        rc, rep = call(nv=0)
        assert rc == 0 and rep.n_updates == 0
        untouched()
        # mesh: fenced outputs
        pv, pt = bufs.alloc(4096), bufs.alloc(4096)
        f4 = np.full(4096, SENT, np.uint8)
        for kw in (dict(cv=vol_with(voxel=-1.0)), dict(cv=vol_with(weight=host.ctypes.data)), dict(mw=0.0), dict(mw=float("nan")),
                   dict(cap=(-1, 10)), dict(cap=(10, -1)), dict(outs=(host.ctypes.data, pt)), dict(outs=(pv, None))):
            lib.ps_host_to_dev(pv, f4.ctypes.data, 4096)
            lib.ps_host_to_dev(pt, f4.ctypes.data, 4096)
            r = api.PsMeshReport(-7, -7, -7)
            cv = kw.get("cv") or vol.c_volume()
            cap = kw.get("cap", (100, 100))
            outs = kw.get("outs", (pv, pt))
            rc = lib.ps_tsdf_mesh(0, C.byref(cv), C.byref(api.PsMeshParams(kw.get("mw", 1.0), 0)), cap[0], cap[1], outs[0], outs[1], C.byref(r))
            assert rc == PS_ERR_ARG and (r.n_cells, r.n_vertices, r.n_triangles) == (-7, -7, -7), kw
            assert (bufs.download(pv, 4096, np.uint8) == SENT).all() and (bufs.download(pt, 4096, np.uint8) == SENT).all()
        assert lib.ps_volume_clear(0, C.byref(vol_with(ny=1))) == PS_ERR_ARG
    finally:
        bufs.free()
        vol.free()


def _plane_distance(X):
    d = []
    for n, dist in PLANES:
        n = np.asarray(n, np.float64)
        d.append(np.abs(X @ n - dist) / np.linalg.norm(n))
    return np.min(d, 0)


def test_against_truth_640():
    """the six rendered views at 640 x 480: depth_maps with the filter, then TsdfVolume with the filter's masks over the
    filtered points' bounds; every vertex's distance to the nearest of the scene's planes"""
    from test_depth import _true_range
    imgs, cams, poses, truth = _rendered(0.5)
    refs = list(range(6))
    sources = [[s for s in refs if s != r] for r in refs]
    ranges = [_true_range(truth[r]) for r in refs]
    dm = api.depth_maps(imgs, cams, poses, refs, sources, ranges, n_depths=128, radius=3, top_k=3, max_cost=0.5,
                        filter=dict(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2))
    P = dm.points["X"].astype(np.float64)
    lo, hi = np.percentile(P, 0.5, 0), np.percentile(P, 99.5, 0)
    voxel = float((hi - lo).max() / 255)
    lo, hi = lo - 4 * voxel, hi + 4 * voxel
    shape = tuple(int(v) for v in np.ceil((hi - lo) / voxel) + 1)
    vol = api.TsdfVolume(lo, voxel, shape)
    rep = vol.integrate(imgs, cams, poses, dm.depth, masks=dm.n_consistent, trunc=3 * voxel, min_consistent=2)
    m = vol.mesh(min_weight=2.0)
    vol.free()
    d = _plane_distance(m.vertices["X"].astype(np.float64)) / voxel
    med, p90 = float(np.median(d)), float(np.percentile(d, 90))
    boundary, dup, _ = mo.topology(m.triangles, len(m.vertices))
    print("640 x 480: volume", shape, "voxel", voxel, "integration", rep, "mesh", m.report, "distance to the planes in voxels: median",
          med, "p90", p90, "p99", float(np.percentile(d, 99)), "boundary edges", len(boundary), "duplicated directed edges", dup)
    # measured on the H100: a 253 x 218 x 264 volume at 0.0234, 845 k triangles, distance to the planes 0.19 voxel at
    # the median, 0.57 at p90 and 1.15 at p99; the surface is open where the views' coverage ends
    assert dup == 0 and m.report["triangles"] > 500000
    assert med < 0.25 and p90 < 0.75


def test_cpp_api_against_c_abi(tmp_path):
    """mesh_check: popsift::DeviceVolume / integrateDepthMaps / extractMesh against the C ABI on random views, identical
    bytes"""
    from popsift_b200 import build as B
    imgs, cams, poses, depths, _ = _random_views(9, 4)
    h, w = imgs[0].shape
    args = [B.MESH_CHECK, str(w), str(h), str(len(imgs)), "0.08", "1.0", "0.025", "64", "56", "60", "-0.8", "-0.7", "-0.75"]
    for k, (im, D) in enumerate(zip(imgs, depths)):
        fi, fd = tmp_path / ("v%d.raw" % k), tmp_path / ("d%d.raw" % k)
        im.tofile(fi)
        D.astype(F32).tofile(fd)
        args += [str(fi), str(fd)]
    for cam, (R, t) in zip(cams, poses):
        args += ["%.9g" % v for v in cam] + ["%.17g" % v for v in np.r_[R.ravel(), t]]
    out = subprocess.run(args, capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    assert int(out.stdout.split()[3]) > 0
