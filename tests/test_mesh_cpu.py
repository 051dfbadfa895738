"""The mesh contracts (tests/mesh_oracle.py) on their own: the Kuhn split and its triangle table, marching tetrahedra on
analytic signed distance fields, holes in the weights, integration on planted depth maps; the kernels' math built for
the host (tests/cpp/mesh_math_check.cpp) against the oracle; the header's exports and layouts.  No GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import mesh_oracle as mo                  # noqa: E402

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the split and the table ------------------------------------------------------------------------------------------

def test_kuhn_tetrahedra():
    tets = mo.kuhn_tets()
    vols = []
    for v in tets:
        P = [mo._corner(int(c)) for c in v]
        vols.append(np.linalg.det(np.stack([P[1] - P[0], P[2] - P[0], P[3] - P[0]])) / 6.0)
        # every edge joins componentwise-ordered corners: a lower corner and a 0/1 direction
        for a in range(4):
            for b in range(a + 1, 4):
                lo, hi = sorted((int(v[a]), int(v[b])), key=lambda c: bin(c).count("1"))
                assert lo & hi == lo
    assert np.all(np.array(vols) > 0) and abs(sum(vols) - 1.0) < 1e-12
    # the 19 edges of the split are those of the tetrahedra
    edges = {mo.edge_code(int(v[a]), int(v[b])) for v in tets for a in range(4) for b in range(a + 1, 4)}
    assert sorted(edges) == sorted((a << 3) | d for a, d in mo.cell_edges()) and len(edges) == 19


def test_face_diagonals_agree_between_neighbours():
    """each face of a cell is split along its lowest-to-highest diagonal, so the two cells sharing it agree"""
    tets = mo.kuhn_tets()
    diag = set()
    for v in tets:
        for a in range(4):
            for b in range(a + 1, 4):
                e = mo.edge_code(int(v[a]), int(v[b]))
                if bin(e & 7).count("1") == 2:
                    diag.add(e)
    for axis in range(3):
        bit = 1 << axis
        for side in (0, 1):
            # face diagonals of the face x_axis = side, in the cell's corner coordinates
            on = {e for e in diag if not (e & 7) & bit and ((e >> 3) & bit) == side * bit}
            assert len(on) == 1
            e = on.pop()
            lo, d = e >> 3, e & 7
            assert lo & ~bit == 0           # from the face's lowest corner to its highest
            if side == 1:
                # the neighbour's face at x_axis = 0 is this face shifted by one cell
                other = {f for f in diag if not (f & 7) & bit and ((f >> 3) & bit) == 0}
                assert other == {((lo & ~bit) << 3) | d}


def _mesh_math(requests):
    from popsift_b200 import build as B
    B.build()
    out = subprocess.run([B.MESH_MATH_CHECK], input="\n".join(requests) + "\n", capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return [line.split()[1:] for line in out.stdout.splitlines()]


def test_kernel_table_equals_oracle():
    (row,) = _mesh_math(["k"])
    vals = np.array([int(v) for v in row])
    count, tri = mo.triangle_table()
    tets = mo.kuhn_tets()
    assert np.array_equal(vals[:24].reshape(6, 4), tets)
    assert all(np.array_equal(vals[24:40], count[t]) for t in range(6))
    got = vals[40:40 + 576].reshape(6, 16, 2, 3)
    for t in range(6):
        for c in range(16):
            assert np.array_equal(got[t, c, :count[t, c]], tri[t, c, :count[t, c]]), (t, c)
    assert [int(v) for v in vals[616:]] == [(a << 3) | d for a, d in mo.cell_edges()]
    # the per-cell counts of every mask
    rows = _mesh_math(["c %d" % m for m in range(256)])
    nk, nt = mo.cell_counts(np.arange(256))
    assert [int(r[0]) for r in rows] == nk.tolist() and [int(r[1]) for r in rows] == nt.tolist()


# ---- analytic fields -------------------------------------------------------------------------------------------------

def _field(kind, n=24):
    o = (-1.2, -1.2, -1.2)
    h = 2.4 / (n - 1)
    X, Y, Z = mo.grid_points(o, h, (n, n, n))
    if kind == "sphere":
        d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.9
        vol = 4.0 / 3.0 * np.pi * 0.9 ** 3
        dist = lambda P: np.abs(np.linalg.norm(P, axis=1) - 0.9)          # noqa: E731
    elif kind == "torus":
        q = np.sqrt(X ** 2 + Y ** 2) - 0.7
        d = np.sqrt(q ** 2 + Z ** 2) - 0.25
        vol = 2 * np.pi ** 2 * 0.7 * 0.25 ** 2
        dist = lambda P: np.abs(np.hypot(np.hypot(P[:, 0], P[:, 1]) - 0.7, P[:, 2]) - 0.25)   # noqa: E731
    elif kind == "boxes":
        def box(c, b):
            q = np.abs(np.stack([X - c[0], Y - c[1], Z - c[2]])) - np.asarray(b)[:, None, None, None]
            return np.linalg.norm(np.maximum(q, 0), axis=0) + np.minimum(q.max(0), 0)
        # two boxes touching along the face x = 0.05 (off the grid planes)
        d = np.minimum(box((-0.45, 0.0, 0.0), (0.5, 0.6, 0.5)), box((0.45, 0.1, 0.05), (0.4, 0.5, 0.6)))
        vol = None
        dist = None
    else:   # a slab one cell thick: grid points at z = 0 inside, z = +-h outside
        q = np.abs(np.stack([X, Y, Z])) - np.array([0.8, 0.7, h / 2])[:, None, None, None]
        d = np.linalg.norm(np.maximum(q, 0), axis=0) + np.minimum(q.max(0), 0)
        vol = None
        dist = None
    T = d.astype(F32)
    return (T, np.ones_like(T), np.zeros_like(T)), o, h, vol, dist


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("boxes", 2), ("slab", 2)])
def test_analytic_fields(kind, chi):
    vol, o, h, true_vol, dist = _field(kind)
    V, tris, rep, keys = mo.mesh(vol, o, h)
    boundary, dup, euler = mo.topology(tris, len(V))
    assert len(boundary) == 0 and dup == 0, kind            # closed, every directed edge paired with its reverse
    assert euler == chi, (kind, euler)
    assert rep[1] == len(np.unique(tris)) == len(V)         # vertices: exactly the referenced edges
    assert np.all(np.diff(keys) > 0)
    sv = mo.signed_volume(V[:, :3], tris)
    assert sv > 0
    if true_vol is not None:
        # linear interpolation along edges of an exact distance field: within a fifth of a voxel (0.15 on the torus, whose
        # tube radius is 2.4 voxels), enclosed volume within 4 %
        assert dist(V[:, :3].astype(np.float64)).max() < 0.2 * h, kind
        assert abs(sv / true_vol - 1) < 0.04, (kind, sv / true_vol)
    print(kind, rep, "chi", euler, "volume", sv, true_vol)


def test_weight_hole_gives_boundary_only_there():
    vol, o, h, _, _ = _field("sphere")
    T, W, G = vol
    W = W.copy()
    W[:, :, 18:] = 0.5                                     # grid points x >= 18 unobserved at min_weight 1
    V, tris, rep, _ = mo.mesh((T, W, G), o, h, min_weight=1.0)
    boundary, dup, _ = mo.topology(tris, len(V))
    assert dup == 0 and len(boundary) > 0
    # every boundary edge lies on the last meshed cell layer: both its vertices at x <= 18 h from the origin, with
    # cells up to x index 17 meshed, so on the face x = 17 .. 18 region
    x = V[np.unique(boundary.ravel()), 0] - o[0]
    assert np.all(x >= 17 * h - 1e-6) and np.all(x <= 18 * h + 1e-6)
    # and nothing was meshed beyond
    assert (V[:, 0] - o[0]).max() <= 18 * h + 1e-6


# ---- integration ----------------------------------------------------------------------------------------------------

def _plane_view(w=40, h=30, z=2.0):
    """a camera at the origin looking down +z at a plane z = const"""
    cam = np.array([30.0, 30.0, (w - 1) / 2, (h - 1) / 2], np.float32)
    depth = np.full((h, w), z, np.float32)
    grey = (np.arange(w * h) % 251).reshape(h, w).astype(np.uint8)
    return cam, (np.eye(3), np.zeros(3)), depth, grey


def test_integration_rules():
    cam, pose, depth, grey = _plane_view()
    depth[0:10, 0:10] = 0.0                                 # unknown pixels
    ncons = np.full(depth.shape, 3, np.uint8)
    ncons[20:, 30:] = 1                                     # masked at min_consistent 2
    origin, voxel, shape = (-0.3, -0.2, 1.5), 0.05, (13, 9, 21)
    nx, ny, nz = shape
    zero = np.zeros((nz, ny, nx), F32)
    trunc = 0.2
    (T, W, G), (n_upd, touched) = mo.integrate((zero, zero, zero), origin, voxel, [grey], [cam], [pose], [depth], [ncons], trunc=trunc,
                                               min_consistent=2)
    X, Y, Z = mo.grid_points(origin, voxel, shape)
    u = 30.0 * X / Z + cam[2]
    v = 30.0 * Y / Z + cam[3]
    qx, qy = np.floor(u + 0.5).astype(int), np.floor(v + 0.5).astype(int)
    inside = (qx >= 0) & (qx < 40) & (qy >= 0) & (qy < 30)
    known = inside & (depth[np.clip(qy, 0, 29), np.clip(qx, 0, 39)] > 0) & (ncons[np.clip(qy, 0, 29), np.clip(qx, 0, 39)] >= 2)
    sdf = 2.0 - Z
    tr = np.float64(F32(trunc))                             # trunc is a float of the contract
    upd = known & (sdf >= -tr)
    assert np.array_equal(W == 1, upd) and np.all(W[~upd] == 0) and np.all(T[~upd] == 0)
    assert n_upd == touched == int(upd.sum())
    # tau by the formula, free space at 1
    assert np.array_equal(T[upd], np.minimum(1.0, sdf[upd] / np.float64(F32(trunc))).astype(F32))
    assert np.all(T[upd & (sdf > tr)] == 1.0)
    assert np.any(T[upd] < 0) and np.any((T[upd] > 0) & (T[upd] < 1))
    # behind -trunc: untouched
    assert not np.any(upd & (sdf < -tr)) and np.any(known & (sdf < -tr))
    # the grey level of the pixel, the unknown pixels and the mask honoured
    assert np.array_equal(G[upd], grey[qy[upd], qx[upd]].astype(F32))
    assert not np.any(upd & inside & (qx < 10) & (qy < 10)) and not np.any(upd & inside & (qx >= 30) & (qy >= 20))


def test_split_calls_equal_one_call():
    rng = np.random.default_rng(3)
    views = []
    for k in range(5):
        cam, _, depth, grey = _plane_view(z=1.8 + 0.1 * k)
        depth *= F32(1) + rng.normal(0, 0.02, depth.shape).astype(F32)
        depth[rng.random(depth.shape) < 0.1] = 0
        th = np.radians(rng.normal(0, 3, 3))
        Rx = np.array([[1, 0, 0], [0, np.cos(th[0]), -np.sin(th[0])], [0, np.sin(th[0]), np.cos(th[0])]])
        Ry = np.array([[np.cos(th[1]), 0, np.sin(th[1])], [0, 1, 0], [-np.sin(th[1]), 0, np.cos(th[1])]])
        views.append((cam, (Rx @ Ry, rng.normal(0, 0.05, 3)), depth, (grey + k).astype(np.uint8)))
    origin, voxel, shape = (-0.3, -0.2, 1.5), 0.04, (16, 11, 14)
    nx, ny, nz = shape
    zero = np.zeros((nz, ny, nx), F32)
    args = lambda vs: ([v[3] for v in vs], [v[0] for v in vs], [v[1] for v in vs], [v[2] for v in vs])   # noqa: E731
    one, r1 = mo.integrate((zero, zero, zero), origin, voxel, *args(views), trunc=0.1)
    a, ra = mo.integrate((zero, zero, zero), origin, voxel, *args(views[:2]), trunc=0.1)
    b, rb = mo.integrate(a, origin, voxel, *args(views[2:]), trunc=0.1)
    for x, y in zip(one, b):
        assert x.tobytes() == y.tobytes()
    assert r1[0] == ra[0] + rb[0] and r1[0] > 0


def test_host_math_against_oracle():
    rng = np.random.default_rng(5)
    reqs, expect = [], []
    for _ in range(200):
        origin = rng.normal(0, 1, 3)
        voxel = rng.uniform(0.001, 0.1)
        i, j, k = (int(v) for v in rng.integers(0, 2048, 3))
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        th = rng.uniform(0, np.pi)
        S = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.cos(th) * np.eye(3) + np.sin(th) * S + (1 - np.cos(th)) * np.outer(a, a)
        t = rng.normal(0, 1, 3) + np.array([0, 0, 80.0 * voxel])
        cam = np.array([rng.uniform(50, 500), rng.uniform(50, 500), rng.uniform(0, 300), rng.uniform(0, 200)], np.float32)
        w, h = int(rng.integers(1, 640)), int(rng.integers(1, 480))
        reqs.append("p " + " ".join("%.17g" % v for v in [*origin, voxel, i, j, k, *R.ravel(), *t, *cam, w, h]))
        Xg = [origin[0] + voxel * float(i), origin[1] + voxel * float(j), origin[2] + voxel * float(k)]
        Xc = [R[r, 0] * Xg[0] + R[r, 1] * Xg[1] + R[r, 2] * Xg[2] + t[r] for r in range(3)]
        expect.append((Xg, Xc, cam, w, h))
    rows = _mesh_math(reqs)
    found = 0
    for row, (Xg, Xc, cam, w, h) in zip(rows, expect):
        vals = [float(v) for v in row[:6]]
        assert vals == Xg + Xc
        ok, qx, qy = int(row[6]), int(row[7]), int(row[8])
        e_ok = Xc[2] > 0
        if e_ok:
            u = float(cam[0]) * Xc[0] / Xc[2] + float(cam[2])
            v = float(cam[1]) * Xc[1] / Xc[2] + float(cam[3])
            fu, fv = np.floor(u + 0.5), np.floor(v + 0.5)
            e_ok = 0 <= fu < w and 0 <= fv < h
        assert ok == int(e_ok)
        if ok:
            found += 1
            assert (qx, qy) == (int(fu), int(fv))
    assert found > 10
    # tau and the update
    reqs, exp = [], []
    for _ in range(300):
        D = F32(rng.uniform(0.5, 3))
        z = float(D) + rng.normal(0, 0.2)
        tr = F32(rng.uniform(0.01, 0.3))
        reqs.append("t %.9g %.17g %.9g" % (D, z, tr))
        sdf = np.float64(D) - z
        exp.append((0, None) if sdf < -np.float64(tr) else (1, F32(min(1.0, sdf / np.float64(tr)))))
    for row, (ok, tau) in zip(_mesh_math(reqs), exp):
        assert int(row[0]) == ok and (tau is None or F32(row[1]) == tau)
    reqs, exp = [], []
    for _ in range(300):
        T, W, G = F32(rng.uniform(-1, 1)), F32(rng.integers(0, 50)), F32(rng.uniform(0, 255))
        tau, g = F32(rng.uniform(-1, 1)), F32(rng.integers(0, 256))
        reqs.append("u %.9g %.9g %.9g %.9g %.9g" % (T, W, G, tau, g))
        Tn, Wn, Gn = mo.fold(np.array([T]), np.array([W]), np.array([G]), np.array([True]), np.array([tau]), np.array([g]))
        exp.append((Tn[0], Wn[0], Gn[0]))
    for row, e in zip(_mesh_math(reqs), exp):
        assert tuple(F32(v) for v in row) == e
    # the edge vertex against mo.vertex_records on a random volume
    nx, ny, nz = 7, 5, 6
    T = rng.normal(0, 1, (nz, ny, nx)).astype(F32)
    G = rng.uniform(0, 255, (nz, ny, nx)).astype(F32)
    origin, voxel = (0.3, -1.7, 2.2), 0.037
    keys, reqs = [], []
    Tf, Gf = T.ravel(), G.ravel()
    for g in range(nx * ny * nz):
        i, j, k = g % nx, (g // nx) % ny, g // (nx * ny)
        for d in range(1, 8):
            if i + (d & 1) >= nx or j + (d >> 1 & 1) >= ny or k + (d >> 2 & 1) >= nz:
                continue
            gb = g + (d & 1) + nx * ((d >> 1 & 1) + ny * (d >> 2 & 1))
            if (Tf[g] < 0) == (Tf[gb] < 0):
                continue
            keys.append(8 * g + d)
            reqs.append("v %.9g %.9g %.9g %.9g %d %d %d %d %.9g %.9g %.9g %.9g" % (F32(origin[0]), F32(origin[1]), F32(origin[2]), F32(voxel),
                                                                                   i, j, k, d, Tf[g], Tf[gb], Gf[g], Gf[gb]))
    ref = mo.vertex_records(T, G, origin, voxel, keys)
    got = np.array([[F32(v) for v in row] for row in _mesh_math(reqs)], F32)
    assert len(keys) > 50 and got.tobytes() == ref.tobytes()


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_mesh.h is exported and listed in api.MESH_EXPORTS, apart from the others; the ctypes
    structures and the vertex dtype match the header"""
    import ctypes as C
    import re
    from popsift_b200 import api
    body = open(os.path.join(ROOT, "include", "popsift_b200_mesh.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.MESH_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS,
                  api.BUNDLE_EXPORTS, api.GLOBAL_EXPORTS, api.VIEWGRAPH_EXPORTS, api.TWOVIEW_EXPORTS, api.DEPTH_EXPORTS):
        assert not set(api.MESH_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.MESH_EXPORTS:
        assert hasattr(lib, name)
    for struct, cls, size in (("ps_volume", api.PsVolume, 72), ("ps_tsdf_params", api.PsTsdfParams, 8),
                              ("ps_mesh_params", api.PsMeshParams, 8), ("ps_tsdf_report", api.PsTsdfReport, 16),
                              ("ps_mesh_report", api.PsMeshReport, 24)):
        block = body[body.index("typedef struct %s" % struct):]
        assert C.sizeof(cls) == size and "%d bytes" % size in block[:80]
        block = block[:block.index("} %s;" % struct)]
        names = re.findall(r"\b(\w+)\s*(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct, names)
    block = body[body.index("typedef struct ps_mesh_vertex"):]
    block = block[:block.index("} ps_mesh_vertex;")]
    assert "16 bytes" in block[:80] and api.MESH_VERTEX_DTYPE.itemsize == 16
    assert re.findall(r"\b(\w+)\s*(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S)) == list(api.MESH_VERTEX_DTYPE.names)
