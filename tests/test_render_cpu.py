"""ps_mesh_render and ps_mesh_texture without a GPU: the rules of tests/render_oracle.py on planted scenes (perspective-
correct depth, occlusion, the tie rule, a closed mesh without cracks, culling; the view choice; the atlas layout and its
margins), the OBJ / MTL / PNG writer, the host build of k_render.h (tests/cpp/render_math_check.cpp) against the oracle,
and the header's exports and layouts."""
import os
import re
import struct
import subprocess
import sys
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
import mesh_oracle as mo                                   # noqa: E402
import render_oracle as ro                                 # noqa: E402

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAM = np.array([100.0, 100.0, 32.0, 24.0], F32)
W, H = 64, 48
EYE = (np.eye(3), np.zeros(3))


def _verts(X, grey=None):
    X = np.asarray(X, np.float64).reshape(-1, 3)
    g = np.zeros(len(X)) if grey is None else np.asarray(grey, np.float64)
    return np.concatenate([X, g[:, None]], 1).astype(F32)


def _look_at(C, target=(0.0, 0.0, 5.0)):
    C = np.asarray(C, np.float64)
    z = np.asarray(target, np.float64) - C
    z /= np.linalg.norm(z)
    x = np.cross([0.0, 1.0, 0.0] if abs(z[1]) < 0.9 else [1.0, 0.0, 0.0], z)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z])
    return R, -R @ C


def test_planar_depth_is_perspective_correct():
    """the depth of a triangle in a slanted plane equals the ray-plane intersection at every covered pixel"""
    n, d = np.array([0.3, -0.2, 1.0]), 4.0
    P = [(-1.5, -1.0), (1.8, -0.9), (0.1, 1.4)]
    X = [(x, y, (d - n[0] * x - n[1] * y) / n[2]) for x, y in P]
    depth, tri, rep = ro.render(_verts(X), [[0, 1, 2]], [CAM], [EYE], [(W, H)])
    D = depth[0].astype(np.float64)
    y, x = np.nonzero(tri[0] == 0)
    ray = np.stack([(x - CAM[2]) / CAM[0], (y - CAM[3]) / CAM[1], np.ones(len(x))], 1)
    truth = d / (ray @ n)
    assert len(x) > 300 and rep["drawn"] == 1 and rep["covered"] == len(x)
    assert np.abs(D[y, x] / truth - 1).max() < 1e-6
    # an affine interpolation of z in the image would be off by far more
    assert (D[tri[0] < 0] == 0).all()


def test_occlusion_and_tie_rule():
    # a nearer triangle (index 1) in front of a farther one (index 0)
    far = [(-2, -2, 6), (2, -2, 6), (0, 2, 6)]
    near = [(-0.5, -0.5, 3), (0.5, -0.5, 3), (0, 0.5, 3)]
    depth, tri, _ = ro.render(_verts(far + near), [[0, 1, 2], [3, 4, 5]], [CAM], [EYE], [(W, H)])
    assert (tri[0] == 1).sum() > 50 and (tri[0] == 0).sum() > 50
    assert (depth[0][tri[0] == 1] == 3).all() and (depth[0][tri[0] == 0] == 6).all()
    # equal depths on exactly representable coordinates: the lower index wins, whatever the order in the list
    quad = [(-1, -1, 4), (1, -1, 4), (1, 1, 4), (-1, 1, 4)]
    for tris in ([[0, 1, 2], [0, 2, 3], [2, 1, 0]], [[2, 1, 0], [0, 2, 3], [0, 1, 2]]):
        _, tri, _ = ro.render(_verts(quad), tris, [CAM], [EYE], [(W, H)])
        both = [m for m in range(3) if sorted(tris[m]) == [0, 1, 2]]
        assert not (tri[0] == max(both)).any() and (tri[0] == min(both)).sum() > 100
        # the shared diagonal's pixels belong to both triangles of the quad; the z-buffer gives them one
        assert (tri[0] >= 0).sum() == 51 * 48


def _sphere_mesh(n=40, r=0.8):
    o, h = (-1.0, -1.0, -1.0), 2.0 / (n - 1)
    X, Y, Z = mo.grid_points(o, h, (n, n, n))
    T = (np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - r).astype(F32)
    V, tris, rep, _ = mo.mesh((T, np.ones_like(T), np.full(T.shape, 100.0, F32)), o, h, 1.0)
    return V, tris, h


def test_closed_sphere_renders_without_cracks():
    V, tris, h = _sphere_mesh()
    boundary, dup, chi = mo.topology(tris, len(V))
    assert len(boundary) == 0 and chi == 2
    for C in ((0.0, 0.0, -3.0), (1.7, -1.1, -2.3), (0.3, 2.9, 0.4)):
        R, t = _look_at(C, (0.0, 0.0, 0.0))
        depth, tri, rep = ro.render(V, tris, [CAM], [(R, t)], [(W, H)])
        # pixels whose ray passes the centre closer than r - 2 voxels see the sphere
        y, x = np.mgrid[0:H, 0:W].astype(np.float64)
        d = R.T @ np.stack([(x.ravel() - CAM[2]) / CAM[0], (y.ravel() - CAM[3]) / CAM[1], np.ones(H * W)])
        d /= np.linalg.norm(d, axis=0)
        o = np.asarray(C)
        dist = np.linalg.norm(o[:, None] - (o @ d) * d, axis=0)
        inside = dist < 0.8 - 2 * h
        assert inside.sum() > 500
        assert (tri[0].ravel()[inside] >= 0).all(), C
        # the nearest surface: the depth is that of the front of the sphere, not the back
        front = (-(o @ d) - np.sqrt(np.maximum(0.8 ** 2 - dist ** 2, 0))) * (R @ d)[2]
        assert np.abs(depth[0].ravel()[inside] - front[inside]).max() < 1.5 * h


def test_culling():
    ok = [(-0.5, -0.5, 3), (0.5, -0.5, 3), (0, 0.5, 3)]
    cases = {
        "behind z_near": [(-0.5, -0.5, 3), (0.5, -0.5, 3), (0, 0.5, -1)],
        "straddles z_near": [(-0.5, -0.5, 3), (0.5, -0.5, 3), (0, 0.5, 0.0005)],
        "degenerate": [(-0.5, -0.5, 3), (0.0, 0.0, 3), (0.5, 0.5, 3)],
        "off image": [(5, 5, 3), (6, 5, 3), (5, 6, 3)],
        "between pixels": [(0.001, 0.001, 3), (0.002, 0.001, 3), (0.001, 0.002, 3)],
    }
    _, _, rep = ro.render(_verts(ok), [[0, 1, 2]], [CAM], [EYE], [(W, H)])
    assert rep["drawn"] == 1
    for name, X in cases.items():
        depth, tri, rep = ro.render(_verts(X), [[0, 1, 2]], [CAM], [EYE], [(W, H)], z_near=1e-3)
        assert rep["drawn"] == 0 and rep["covered"] == 0 and (tri[0] == -1).all() and (depth[0] == 0).all(), name
    # the big-triangle count: boxes above 64 pixels
    small = [(0.0, 0.0, 3), (0.09, 0.0, 3), (0.0, 0.09, 3)]
    _, _, rep = ro.render(_verts([(-3, -3, 3), (3, -3, 3), (0, 3, 3)] + small), [[0, 1, 2], [3, 4, 5]], [CAM], [EYE], [(W, H)])
    assert rep["drawn"] == 2 and rep["big"] == 1


TRI = [(-0.5, 0.5, 5.0), (0.5, -0.5, 5.0), (-0.5, -0.5, 5.0)]   # normal (0, 0, -1), towards the cameras at z < 5


def _select(views, depths=None, min_cos=0.1, depth_tol=0.01, grey=(10, 20, 30)):
    V = _verts(TRI, grey)
    cams = [CAM] * len(views)
    sizes = [(W, H)] * len(views)
    depths = depths or [np.zeros((H, W), F32) for _ in views]
    return ro.select(V, [[0, 1, 2]], cams, views, sizes, depths, min_cos=min_cos, depth_tol=depth_tol)[0]


def test_view_choice():
    plain, near = EYE, (np.eye(3), np.array([0.0, 0.0, -2.0]))
    back = _look_at((0.0, 0.0, 10.0))
    graze = _look_at((20.0, 0.0, 3.0))
    assert _select([plain]) == 0 and _select([near]) == 0
    # the largest projected area wins, ties go to the lowest view
    assert _select([plain, near]) == 1 and _select([near, plain]) == 0 and _select([plain, plain]) == 0
    # back-facing and grazing views are rejected
    assert _select([back]) == -1 and _select([graze]) == -1 and _select([graze], min_cos=0.09) == 0
    # occluded: a depth map with something nearer in front; within the tolerance it is not
    assert _select([near], depths=[np.full((H, W), 2.5, F32)]) == -1
    assert _select([near], depths=[np.full((H, W), 3.0 / 1.005, F32)]) == 0
    assert _select([near], depths=[np.full((H, W), 3.0 / 1.02, F32)]) == -1
    # the triangle's own rendered depth does not occlude it
    V = _verts(TRI)
    D, _, _ = ro.render(V, [[0, 1, 2]], [CAM], [near], [(W, H)])
    assert _select([near], depths=D) == 0
    # a probe outside the image rejects the view
    assert _select([(np.eye(3), np.array([0.25, 0.0, -4.5]))]) == -1


def test_fallback_and_atlas_layout():
    from popsift_b200 import api
    rng = np.random.default_rng(3)
    n_tri, cell, cpr = 5, 6, 2
    X = rng.normal(size=(7, 3)) + [0, 0, 5]
    g = rng.uniform(0, 255, 7)
    V = _verts(X, g)
    tris = rng.integers(0, 7, (n_tri, 3))
    atlas = ro.atlas(V, tris, [], [], [], np.full(n_tri, -1), cell, cpr)
    uv, Wa, Ha = api.atlas_uv(n_tri, cell, cpr)
    assert atlas.shape == (Ha, Wa) == (18, 12)
    assert (uv[3] == [[cell + 1, cell + 1], [2 * cell - 1, cell + 1], [cell + 1, 2 * cell - 1]]).all()
    assert (atlas[12:, 6:] == 0).all()                         # the cell past the last triangle
    assert api.atlas_cells_per_row(10 ** 6, 8) == 1000 and api.atlas_cells_per_row(10 ** 9, 8) == 65535 // 8
    for m in range(n_tri):
        cx, cy = m % cpr, m // cpr
        P0, P1, P2 = uv[m]
        for j in range(cell):
            for i in range(cell):
                q = np.array([cx * cell + i + 0.5, cy * cell + j + 0.5])
                # the nearest point of the triangle P0 P1 P2 to the texel centre, by dense search on its boundary and inside
                s = np.linspace(0, 1, 401)
                a, b = np.meshgrid(s, s)
                keep = a + b <= 1
                pts = P0 + a[keep, None] * (P1 - P0) + b[keep, None] * (P2 - P0)
                k = np.argmin(((pts - q) ** 2).sum(1))
                u, v = ro.texel_uv(np.array([i]), np.array([j]), cell)
                assert abs(u[0] - a[keep][k]) < 3e-3 and abs(v[0] - b[keep][k]) < 3e-3
                S = (1 - u[0] - v[0]) * g[tris[m, 0]] + u[0] * g[tris[m, 1]] + v[0] * g[tris[m, 2]]
                assert atlas[cy * cell + j, cx * cell + i] == ro.to_u8(np.array([S]))[0]


def _png_decode(path):
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, ihdr = 8, b"", None
    while pos < len(data):
        n, tag = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xffffffff
        if tag == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + n
    w, h, depth, ctype = ihdr[:4]
    assert depth == 8 and ctype == 0
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, w + 1)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:]


def test_write_obj_round_trip(tmp_path):
    from popsift_b200 import api
    rng = np.random.default_rng(5)
    V = np.zeros(9, api.MESH_VERTEX_DTYPE)
    V["X"] = rng.normal(size=(9, 3))
    tris = rng.integers(0, 9, (11, 3)).astype(np.int32)
    mesh = api.Mesh(V, tris, {})
    uv, Wa, Ha = api.atlas_uv(11, 8, 4)
    tex = api.TexturedMesh(rng.integers(0, 256, (Ha, Wa)).astype(np.uint8), np.zeros(11, np.int32), uv, {})
    paths = api.write_obj(str(tmp_path / "m.obj"), mesh, tex)
    assert paths == [str(tmp_path / f) for f in ("m.obj", "m.mtl", "m.png")]
    lines = open(paths[0]).read().splitlines()
    assert lines[0] == "mtllib m.mtl"
    v = np.array([[float(x) for x in l.split()[1:]] for l in lines if l.startswith("v ")])
    vt = np.array([[float(x) for x in l.split()[1:]] for l in lines if l.startswith("vt ")])
    f = [[tuple(int(k) for k in c.split("/")) for c in l.split()[1:]] for l in lines if l.startswith("f ")]
    assert np.array_equal(v.astype(F32), V["X"]) and len(f) == 11
    for m, face in enumerate(f):
        assert [c[0] - 1 for c in face] == list(tris[m])
        got = vt[[c[1] - 1 for c in face]]
        assert np.allclose(got[:, 0] * Wa, uv[m, :, 0]) and np.allclose((1 - got[:, 1]) * Ha, uv[m, :, 1])
    assert "map_Kd m.png" in open(paths[1]).read()
    assert np.array_equal(_png_decode(paths[2]), tex.atlas)
    # without a texture: positions and faces only
    plain = api.write_obj(str(tmp_path / "p.obj"), mesh)
    body = open(plain[0]).read()
    assert plain == [str(tmp_path / "p.obj")] and "vt" not in body and body.count("\nf ") == 11


def _math(requests):
    from popsift_b200 import build as B
    assert os.path.exists(B.RENDER_MATH_CHECK), "python -m popsift_b200.build builds render_math_check"
    out = subprocess.run([B.RENDER_MATH_CHECK], input="\n".join(requests) + "\n", capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    return [l.split()[1:] for l in out.stdout.splitlines()]


def _g(v):
    return "%.17g" % v


def test_render_math_check_matches_oracle():
    rng = np.random.default_rng(11)
    reqs, expect = [], []
    for _ in range(400):
        cam = np.array([rng.uniform(50, 150), rng.uniform(50, 150), rng.uniform(20, 40), rng.uniform(15, 30)], F32)
        R, t = _look_at(rng.normal(size=3) * 0.5, rng.normal(size=3) * 0.3 + [0, 0, 4])
        X = (rng.normal(size=(3, 3)) * rng.choice([0.05, 0.5, 3.0]) + [0, 0, 4]).astype(F32).astype(np.float64)
        zn = float(F32(rng.choice([1e-3, 3.9])))
        drawn, P, Z, A, box = ro.setup(cam, R, t, X, np.array([[0, 1, 2]]), W, H, zn)
        x, y = (int(rng.integers(box[0, 0], box[0, 1] + 1)), int(rng.integers(box[0, 2], box[0, 3] + 1))) if drawn[0] else (5, 5)
        cov, z, _ = ro.cover(P, Z, A, np.array([x]), np.array([y]))
        c = bool(drawn[0] and x >= box[0, 0] and x <= box[0, 1] and y >= box[0, 2] and y <= box[0, 3] and cov[0])
        a = list(cam) + list(R.ravel()) + list(t) + [W, H, zn] + list(X.ravel()) + [x, y]
        reqs.append("r " + " ".join(_g(float(v)) for v in a))
        expect.append((int(drawn[0]), A[0] if drawn[0] else 0.0, tuple(box[0]) if drawn[0] else (0, 0, 0, 0), int(c),
                       float(z[0]) if c else 0.0, int(ro.key(z, np.array([7]))[0]) if c else 0))
    got = _math(reqs)
    n_cov = 0
    for g, e in zip(got, expect):
        assert int(g[0]) == e[0]
        if e[0]:
            assert float(g[1]) == e[1] and tuple(int(v) for v in g[2:6]) == e[2]
        assert int(g[6]) == e[3]
        if e[3]:
            n_cov += 1
            assert F32(float(g[7])) == F32(e[4]) and int(g[8]) == e[5]
    assert n_cov > 20
    # facing, probes and score
    reqs, expect = [], []
    for _ in range(200):
        R, t = _look_at(rng.normal(size=3) * 2.0)
        X = (rng.normal(size=(3, 3)) * 0.5 + [0, 0, 5]).astype(F32).astype(np.float64)
        D = np.where(rng.random((6, 8)) < 0.5, rng.uniform(1, 8, (6, 8)), 0).astype(F32)
        cam = np.array([8.0, 8.0, 4.0, 3.0], F32)
        V = _verts(X)
        mc, tol = float(F32(rng.uniform(0, 0.5))), float(F32(0.01))
        view = ro.select(V, [[0, 1, 2]], [cam], [(R, t)], [(8, 6)], [D], min_cos=mc, depth_tol=tol, z_near=1e-3)[0]
        c = ro.centre(R, t)
        a = list(cam) + list(R.ravel()) + list(t) + list(c) + [8, 6, float(F32(1e-3)), 1.0 + tol, mc] + list(X.ravel()) + list(D.ravel())
        reqs.append("f " + " ".join(_g(float(v)) for v in a))
        expect.append(view)
    got = _math(reqs)
    assert sum(e == 0 for e in expect) > 5
    for g, e in zip(got, expect):
        assert (int(g[0]) and int(g[1])) == (e == 0)
    # texel barycentrics and bilinear samples
    reqs, expect = [], []
    for cell in (3, 4, 8, 17, 64):
        for j in range(cell):
            for i in range(cell):
                reqs.append("u %d %d %d" % (i, j, cell))
                u, v = ro.texel_uv(np.array([i]), np.array([j]), cell)
                expect.append((u[0], v[0]))
    got = _math(reqs)
    assert all(float(g[0]) == e[0] and float(g[1]) == e[1] for g, e in zip(got, expect))
    img = rng.integers(0, 256, (5, 7)).astype(np.uint8)
    pts = np.concatenate([rng.uniform(-1, 8, (300, 2)), [[6, 4], [0, 0], [6.0, 2.5], [-3, 9]]])
    got = _math(["b 7 5 %s %s %s" % (_g(x), _g(y), " ".join(str(int(v)) for v in img.ravel())) for x, y in pts])
    S = ro.bilinear(img, pts[:, 0], pts[:, 1])
    assert all(float(g[0]) == s and int(g[1]) == int(ro.to_u8(np.array([s]))[0]) for g, s in zip(got, S))


def test_header_exports_and_layouts():
    """every ps_*( of popsift_b200_render.h is exported and listed in api.RENDER_EXPORTS, apart from the others; the ctypes
    structures match the header"""
    import ctypes as C
    from popsift_b200 import api
    body = open(os.path.join(ROOT, "include", "popsift_b200_render.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert sorted(set(re.findall(r"\b(ps_\w+)\(", hdr))) == sorted(api.RENDER_EXPORTS)
    for other in (api.EXPORTS, api.GUIDED_EXPORTS, api.RETRIEVAL_EXPORTS, api.TRACKS_EXPORTS, api.POSE_EXPORTS, api.TRIANGULATE_EXPORTS,
                  api.BUNDLE_EXPORTS, api.GLOBAL_EXPORTS, api.VIEWGRAPH_EXPORTS, api.TWOVIEW_EXPORTS, api.DEPTH_EXPORTS, api.MESH_EXPORTS):
        assert not set(api.RENDER_EXPORTS) & set(other)
    lib = api.load_library()
    for name in api.RENDER_EXPORTS:
        assert hasattr(lib, name)
    for struct_name, cls, size in (("ps_render_params", api.PsRenderParams, 8), ("ps_render_report", api.PsRenderReport, 24),
                                   ("ps_texture_params", api.PsTextureParams, 24), ("ps_texture_report", api.PsTextureReport, 16)):
        block = body[body.index("typedef struct %s" % struct_name):]
        assert C.sizeof(cls) == size and "%d bytes" % size in block[:80]
        block = block[:block.index("} %s;" % struct_name)]
        names = re.findall(r"\b(\w+)\s*(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", block, flags=re.S))
        assert names == [f[0] for f in cls._fields_], (struct_name, names)
