"""ps_mesh_render and ps_mesh_texture (include/popsift_b200_render.h) restated in numpy: float64 in the header's operation
order, float32 where the header rounds.  Vectorised over triangles, candidate pixels and texels."""
import numpy as np

F32, F64 = np.float32, np.float64


def positions(vertices):
    """(n, 3) float64 positions of a MESH_VERTEX_DTYPE array or a float32 (n, 4) array, and the (n,) grey levels"""
    v = np.asarray(vertices)
    if v.dtype.names:
        return v["X"].astype(F64), v["grey"].astype(F64)
    v = np.asarray(v, F32).reshape(-1, 4)
    return v[:, :3].astype(F64), v[:, 3].astype(F64)


def project(cam, R, t, X, z_near):
    """render step 1 for points X (n, 3): (ok, p (n, 2), z)"""
    cam = np.asarray(cam, F32).astype(F64)
    R, t = np.asarray(R, F64), np.asarray(t, F64)
    Xc = [R[r, 0] * X[:, 0] + R[r, 1] * X[:, 1] + R[r, 2] * X[:, 2] + t[r] for r in range(3)]
    with np.errstate(all="ignore"):
        ok = np.isfinite(Xc[0]) & np.isfinite(Xc[1]) & np.isfinite(Xc[2]) & (Xc[2] >= z_near)
        p = np.stack([cam[0] * Xc[0] / Xc[2] + cam[2], cam[1] * Xc[1] / Xc[2] + cam[3]], 1)
    ok &= np.isfinite(p).all(1)
    return ok, p, Xc[2]


def edge(a, b, x, y):
    """E(a, b; x, y) = (b_x - a_x)(y - a_y) - (b_y - a_y)(x - a_x)"""
    return (b[..., 0] - a[..., 0]) * (y - a[..., 1]) - (b[..., 1] - a[..., 1]) * (x - a[..., 0])


def setup(cam, R, t, X, tris, w, h, z_near):
    """render steps 1-2 per triangle: drawn mask, p (m, 3, 2), z (m, 3), A (m,), box (m, 4) = x0, x1, y0, y1"""
    m = len(tris)
    ok, p, z = project(cam, R, t, X, z_near)
    P, Z = p[tris], z[tris]
    drawn = ok[tris].all(1)
    with np.errstate(all="ignore"):
        A = edge(P[:, 0], P[:, 1], P[:, 2, 0], P[:, 2, 1])
        drawn &= np.isfinite(A) & (A != 0)
        lx = np.maximum(np.ceil(np.minimum(np.minimum(P[:, 0, 0], P[:, 1, 0]), P[:, 2, 0])), 0.0)
        hx = np.minimum(np.floor(np.maximum(np.maximum(P[:, 0, 0], P[:, 1, 0]), P[:, 2, 0])), w - 1.0)
        ly = np.maximum(np.ceil(np.minimum(np.minimum(P[:, 0, 1], P[:, 1, 1]), P[:, 2, 1])), 0.0)
        hy = np.minimum(np.floor(np.maximum(np.maximum(P[:, 0, 1], P[:, 1, 1]), P[:, 2, 1])), h - 1.0)
    drawn &= (lx <= hx) & (ly <= hy)
    box = np.zeros((m, 4), np.int64)
    box[drawn] = np.stack([lx, hx, ly, hy], 1)[drawn].astype(np.int64)
    return drawn, P, Z, A, box


def _candidates(box, sel, chunk=1 << 22):
    """(triangle, x, y) of every candidate pixel of the triangles sel, in chunks of about `chunk` candidates"""
    bw = box[sel, 1] - box[sel, 0] + 1
    bh = box[sel, 3] - box[sel, 2] + 1
    cnt = bw * bh
    start = 0
    while start < len(sel):
        cum = np.cumsum(cnt[start:])
        stop = start + max(1, int(np.searchsorted(cum, chunk, side="right")))
        c = cnt[start:stop]
        tri = np.repeat(np.arange(start, stop), c)
        first = np.repeat(np.cumsum(c) - c, c)
        local = np.arange(int(c.sum())) - first
        yield sel[tri], box[sel[tri], 0] + local % bw[tri], box[sel[tri], 2] + local // bw[tri]
        start = stop


def cover(P, Z, A, x, y):
    """render steps 3-4 for candidates of triangles (P, Z, A rows per candidate): covered mask, float32 depth, and the
    smallest |lambda_i|"""
    fx, fy = x.astype(F64), y.astype(F64)
    E0, E1, E2 = edge(P[:, 1], P[:, 2], fx, fy), edge(P[:, 2], P[:, 0], fx, fy), edge(P[:, 0], P[:, 1], fx, fy)
    pos = A > 0
    cov = np.where(pos, (E0 >= 0) & (E1 >= 0) & (E2 >= 0), (E0 <= 0) & (E1 <= 0) & (E2 <= 0))
    l0, l1, l2 = E0 / A, E1 / A, E2 / A
    with np.errstate(all="ignore"):
        z = (1.0 / (l0 / Z[:, 0] + l1 / Z[:, 1] + l2 / Z[:, 2])).astype(F32)
    return cov, z, np.minimum(np.minimum(np.abs(l0), np.abs(l1)), np.abs(l2))


def key(z, m):
    return (z.astype(F32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | m.astype(np.uint64)


EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def render(vertices, tris, cams, poses, sizes, z_near=1e-3, margins=False, big=64):
    """ps_mesh_render: per view (depth, tri), the report (drawn, big, covered), and with margins=True per view a mask of the
    pixels whose winner is clear: every |lambda_i| of the winner > 1e-9 and the second-best depth more than 1e-6
    relative behind (or no second)"""
    X, _ = positions(vertices)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    zn = float(F32(z_near))
    depths, tri_maps, clear_maps = [], [], []
    n_drawn = n_big = n_cov = 0
    for cam, (R, t), (w, h) in zip(cams, poses, sizes):
        zb = np.full(w * h, EMPTY, np.uint64)
        drawn, P, Z, A, box = setup(cam, R, t, X, tris, w, h, zn)
        sel = np.flatnonzero(drawn)
        area = (box[sel, 1] - box[sel, 0] + 1) * (box[sel, 3] - box[sel, 2] + 1)
        n_drawn += len(sel)
        n_big += int((area > big).sum())
        kept = []
        for m, x, y in _candidates(box, sel):
            cov, z, lmin = cover(P[m], Z[m], A[m], x, y)
            pix = y[cov] * w + x[cov]
            np.minimum.at(zb, pix, key(z[cov], m[cov]))
            if margins:
                kept.append((pix, z[cov], m[cov], lmin[cov]))
        hit = zb != EMPTY
        n_cov += int(hit.sum())
        D = np.where(hit, (zb >> np.uint64(32)).astype(np.uint32).view(F32), F32(0)).astype(F32)
        T = np.where(hit, (zb & np.uint64(0xFFFFFFFF)).astype(np.int64), -1).astype(np.int32)
        depths.append(D.reshape(h, w))
        tri_maps.append(T.reshape(h, w))
        if margins:
            clear = np.ones(w * h, bool)
            second = np.full(w * h, np.inf)
            for pix, z, m, lmin in kept:
                win = T[pix] == m
                clear[pix[win & (lmin <= 1e-9)]] = False
                np.minimum.at(second, pix[~win], z[~win].astype(F64))
            gap = second - D.astype(F64)
            clear &= ~(hit & (gap <= 1e-6 * np.maximum(D.astype(F64), 1e-30)))
            clear_maps.append(clear.reshape(h, w))
    rep = {"drawn": n_drawn, "big": n_big, "covered": n_cov}
    return (depths, tri_maps, rep, clear_maps) if margins else (depths, tri_maps, rep)


def frame(X, tris):
    """texture step 1: centroid and normal per triangle"""
    V0, V1, V2 = X[tris[:, 0]], X[tris[:, 1]], X[tris[:, 2]]
    C = (V0 + V1 + V2) / 3.0
    a, b = V1 - V0, V2 - V0
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    return (V0, V1, V2), C, n


def centre(R, t):
    R, t = np.asarray(R, F64), np.asarray(t, F64)
    return np.array([-(R[0, k] * t[0] + R[1, k] * t[1] + R[2, k] * t[2]) for k in range(3)])


def select(vertices, tris, cams, poses, sizes, depths, min_cos=0.1, depth_tol=0.01, z_near=1e-3):
    """texture steps 1-3: the view per triangle (-1 without a candidate)"""
    X, _ = positions(vertices)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    (V0, V1, V2), C, n = frame(X, tris)
    zn, tol1, mc = float(F32(z_near)), 1.0 + float(F32(depth_tol)), float(F32(min_cos))
    best = np.full(len(tris), -1, np.int32)
    best_score = np.full(len(tris), -1.0)
    for v, (cam, (R, t), (w, h), D) in enumerate(zip(cams, poses, sizes, depths)):
        d = centre(R, t)[None, :] - C
        nd = n[:, 0] * d[:, 0] + n[:, 1] * d[:, 1] + n[:, 2] * d[:, 2]
        nn = np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
        dd = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
        cand = (nd > 0) & (nd >= mc * nn * dd)
        Dm = np.asarray(D, F32).reshape(h, w)
        ps = []
        for Pk in (V0, V1, V2, C):
            ok, p, z = project(cam, R, t, Pk, zn)
            with np.errstate(all="ignore"):
                qx, qy = np.floor(p[:, 0] + 0.5), np.floor(p[:, 1] + 0.5)
                ok &= (qx >= 0) & (qx < w) & (qy >= 0) & (qy < h)
            qxi, qyi = np.where(ok, qx, 0).astype(np.int64), np.where(ok, qy, 0).astype(np.int64)
            Dq = Dm[qyi, qxi].astype(F64)
            ok &= ~((Dq > 0) & (z > Dq * tol1))
            cand &= ok
            ps.append(p)
        with np.errstate(all="ignore"):
            score = np.abs(edge(ps[0], ps[1], ps[2][:, 0], ps[2][:, 1])) / 2.0
        win = cand & (score > best_score)
        best[win] = v
        best_score[win] = score[win]
    return best


def texel_uv(i, j, cell):
    """texture step 5: the clamped (u, v) of texels (i, j)"""
    s = float(cell - 2)
    u = np.maximum((i.astype(F64) + 0.5 - 1.0) / s, 0.0)
    v = np.maximum((j.astype(F64) + 0.5 - 1.0) / s, 0.0)
    over = u + v > 1.0
    uu = np.minimum(np.maximum((u - v + 1.0) / 2.0, 0.0), 1.0)
    return np.where(over, uu, u), np.where(over, 1.0 - uu, v)


def bilinear(img, x, y):
    """texture step 6: the clamped bilinear sample of a uint8 image"""
    h, w = img.shape
    x = np.fmin(np.fmax(x, 0.0), w - 1.0)
    y = np.fmin(np.fmax(y, 0.0), h - 1.0)
    u0 = np.minimum(np.floor(x).astype(np.int64), w - 2)
    v0 = np.minimum(np.floor(y).astype(np.int64), h - 2)
    a, c = x - u0, y - v0
    I = img.astype(F64)
    return (1.0 - c) * ((1.0 - a) * I[v0, u0] + a * I[v0, u0 + 1]) + c * ((1.0 - a) * I[v0 + 1, u0] + a * I[v0 + 1, u0 + 1])


def to_u8(S):
    return np.fmin(np.fmax(np.floor(S + 0.5), 0.0), 255.0).astype(np.uint8)


def texel_points(vertices, tris, cell, m, i, j):
    """texture steps 5-6: the world point X (k, 3) and the fallback value S of texels (i, j) of triangles m"""
    X, g = positions(vertices)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    u, v = texel_uv(i, j, cell)
    b = (1.0 - u - v, u, v)
    T = tris[m]
    P = b[0][:, None] * X[T[:, 0]] + b[1][:, None] * X[T[:, 1]] + b[2][:, None] * X[T[:, 2]]
    S = b[0] * g[T[:, 0]] + b[1] * g[T[:, 1]] + b[2] * g[T[:, 2]]
    return P, S


def atlas(vertices, tris, images, cams, poses, view, cell, cells_per_row):
    """texture steps 4-6: the uint8 atlas (H, W) given the view per triangle"""
    n_tri = len(view)
    W, H = cells_per_row * cell, -(-n_tri // cells_per_row) * cell
    Y, Xa = np.mgrid[0:H, 0:W]
    Y, Xa = Y.ravel(), Xa.ravel()
    cx, cy = Xa // cell, Y // cell
    m = cy * cells_per_row + cx
    out = np.zeros(H * W, np.uint8)
    live = np.flatnonzero(m < n_tri)
    mm = m[live]
    P, S = texel_points(vertices, tris, cell, mm, Xa[live] - cx[live] * cell, Y[live] - cy[live] * cell)
    vw = np.asarray(view)[mm]
    for v in np.unique(vw[vw >= 0]):
        sel = vw == v
        cam, (R, t) = cams[v], poses[v]
        _, p, _ = project(cam, R, t, P[sel], -np.inf)
        S[sel] = bilinear(np.asarray(images[v], np.uint8), p[:, 0], p[:, 1])
    out[live] = to_u8(S)
    return out.reshape(H, W)
