"""The contracts of ps_tsdf_integrate and ps_tsdf_mesh (include/popsift_b200_mesh.h) in numpy, written from the header's
steps with nothing shared with the device code: float64 for the grid points, the projection and the signed distance,
float32 for the running averages and the mesh vertices, each in the header's operation order.  Volumes are numpy arrays
of shape (nz, ny, nx), so that their C-order flattening is the header's index i + nx (j + ny k)."""
import itertools

import numpy as np

F32 = np.float32


# ---- the Kuhn (Freudenthal) split and the triangle rule ---------------------------------------------------------------

def _corner(c):
    """cell corner code c = ex + 2 ey + 4 ez as an integer vector"""
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1])


def kuhn_tets():
    """The 6 tetrahedra of a cell as corner codes: for each permutation (a, b, c) of the axes in lexicographic order, the
    path 0, e_a, e_a + e_b, (1, 1, 1); odd permutations swap their second and third corners, so that every tetrahedron
    is positively oriented."""
    out = []
    for p in itertools.permutations(range(3)):
        a, b = p[0], p[1]
        v = [0, 1 << a, (1 << a) | (1 << b), 7]
        inversions = sum(1 for i in range(3) for j in range(i + 1, 3) if p[i] > p[j])
        if inversions % 2:
            v[1], v[2] = v[2], v[1]
        out.append(v)
    return np.array(out, np.int64)


def edge_code(c0, c1):
    """the edge between two corners of a tetrahedron as (lower corner) << 3 | direction; the corners of a Kuhn
    tetrahedron are ordered componentwise, so the lower one is the one with the fewer set bits"""
    lo, hi = (c0, c1) if bin(c0).count("1") < bin(c1).count("1") else (c1, c0)
    assert lo & hi == lo and lo != hi
    return (lo << 3) | (hi - lo)


def cell_edges():
    """the 19 edges of the split cell: (lower corner a, direction d) with a & d == 0, in (d, a) order"""
    return [(a, d) for d in range(1, 8) for a in range(8) if a & d == 0]


def triangle_table():
    """(count[6][16], tri[6][16][2][3]) of edge codes.  Case bit m is set when local corner m is inside.
    1 inside corner a: the triangle on its edges to the others, in local order; 3 inside: the triangle on the edges to
    the outside corner b from the inside ones, in local order; 2 inside a < b, outside c < d: the quad (ac, ad, bd, bc)
    split along the diagonal ac-bd into (ac, ad, bd) and (ac, bd, bc).  Each triangle is then oriented so that its
    normal points from the inside corners' centroid to the outside corners' at edge midpoints: swapped (v0, v2, v1)
    where it does not."""
    tets = kuhn_tets()
    count = np.zeros((6, 16), np.int64)
    tri = np.zeros((6, 16, 2, 3), np.int64)
    for t in range(6):
        v = [int(c) for c in tets[t]]
        for case in range(16):
            ins = [m for m in range(4) if case >> m & 1]
            outs = [m for m in range(4) if not case >> m & 1]
            if len(ins) == 1:
                a = ins[0]
                tris = [[(a, o) for o in outs]]
            elif len(ins) == 3:
                b = outs[0]
                tris = [[(i, b) for i in ins]]
            elif len(ins) == 2:
                a, b = ins
                c, d = outs
                tris = [[(a, c), (a, d), (b, d)], [(a, c), (b, d), (b, c)]]
            else:
                tris = []
            count[t, case] = len(tris)
            cin = np.mean([_corner(v[m]) for m in ins], 0) if ins else None
            cout = np.mean([_corner(v[m]) for m in outs], 0) if outs else None
            for n, tr in enumerate(tris):
                P = [(_corner(v[m0]) + _corner(v[m1])) / 2.0 for m0, m1 in tr]
                nrm = np.cross(P[1] - P[0], P[2] - P[0])
                if nrm @ (cout - cin) < 0:
                    tr = [tr[0], tr[2], tr[1]]
                tri[t, case, n] = [edge_code(v[m0], v[m1]) for m0, m1 in tr]
    return count, tri


# ---- integration ------------------------------------------------------------------------------------------------------

def grid_points(origin, voxel, shape):
    """X_g of every grid point as three (nz, ny, nx) float64 arrays: origin + voxel (i, j, k)"""
    nx, ny, nz = shape
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    o = [float(v) for v in origin]
    h = float(voxel)
    return o[0] + h * i.astype(np.float64), o[1] + h * j.astype(np.float64), o[2] + h * k.astype(np.float64)


def view_update(X, cam, pose, depth, grey, ncons, trunc, min_consistent):
    """steps 1-5 for one view over points X (three float64 arrays): (ok, tau float32, grey level float32)"""
    R, t = (np.asarray(a, np.float64) for a in pose)
    R = R.reshape(3, 3)
    t = t.reshape(3)
    Xc = [R[r, 0] * X[0] + R[r, 1] * X[1] + R[r, 2] * X[2] + t[r] for r in range(3)]
    fx, fy, cx, cy = (float(F32(v)) for v in cam)
    h, w = depth.shape
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = fx * Xc[0] / Xc[2] + cx
        v = fy * Xc[1] / Xc[2] + cy
        qu, qv = np.floor(u + 0.5), np.floor(v + 0.5)
    ok = (Xc[2] > 0) & (qu >= 0) & (qu < w) & (qv >= 0) & (qv < h)
    qx = np.where(ok, qu, 0).astype(np.int64)
    qy = np.where(ok, qv, 0).astype(np.int64)
    D = np.asarray(depth, F32)[qy, qx]
    ok &= D > 0
    if min_consistent > 0:
        ok &= np.asarray(ncons)[qy, qx] >= min_consistent
    tr = float(F32(trunc))
    sdf = D.astype(np.float64) - Xc[2]
    ok &= ~(sdf < -tr)
    with np.errstate(invalid="ignore", over="ignore"):
        tau = np.minimum(1.0, sdf / tr).astype(F32)
    return ok, tau, np.asarray(grey)[qy, qx].astype(F32)


def fold(T, W, G, ok, tau, g):
    """step 6 where ok: W' = W + 1, T' = (T W + tau) / W', G' = (G W + g) / W', all float32"""
    Wn = W + F32(1)
    Tn = (T * W + tau) / Wn
    Gn = (G * W + g) / Wn
    return np.where(ok, Tn, T), np.where(ok, Wn, W), np.where(ok, Gn, G)


def integrate(vol, origin, voxel, images, cams, poses, depths, masks=None, trunc=0.1, min_consistent=0):
    """ps_tsdf_integrate: vol = (T, W, G) float32 (nz, ny, nx) arrays; returns the new volume and the report
    (updates, voxels touched)"""
    T, W, G = (np.array(a, F32) for a in vol)
    nz, ny, nx = T.shape
    X = grid_points(origin, voxel, (nx, ny, nz))
    n_upd = np.zeros(T.shape, np.int64)
    for k in range(len(images)):
        ok, tau, g = view_update(X, cams[k], poses[k], depths[k], images[k], None if masks is None else masks[k], trunc, min_consistent)
        T, W, G = fold(T, W, G, ok, tau, g)
        n_upd += ok
    return (T, W, G), (int(n_upd.sum()), int((n_upd > 0).sum()))


# ---- extraction -------------------------------------------------------------------------------------------------------

def corner_offsets(nx, ny):
    return np.array([(c & 1) + nx * ((c >> 1) & 1) + nx * ny * ((c >> 2) & 1) for c in range(8)], np.int64)


def active_cells(T, W, min_weight):
    """(cell lower corners g in ascending order, their 8-bit inside masks) of the meshed cells with a sign change"""
    nz, ny, nx = T.shape
    Tf, Wf = T.ravel(), W.ravel()
    k, j, i = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    g = (i + nx * (j + ny * k)).ravel().astype(np.int64)
    off = corner_offsets(nx, ny)
    meshed = np.ones(len(g), bool)
    mask = np.zeros(len(g), np.int64)
    for c in range(8):
        meshed &= Wf[g + off[c]] >= F32(min_weight)
        mask |= (Tf[g + off[c]] < 0).astype(np.int64) << c
    act = meshed & (mask != 0) & (mask != 255)
    return g[act], mask[act]


def cell_counts(mask):
    """per cell mask: (sign-changing edges among the 19, triangles)"""
    count, _ = triangle_table()
    tets = kuhn_tets()
    nk = np.zeros(len(mask), np.int64)
    for a, d in cell_edges():
        nk += ((mask >> a) & 1) != ((mask >> (a + d)) & 1)
    nt = np.zeros(len(mask), np.int64)
    for t in range(6):
        case = sum(((mask >> int(tets[t, m])) & 1) << m for m in range(4))
        nt += count[t][case]
    return nk, nt


def mesh(vol, origin, voxel, min_weight=1.0):
    """ps_tsdf_mesh: (vertices float32 (n, 4) = X, grey; triangles int32 (m, 3); report (cells, vertices, triangles);
    the vertices' keys)"""
    T, W, G = (np.asarray(a, F32) for a in vol)
    nz, ny, nx = T.shape
    count, tri = triangle_table()
    tets = kuhn_tets()
    g, mask = active_cells(T, W, min_weight)
    keys = np.zeros((len(g), 6, 2, 3), np.int64)
    valid = np.zeros((len(g), 6, 2), bool)
    off = corner_offsets(nx, ny)
    for t in range(6):
        case = sum(((mask >> int(tets[t, m])) & 1) << m for m in range(4))
        n = count[t][case]
        for s in range(2):
            valid[:, t, s] = n > s
            e = tri[t][case, s]                                 # (cells, 3) edge codes
            keys[:, t, s] = (g[:, None] + off[e >> 3]) * 8 + (e & 7)
    tk = keys[valid]                                            # (cell, tet, triangle) order
    verts = np.unique(tk)
    tris = np.searchsorted(verts, tk).astype(np.int32).reshape(-1, 3)
    return vertex_records(T, G, origin, voxel, verts), tris, (len(g), len(verts), len(tris)), verts


def vertex_records(T, G, origin, voxel, keys):
    """the vertex of each edge key (g << 3 | d): s = T_a / (T_a - T_b), X = o + h (a + s d) with o, h rounded to float,
    grey = G_a + s (G_b - G_a), all float32"""
    nz, ny, nx = T.shape
    Tf, Gf = T.ravel(), G.ravel()
    keys = np.asarray(keys, np.int64)
    ga, d = keys >> 3, keys & 7
    dx, dy, dz = d & 1, (d >> 1) & 1, (d >> 2) & 1
    gb = ga + dx + nx * (dy + ny * dz)
    s = Tf[ga] / (Tf[ga] - Tf[gb])
    ai, aj, ak = ga % nx, (ga // nx) % ny, ga // (nx * ny)
    h = F32(voxel)
    out = np.zeros((len(keys), 4), F32)
    for c, (a, dd) in enumerate(((ai, dx), (aj, dy), (ak, dz))):
        out[:, c] = F32(origin[c]) + h * (a.astype(F32) + s * dd.astype(F32))
    out[:, 3] = Gf[ga] + s * (Gf[gb] - Gf[ga])
    return out


# ---- mesh checks --------------------------------------------------------------------------------------------------------

def directed_edges(tris):
    t = np.asarray(tris, np.int64)
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def topology(tris, n_vertices):
    """(boundary directed edges: those without their reverse, duplicated directed edges, Euler characteristic V - E + F
    over the referenced vertices)"""
    e = directed_edges(tris)
    n = max(int(n_vertices), 1)
    code = e[:, 0] * n + e[:, 1]
    rev = e[:, 1] * n + e[:, 0]
    uniq, cnt = np.unique(code, return_counts=True)
    dup = int((cnt > 1).sum())
    boundary = e[~np.isin(code, rev)]
    und = np.unique(np.sort(e, 1), axis=0)
    V = len(np.unique(np.asarray(tris).ravel()))
    return boundary, dup, V - len(und) + len(tris)


def signed_volume(X, tris):
    """sum over triangles of det(v0, v1, v2) / 6: the enclosed volume of a closed mesh with outward normals"""
    P = np.asarray(X, np.float64)[np.asarray(tris, np.int64)]
    return float(np.einsum("ij,ij->i", P[:, 0], np.cross(P[:, 1], P[:, 2])).sum() / 6.0)
