"""The contract of ps_depth_maps and ps_depth_filter (include/popsift_b200_depth.h) in float64 numpy, written from the
header's steps with nothing shared with the device code.  Box sums by integral images, with a count of valid samples
carried beside the sums (a NaN in a cumulative sum would poison everything after it)."""
import numpy as np


def K(cam):
    fx, fy, cx, cy = (float(v) for v in cam)
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


def planes(d_min, d_max, n):
    """step 2: the inverse depths iota_k"""
    i0, i1 = 1.0 / float(d_min), 1.0 / float(d_max)
    return i0 + np.arange(n) * (i1 - i0) / (n - 1)


def warp(cam_r, pose_r, cam_s, pose_s, x, y, z, w_s, h_s):
    """step 3 by the explicit 3-D route: (u, v, valid) of reference pixels (x, y) on the plane z"""
    Rr, tr = (np.asarray(a, np.float64) for a in pose_r)
    Rs, ts = (np.asarray(a, np.float64) for a in pose_s)
    ray = np.linalg.solve(K(cam_r), np.stack([x, y, np.ones_like(x)]).reshape(3, -1))
    X = Rr.T @ (z * ray - tr[:, None])
    Xs = Rs @ X + ts[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        p = K(cam_s) @ Xs
        u, v = p[0] / p[2], p[1] / p[2]
    valid = (Xs[2] > 0) & (u >= 0) & (u <= w_s - 1) & (v >= 0) & (v <= h_s - 1)
    return u.reshape(np.shape(x)), v.reshape(np.shape(x)), valid.reshape(np.shape(x))


def homography(cam_r, pose_r, cam_s, pose_s):
    """the plane-induced map of step 3: (u, v, w) ~ H (x, y, 1) + iota b"""
    Rr, tr = (np.asarray(a, np.float64) for a in pose_r)
    Rs, ts = (np.asarray(a, np.float64) for a in pose_s)
    Rrel = Rs @ Rr.T
    trel = ts - Rrel @ tr
    return K(cam_s) @ Rrel @ np.linalg.inv(K(cam_r)), K(cam_s) @ trel


def bilinear(img, u, v, valid):
    """step 3's sample: the bilinear value at (u, v) with u0 = min(floor(u), w - 2); 0 where not valid"""
    h, w = img.shape
    I = img.astype(np.float64)
    uu, vv = np.where(valid, u, 0.0), np.where(valid, v, 0.0)
    u0 = np.minimum(np.floor(uu), w - 2).astype(np.int64)
    v0 = np.minimum(np.floor(vv), h - 2).astype(np.int64)
    fu, fv = uu - u0, vv - v0
    val = (1 - fv) * ((1 - fu) * I[v0, u0] + fu * I[v0, u0 + 1]) + fv * ((1 - fu) * I[v0 + 1, u0] + fu * I[v0 + 1, u0 + 1])
    return np.where(valid, val, 0.0)


def box(a, r):
    """sum over each (2r+1)^2 window centred at the pixels whose window is inside; zero elsewhere"""
    h, w = a.shape
    S = np.zeros((h + 1, w + 1))
    S[1:, 1:] = np.cumsum(np.cumsum(a, 0), 1)
    d = 2 * r + 1
    out = np.zeros((h, w))
    if h >= d and w >= d:
        out[r:h - r, r:w - r] = S[d:, d:] - S[:-d, d:] - S[d:, :-d] + S[:-d, :-d]
    return out


def candidates(h, w, r):
    c = np.zeros((h, w), bool)
    c[r:h - r, r:w - r] = True
    return c


def ncc(m, A, AA, B, BB, AB, floor_m2):
    """step 5 from the sums: (valid, c)"""
    vr, vs = m * AA - A * A, m * BB - B * B
    ok = (vr > floor_m2) & (vs > floor_m2)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.clip(1.0 - (m * AB - A * B) / np.sqrt(vr * vs), 0.0, 2.0)
    return ok, np.where(ok, c, np.inf)


def aggregate(costs, top_k, min_sources):
    """step 6 on a stack (n_sources, ...) with +inf for invalid sources: (C, n_v)"""
    nv = np.isfinite(costs).sum(0)
    srt = np.sort(costs, 0)
    kk = np.minimum(nv, top_k)
    csum = np.cumsum(np.where(np.isfinite(srt), srt, 0.0), 0)
    idx = np.clip(kk - 1, 0, max(len(costs) - 1, 0))
    s = np.take_along_axis(csum, idx[None], 0)[0] if len(costs) else np.zeros(nv.shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        C = np.where((nv >= min_sources) & (nv > 0), s / np.maximum(kk, 1), np.inf)
    return C, nv


def parabola(cm, c0, cp, k, n):
    """step 8: delta"""
    cm, c0, cp, k = np.broadcast_arrays(np.asarray(cm, np.float64), np.asarray(c0, np.float64), np.asarray(cp, np.float64), k)
    with np.errstate(invalid="ignore"):
        den = cm - 2 * c0 + cp
    ok = (k > 0) & (k < n - 1) & np.isfinite(cm) & np.isfinite(cp) & (den > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.clip((cm - cp) / (2 * den), -0.5, 0.5)
    return np.where(ok, d, 0.0)


def depth_map(ref_img, cam_r, pose_r, sources, d_min, d_max, n_depths=64, radius=3, top_k=3, min_sources=1, max_cost=0.5,
              min_var=1.0, stack=False):
    """Steps 1-9 for one reference.  sources: [(img, cam, pose)].  Returns dict(depth, cost, n_src, k (-1 without a
    winner), C (n, h, w) when stack, valid_var: the pixels whose reference window and every valid source window have
    variance > 1.001 x the floor at k*... (see var_margin))."""
    h, w = ref_img.shape
    r = radius
    m = float((2 * r + 1) ** 2)
    floor_m2 = m * m * float(min_var)
    I = ref_img.astype(np.float64)
    cand = candidates(h, w, r)
    A, AA = box(I, r), box(I * I, r)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    iota = planes(d_min, d_max, n_depths)
    C = np.full((n_depths, h, w), np.inf)
    NV = np.zeros((n_depths, h, w), np.int32)
    VMIN = np.full((n_depths, h, w), np.inf)     # smallest var_s / m^2 over the valid sources
    for k in range(n_depths):
        costs = []
        vmin = np.full((h, w), np.inf)
        for img_s, cam_s, pose_s in sources:
            hs, ws = img_s.shape
            u, v, val = warp(cam_r, pose_r, cam_s, pose_s, x, y, 1.0 / iota[k], ws, hs)
            S = bilinear(img_s, u, v, val)
            n_ok = box(val.astype(np.float64), r)
            B, BB, AB = box(S, r), box(S * S, r), box(I * S, r)
            full = cand & (n_ok == m)
            ok, c = ncc(m, A, AA, B, BB, AB, floor_m2)
            good = full & ok
            costs.append(np.where(good, c, np.inf))
            vmin = np.where(good, np.minimum(vmin, (m * BB - B * B) / (m * m)), vmin)
        Ck, nv = aggregate(np.array(costs) if costs else np.zeros((0, h, w)), top_k, min_sources)
        C[k] = np.where(cand, Ck, np.inf)
        NV[k] = nv
        VMIN[k] = vmin
    has = np.isfinite(C).any(0)
    kstar = np.where(has, np.argmin(C, 0), -1)
    kk = np.maximum(kstar, 0)
    c0 = np.take_along_axis(C, kk[None], 0)[0]
    cm = np.take_along_axis(C, np.maximum(kk - 1, 0)[None], 0)[0]
    cp = np.take_along_axis(C, np.minimum(kk + 1, n_depths - 1)[None], 0)[0]
    delta = parabola(cm, c0, cp, kk, n_depths)
    di = iota[1] - iota[0]
    depth = np.where(has & (c0 <= max_cost), 1.0 / (iota[kk] + delta * di), 0.0)
    out = dict(depth=depth, cost=np.where(has, c0, np.inf), n_src=np.where(has, np.take_along_axis(NV, kk[None], 0)[0], 0),
               k=kstar, iota=iota)
    # the margin of the winner: the second-best cost at least two planes away, minus the best
    far = C.copy()
    for dk in (-1, 0, 1):
        idx = np.clip(kk + dk, 0, n_depths - 1)
        np.put_along_axis(far, idx[None], np.inf, 0)
    with np.errstate(invalid="ignore"):
        out["margin"] = np.where(has, far.min(0) - c0, np.inf)
    vr = (m * AA - A * A) / (m * m)
    out["var_ok"] = cand & (vr >= 1.001 * min_var) & (np.take_along_axis(VMIN, kk[None], 0)[0] >= 1.001 * min_var)
    if stack:
        out["C"] = C
    return out


def backproject(cam, pose, x, y, D):
    R, t = (np.asarray(a, np.float64) for a in pose)
    ray = np.linalg.solve(K(cam), np.stack([x, y, np.ones_like(x)]).reshape(3, -1))
    return R.T @ (np.asarray(D, np.float64).reshape(1, -1) * ray - t[:, None])


def project(cam, pose, X):
    R, t = (np.asarray(a, np.float64) for a in pose)
    Xc = R @ X + t[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        p = K(cam) @ Xc
        return p[0] / p[2], p[1] / p[2], Xc[2]


def depth_filter(depths, images, cams, poses, refs, sources, max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2):
    """ps_depth_filter: (n_consistent maps, points as a list of (X (3,), ref, x, y, n, grey) in (ref, y, x) order)"""
    where = {int(r): j for j, r in enumerate(refs)}
    ncons, pts = [], []
    for j, r in enumerate(refs):
        D = np.asarray(depths[j], np.float64)
        h, w = D.shape
        y, x = np.mgrid[0:h, 0:w]
        xs, ys, Ds = x.ravel().astype(np.float64), y.ravel().astype(np.float64), D.ravel()
        n = np.zeros(h * w, np.int64)
        has = Ds > 0
        X = backproject(cams[r], poses[r], xs, ys, Ds)
        for s in sources[j]:
            if int(s) not in where:
                continue
            js = where[int(s)]
            Dm = np.asarray(depths[js], np.float64)
            hs, ws = Dm.shape
            u, v, zs = project(cams[s], poses[s], X)
            ok = has & (zs > 0) & (u >= 0) & (u <= ws - 1) & (v >= 0) & (v <= hs - 1)
            qx = np.where(ok, np.floor(np.where(ok, u, 0) + 0.5), 0).astype(np.int64)
            qy = np.where(ok, np.floor(np.where(ok, v, 0) + 0.5), 0).astype(np.int64)
            Dq = np.where(ok, Dm[qy, qx], 0.0)
            ok &= Dq > 0
            X2 = backproject(cams[s], poses[s], qx.astype(np.float64), qy.astype(np.float64), np.where(ok, Dq, 1.0))
            pu, pv, zr = project(cams[r], poses[r], X2)
            with np.errstate(invalid="ignore"):
                ok &= (zr > 0) & (np.hypot(pu - xs, pv - ys) <= max_reproj_error) & (np.abs(zs - Dq) <= max_depth_diff * Dq)
            n += ok
        nc = np.minimum(n, 255).astype(np.uint8)
        ncons.append(nc.reshape(h, w))
        for i in np.flatnonzero(nc >= min_consistent):
            pts.append((X[:, i], j, int(xs[i]), int(ys[i]), int(nc[i]), int(images[r][int(ys[i]), int(xs[i])])))
    return ncons, pts
