"""ps_triangulate_tracks on an SfM-scale synthetic graph and on the rendered chain, with card name and power limit.

  1. Synthetic: 1 000 posed cameras on a sphere around a point cloud, 2 M tracks, geometric lengths from 2 (p = 0.4) plus a
     tail of 0.1 % tracks of 50 .. 500 members; 0.5 px noise, 10 % outlier observations.  Median ms per call (inputs on the
     device, ending in a synchronise), tracks/s, observation tests/s, kernel time per pass (torch.profiler), and the
     operation and byte counts of the track pass computed here: FP64 operations of its observation tests against the
     34 TFLOP/s FP64 (non-tensor) of the H100 SXM data sheet, and the bytes it must move against 3.35 TB/s.  The same
     graph without its tail, timed in the same run, shows whether the long tracks serialise the grid.
  2. The rendered chain (six 1280 x 960 views of test_pose's scene): kernel time of triangulation next to
     ps_tracks_from_matches and ps_verify_batch in one profiled api.triangulated_tracks call.
  3. Context: the numpy oracle on 2 000 tracks of workload 1, extrapolated to 2 M (labelled as such).

    python tools/triangulate_bench.py [--reps N] [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import triangulate_oracle as tro    # noqa: E402
from popsift_b200 import api        # noqa: E402

# FP64 operations of one observation test (k_triangulate.h tri_error2): R X + t (9 mul, 9 add), 1 / z (1 div), X_c iz
# (2 mul), fx p + cx - x and fy q + cy - y (2 mul, 4 add), e_x^2 + e_y^2 (2 mul, 1 add), the comparison (1)
TEST_FLOPS = 31
PEAK_FP64 = 34e12
PEAK_BW = 3.35e12


def make_graph(rng, n_cams=1000, n_tracks=2_000_000, p=0.4, tail=0.001, noise=0.5, outliers=0.1):
    L = 2 + rng.geometric(p, size=n_tracks) - 1
    n_tail = int(n_tracks * tail)
    tail_idx = rng.choice(n_tracks, size=n_tail, replace=False)
    L[tail_idx] = np.exp(rng.uniform(np.log(50), np.log(500), size=n_tail)).astype(np.int64)
    L = np.minimum(L, n_cams)
    # cameras on a sphere of radius 10 looking at the origin
    c = rng.normal(size=(n_cams, 3)); c *= 10.0 / np.linalg.norm(c, axis=1, keepdims=True)
    z = -c / np.linalg.norm(c, axis=1, keepdims=True)
    up = rng.normal(size=(n_cams, 3))
    x = np.cross(up, z); x /= np.linalg.norm(x, axis=1, keepdims=True)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 1)
    t = -np.einsum("nij,nj->ni", R, c)
    f = rng.uniform(800, 1200, size=n_cams)
    cams = np.stack([f, f, np.full(n_cams, 640.0), np.full(n_cams, 480.0)], 1).astype(np.float32)
    X = rng.normal(scale=1.0, size=(n_tracks, 3))
    # each track's cameras: (c0 + k * stride) mod n_cams with stride coprime to n_cams (distinct), then sorted
    strides = np.array([s for s in range(1, 200) if np.gcd(s, n_cams) == 1])
    track = np.repeat(np.arange(n_tracks), L)
    start = np.concatenate([[0], np.cumsum(L)])
    k = np.arange(len(track)) - start[track]
    c0 = rng.integers(0, n_cams, size=n_tracks)
    st = strides[rng.integers(0, len(strides), size=n_tracks)]
    cam = (c0[track] + k * st[track]) % n_cams
    order = np.lexsort((cam, track))
    cam = cam[order]
    Xc = np.einsum("nij,nj->ni", R[cam], X[track]) + t[cam]
    uv = np.stack([cams[cam, 0] * Xc[:, 0] / Xc[:, 2] + cams[cam, 2], cams[cam, 1] * Xc[:, 1] / Xc[:, 2] + cams[cam, 3]], 1)
    uv += rng.normal(scale=noise, size=uv.shape)
    out = rng.random(len(uv)) < outliers
    uv[out] = rng.uniform([0, 0], [1280, 960], size=(int(out.sum()), 2))
    # features of each camera in observation order; global ids
    by_cam = np.lexsort((np.arange(len(cam)), cam))
    rank = np.empty(len(cam), np.int64)
    rank[by_cam] = np.arange(len(cam))
    n_feat = np.bincount(cam, minlength=n_cams)
    feat = np.zeros(len(cam), api.FEATURE_DTYPE)
    feat["x"], feat["y"] = uv[by_cam, 0], uv[by_cam, 1]
    return dict(n_feat=n_feat, feat=feat, cams=cams, poses=[(R[i], t[i]) for i in range(n_cams)], start=start.astype(np.int32),
                members=rank.astype(np.int32), L=L, tail=np.isin(np.arange(n_tracks), tail_idx), uv=uv, cam=cam)


def hyps(L, ns):
    return np.where(L * (L - 1) // 2 <= ns, L * (L - 1) // 2, ns)


class Device:
    """a graph's inputs on the device and one call of ps_triangulate_tracks"""

    def __init__(self, lib, g, bufs):
        self.lib, self.g = lib, g
        self.n = len(g["n_feat"])
        base = bufs.upload(g["feat"])
        off = np.concatenate([[0], np.cumsum(g["n_feat"])])
        self.c_feat = (C.c_void_p * self.n)(*[base + 72 * int(o) for o in off[:-1]])
        self.c_nf = (C.c_int32 * self.n)(*[int(v) for v in g["n_feat"]])
        self.cams = api._c_cameras(g["cams"])
        self.rig = api._c_rigids(g["poses"])
        self.T, self.M = len(g["start"]) - 1, len(g["members"])
        self.d_st, self.d_mem = bufs.upload(g["start"]), bufs.upload(g["members"])
        self.d_pts, self.d_mask, self.d_err = bufs.alloc(self.T * 40), bufs.alloc(self.M), bufs.alloc(self.M * 4)
        self.cnt = api.PsTriangulateCounts()

    def call(self, prm):
        rc = self.lib.ps_triangulate_tracks(0, self.n, self.c_nf, self.c_feat, self.cams.ctypes.data, self.rig, self.T, self.d_st,
                                            self.d_mem, self.M, C.byref(prm), self.d_pts, self.d_mask, self.d_err, C.byref(self.cnt))
        api._check(self.lib, rc, "ps_triangulate_tracks")


def timed(fn, reps):
    import torch
    fn()
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times)), times


def kernel_ms(fn, prefixes):
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in prefixes}
    for e in prof.key_averages():
        for k, pre in prefixes.items():
            if any(p in e.key for p in pre):
                out[k] += e.device_time_total / 1e3
    return out


def main():
    import torch
    reps = 5
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"card": q.stdout.strip()}
    print("card", res["card"], flush=True)
    torch.zeros(1, device="cuda")
    lib = api.load_library()
    rng = np.random.default_rng(0)
    t0 = time.perf_counter()
    g = make_graph(rng)
    print("graph built in %.1f s" % (time.perf_counter() - t0), flush=True)
    ns = 256
    prm = api._tri_params(max_error=4.0, min_angle=1.5, n_samples=ns, refine_iters=10)
    L = g["L"]
    H = hyps(L, ns)
    tests = float((H * L).sum())
    res["graph"] = {"cameras": 1000, "tracks": int(len(L)), "observations": int(L.sum()), "max_length": int(L.max()),
                    "mean_length": float(L.mean()), "tail_tracks": int(g["tail"].sum()), "hypothesis_tests": tests,
                    "tail_share_of_tests": float((H * L)[g["tail"]].sum() / tests)}
    print(json.dumps(res["graph"]), flush=True)
    bufs = api._DevBuffers(lib)
    try:
        dev = Device(lib, g, bufs)
        ms, times = timed(lambda: dev.call(prm), reps)
        counts = dict(zip(api.TRI_STATUS, [int(v) for v in dev.cnt.n_status]))
        kern = kernel_ms(lambda: dev.call(prm), {"ray": ("tri_ray_kernel",), "track": ("tri_track_kernel",), "count": ("tri_count_kernel",)})
        # the track pass: hypothesis tests plus (refinement, rescoring, outputs) about 2 + 2 refine_iters passes over the
        # members of every track with a point; bytes it must move: start (8 / track), rays (40 / member), records
        # (40 / track), mask and error (5 / member)
        passes = float(L.sum()) * (4 + 2 * 10)
        flops = TEST_FLOPS * (tests + passes)
        byts = 8.0 * len(L) + 45.0 * L.sum() + 40.0 * len(L)
        tr_s = kern["track"] * 1e-3
        res["synthetic"] = {"ms_per_call_median": ms, "ms_all": times, "tracks_per_s": len(L) / (ms * 1e-3),
                            "hypothesis_tests_per_s": tests / (ms * 1e-3), "kernel_ms": kern, "counts": counts,
                            "track_pass_fp64_flops": flops, "track_pass_bytes": byts,
                            "track_pass_fp64_tflops": flops / tr_s / 1e12 if tr_s else None,
                            "track_pass_share_of_34_tflops": flops / tr_s / PEAK_FP64 if tr_s else None,
                            "track_pass_share_of_hbm": byts / tr_s / PEAK_BW if tr_s else None}
        print(json.dumps(res["synthetic"]), flush=True)
    finally:
        bufs.free()
    # the same graph without its tail
    keep = ~g["tail"]
    Lk = L[keep]
    st = np.concatenate([[0], np.cumsum(Lk)]).astype(np.int32)
    idx = np.concatenate([np.arange(g["start"][k], g["start"][k + 1]) for k in np.nonzero(g["tail"])[0]]) if g["tail"].any() else []
    mem = np.delete(g["members"], idx)
    g2 = dict(g, start=st, members=mem)
    bufs = api._DevBuffers(lib)
    try:
        dev2 = Device(lib, g2, bufs)
        ms2, _ = timed(lambda: dev2.call(prm), reps)
        kern2 = kernel_ms(lambda: dev2.call(prm), {"track": ("tri_track_kernel",)})
    finally:
        bufs.free()
    tests2 = float((hyps(Lk, ns) * Lk).sum())
    res["synthetic_without_tail"] = {"ms_per_call_median": ms2, "kernel_ms": kern2, "hypothesis_tests": tests2,
                                     "track_kernel_ratio_with_over_without": kern["track"] / kern2["track"] if kern2["track"] else None,
                                     "test_ratio_with_over_without": tests / tests2}
    print(json.dumps(res["synthetic_without_tail"]), flush=True)
    # the oracle on a subset, extrapolated
    sub = rng.choice(len(L), size=2000, replace=False)
    feats = [np.zeros((0, 2), np.float32)]
    t0 = time.perf_counter()
    for k in sub:
        s0, s1 = g["start"][k], g["start"][k + 1]
        cm = g["cam"][s0:s1]
        uv = g["uv"][s0:s1].astype(np.float32)
        tro.triangulate_track(uv[:, 0], uv[:, 1], g["cams"][cm], np.stack([g["poses"][c][0] for c in cm]),
                              np.stack([g["poses"][c][1] for c in cm]), int(k), 4.0, 1.5, 2, ns, 10, 0)
    dt = time.perf_counter() - t0
    del feats
    res["oracle_extrapolated_s_for_2M_tracks_one_core"] = dt / len(sub) * len(L)
    print("oracle: %.1f ms per track, extrapolated %.0f s for the graph" % (dt / len(sub) * 1e3, res["oracle_extrapolated_s_for_2M_tracks_one_core"]),
          flush=True)
    # the rendered chain
    from test_pose import CAMS, W, H as HH, _cast
    from test_triangulate import VIEWS, _view_pose
    y, x = np.mgrid[0:HH, 0:W].astype(np.float64)
    imgs, cams, poses = [], [], []
    for k, (Rv, Cv) in enumerate(VIEWS):
        R, t = _view_pose(Rv, Cv)
        _, v = _cast(CAMS[k % 2], R, t, x.ravel(), y.ravel())
        imgs.append(np.clip(np.rint(v), 0, 255).astype(np.uint8).reshape(HH, W))
        cams.append(CAMS[k % 2]); poses.append((R, t))
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=W, max_height=HH, slots=1)
    sets = [ps.enqueue(W, HH, im).getDev() for im in imgs]
    pairs = [(i, j) for i in range(len(sets)) for j in range(i + 1, len(sets))]

    def chain():
        return api.triangulated_tracks(sets, pairs, cams, poses, verify=dict(model="fundamental", threshold=2.0, seed=1), max_error=2.0)
    tr, tp = chain()
    kc = kernel_ms(chain, {"verify": ("verify_",), "tracks": ("tracks_", "radix_", "scan_"), "triangulate": ("tri_",)})
    res["rendered_chain"] = {"tracks": int(len(tr.start) - 1), "members": int(len(tr.set)), "counts": tp.counts, "kernel_ms": kc}
    print(json.dumps(res["rendered_chain"]), flush=True)
    ps.uninit()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
