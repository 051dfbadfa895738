"""ps_two_view_config_batch on 240 planted pairs of about 2 000 correspondences (pose_bench.py's size): a quarter general
3-D scenes with 50 % inliers, a quarter single planes with parallax, a quarter pure rotations, a quarter general scenes
again, so that steps 3 and 4 run on half of the pairs.  The three RANSACs (ps_verify_batch H and F, ps_relative_pose_batch,
1 024 samples) run once on device-resident rows; the new call is then timed alone with CUDA events around each call
(median over --reps), and its two kernels with torch.profiler in a separate run.  Prints the configurations found, the
card name and power limit.

    python tools/twoview_bench.py [--reps N] [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pose_oracle as po            # noqa: E402
import twoview_oracle as tvo        # noqa: E402
from popsift_b200 import api        # noqa: E402

KERNELS = ("tv_config_kernel", "tv_median_kernel")


def main():
    import torch
    reps = 20
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rng = np.random.default_rng(0)
    sc = []
    for p in range(240):
        n = int(rng.integers(1800, 2200))
        kind = p % 4
        if kind == 1:
            c, cams = tvo.planted_plane(rng, n, 0.5, 0.3)[:2]
        elif kind == 2:
            c, cams = tvo.planted_plane(rng, n, 0.5, 0.3, rotation_only=True)[:2]
        else:
            c, cams = po.planted_pose(rng, n, 0.5, 0.3)[:2]
        sc.append((c, cams))
    corrs = [s[0] for s in sc]
    cams = api._c_cameras(np.asarray([s[1] for s in sc], np.float32))
    n_corr = np.array([len(c) for c in corrs], np.int32)
    start = np.concatenate([[0], np.cumsum(n_corr)])[:len(corrs)].astype(np.int32)
    rows = int(n_corr.sum())
    res = {"card": q.stdout.strip(), "pairs": len(corrs), "rows": rows}
    lib = api.load_library()
    bufs = api._DevBuffers(lib)
    try:
        d_corr = bufs.upload(np.concatenate(corrs))
        P = len(corrs)
        pprm = api._pose_params(2.0, 1024, 0, True)
        cprm = api._two_view_config_params(2.0)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def timed(fn):
            torch.cuda.synchronize()
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1])

        # the three RANSACs once, each timed
        d_h, d_hn, d_hm = bufs.alloc(P * 36), bufs.alloc(P * 4), bufs.alloc(rows)
        d_f, d_fn, d_fm = bufs.alloc(P * 36), bufs.alloc(P * 4), bufs.alloc(rows)
        d_e, d_em = bufs.alloc(P * 128), bufs.alloc(rows)
        d_out, d_mask, d_pts = bufs.alloc(P * 128), bufs.alloc(rows), bufs.alloc(rows * 16)
        st, nc = start.ctypes.data, n_corr.ctypes.data
        ransac = {}
        for name, model, dm, dn, dk in (("verify_h", 0, d_h, d_hn, d_hm), ("verify_f", 1, d_f, d_fn, d_fm)):
            vp = api.PsVerifyParams(model, 1024, 2.0, 1, 0)
            ransac[name] = timed(lambda: api._check(lib, lib.ps_verify_batch(0, P, d_corr, st, nc, C.byref(vp), dm, dn, dk, None), name))
        ransac["relative_pose"] = timed(lambda: api._check(lib, lib.ps_relative_pose_batch(0, P, d_corr, st, nc, cams.ctypes.data,
                                                                                          C.byref(pprm), d_e, d_em, None, None), "pose"))
        info = np.zeros(P, api.TWO_VIEW_INFO_DTYPE)

        def config(points):
            api._check(lib, lib.ps_two_view_config_batch(0, P, d_corr, st, nc, cams.ctypes.data, d_e, d_em, d_fn, d_h, d_hm, C.byref(cprm),
                                                         d_out, d_mask, d_pts if points else None, info.ctypes.data), "config")

        for points in (False, True):
            config(points)      # warm-up
            t = [timed(lambda: config(points)) for _ in range(reps)]
            res["config_ms_median" + ("_points" if points else "")] = float(np.median(t))
            res["config_ms_spread" + ("_points" if points else "")] = [float(np.min(t)), float(np.max(t))]
        res["ransac_ms"] = ransac
        res["configs"] = {name: int((info["config"] == k).sum()) for k, name in enumerate(api.TV_CONFIG)}
        res["configs_by_planted_kind"] = {kind: {name: int((info["config"][i::4] == k).sum()) for k, name in enumerate(api.TV_CONFIG)}
                                          for i, kind in enumerate(("general", "planar", "panoramic", "general2"))}
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                config(True)
            torch.cuda.synchronize()
        kt = {k: 0.0 for k in KERNELS}
        for e in prof.key_averages():
            for k in KERNELS:
                if k in e.key:
                    kt[k] += e.device_time_total / 1e3 / 5
        res["kernel_ms"] = kt
    finally:
        bufs.free()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
