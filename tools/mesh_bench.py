"""ps_tsdf_integrate and ps_tsdf_mesh on three workloads:
  A. test_pose's rendered scene, its six true depth maps at 1280 x 960, fused into 512^3 and 768^3 volumes over the
     scene's bounds (the 0.5 / 99.5 percentiles of the back-projected depths), trunc = 3 voxels, then meshed;
  B. 100 synthetic posed 640 x 480 views on a sphere around a 512^3 volume, with a focal length of about three image
     widths, so each sees a small part of it: what the per-block frustum test saves shows as the share of (block, view)
     pairs it skips, counted on the host with the kernel's rule, and as the time per view against A's;
  C. extraction of A's volumes: the call (count call + fill call, as TsdfVolume.mesh) and each kernel.
Calls are timed with CUDA events (median and spread over --reps calls after a warm-up), kernels by torch.profiler in a
separate run.  Prints (grid point, view) updates per second, the (grid point, view) pairs per second, the classification
pass's algorithmic bytes (tsdf and weight, 8 bytes per grid point) against the 3.35 TB/s of the H100 SXM data sheet, and
the card name and power limit read in the same run.

    python tools/mesh_bench.py [--reps N] [out.json]
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from popsift_b200 import api        # noqa: E402

KERNELS = ("ts_integrate_kernel", "ts_count_kernel", "ts_emit_kernel", "radix_hist_kernel", "radix_scatter_kernel", "ts_unique_kernel",
           "ts_unique_compact_kernel", "ts_vertex_kernel", "ts_triangle_kernel", "scan_block_kernel", "scan_add_kernel")
HBM_TBPS = 3.35


def _time(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def _profile(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                per[k] = per.get(k, 0.0) + e.device_time_total / 1000.0
    return per


def _bounds(depths, cams, poses):
    pts = []
    for D, cam, (R, t) in zip(depths, cams, poses):
        h, w = D.shape
        y, x = np.mgrid[0:h:4, 0:w:4].astype(np.float64)
        d = D[::4, ::4].astype(np.float64)
        fx, fy, cx, cy = (float(v) for v in cam)
        Xc = np.stack([(x - cx) / fx * d, (y - cy) / fy * d, d]).reshape(3, -1)
        pts.append((R.T @ (Xc - t[:, None])).T[d.ravel() > 0])
    P = np.concatenate(pts)
    return np.percentile(P, 0.5, 0), np.percentile(P, 99.5, 0)


def _unseen_share(cams, poses, wh, origin, voxel, n):
    """the share of (32 x 4 x 4 block, view) pairs the kernel's frustum test skips (k_mesh.h's rule, in numpy)"""
    w, h = wh
    bi, bj, bk = np.meshgrid(np.arange(0, n, 32), np.arange(0, n, 4), np.arange(0, n, 4), indexing="ij")
    lo = np.stack([bi, bj, bk], -1).reshape(-1, 3)
    hi = np.minimum(lo + [32, 4, 4], n) - 1
    skipped = 0
    for cam, (R, t) in zip(cams, poses):
        code = np.full(len(lo), 31)
        for c in range(8):
            g = np.where([c & 1, c & 2, c & 4], hi, lo)
            X = np.asarray(origin) + voxel * g
            Xc = X @ R.T + t
            with np.errstate(divide="ignore", invalid="ignore"):
                u = cam[0] * Xc[:, 0] / Xc[:, 2] + cam[2]
                v = cam[1] * Xc[:, 1] / Xc[:, 2] + cam[3]
            cc = (Xc[:, 2] > 0) * (1 | 2 * (u < -1.5) | 4 * (u > w + 0.5) | 8 * (v < -1.5) | 16 * (v > h + 0.5))
            code &= cc
        skipped += int(((code & 1) & ((code & 30) > 0)).sum())
    return skipped / (len(lo) * len(cams))


def _integrate(imgs, cams, poses, depths, origin, voxel, n, reps):
    import torch
    dimg = [torch.from_numpy(im).cuda() for im in imgs]
    ddep = [torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda() for d in depths]
    vol = api.TsdfVolume(origin, voxel, (n, n, n))
    rep = vol.integrate(dimg, cams, poses, ddep, trunc=3 * voxel)
    t = _time(lambda: vol.integrate(dimg, cams, poses, ddep, trunc=3 * voxel), reps)
    per = _profile(lambda: vol.integrate(dimg, cams, poses, ddep, trunc=3 * voxel))
    k = per.get("ts_integrate_kernel", float("nan"))
    pairs = n ** 3 * len(imgs)
    out = dict(volume=n, views=len(imgs), voxel=voxel, call_ms=t, kernel_ms=k, ms_per_view=t[0] / len(imgs), report=rep,
               updates_per_s=rep["updates"] / (k / 1e3), pairs_per_s=pairs / (k / 1e3),
               volume_bytes=24 * n ** 3, volume_TBps=24 * n ** 3 / (k / 1e3) / 1e12)
    return out, vol


def _extract(vol, reps):
    n = vol.shape[0]
    # a fresh clear + one integration leaves weight 1 where one view saw: mesh at min_weight 1
    m = vol.mesh()
    t = _time(lambda: vol.mesh(), reps)
    per = _profile(lambda: vol.mesh())
    # the profile covers TsdfVolume.mesh: the count call and the fill call each launch ts_count_kernel and ts_emit_kernel once
    cls = 8 * n ** 3
    cnt = per.get("ts_count_kernel", float("nan")) / 2
    emit = per.get("ts_emit_kernel", float("nan")) / 2
    return dict(volume=n, report=m.report, call_ms=t, kernels_ms_count_and_fill_calls=per,
                fill_call_kernels_ms=sum(per.values()) / 2 + (per.get("ts_vertex_kernel", 0) + per.get("ts_triangle_kernel", 0)) / 2,
                classification_bytes=cls, count_ms=cnt, count_TBps=cls / (cnt / 1e3) / 1e12,
                count_share_of_hbm=cls / (cnt / 1e3) / 1e12 / HBM_TBPS, emit_ms=emit, emit_TBps=cls / (emit / 1e3) / 1e12)


def main():
    reps = 10
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    import test_depth as td
    imgs, cams, poses, truth = td._rendered(1.0)
    depths = [D.astype(np.float32) for D in truth]
    lo, hi = _bounds(depths, cams, poses)
    res = dict(gpu=q.stdout.strip(), rendered={}, extraction={})
    for n in (512, 768):
        voxel = float((hi - lo).max() / (n - 9))
        origin = lo - 4 * voxel
        a, vol = _integrate(imgs, cams, poses, depths, origin, voxel, n, reps)
        a["skipped_block_views"] = _unseen_share(cams, poses, (1280, 960), origin, voxel, n)
        res["rendered"][n] = a
        vol.clear()
        vol.integrate(imgs, cams, poses, depths, trunc=3 * voxel)
        res["extraction"][n] = _extract(vol, reps)
        vol.free()
    # B: 100 posed views around a 512^3 volume
    import test_mesh as tm
    n = 512
    views = list(tm._random_views(0, 100, w=640, h=480, dist=1.1))
    views[1] = [c * np.array([3.0, 3.0, 1.0, 1.0], np.float32) for c in views[1]]
    voxel = 1.0 / (n - 1)
    origin = (-0.5, -0.5, -0.5)
    b, vol = _integrate(views[0], views[1], views[2], views[3], origin, voxel, n, reps)
    vol.free()
    b["skipped_block_views"] = _unseen_share(views[1], views[2], (640, 480), origin, voxel, n)
    res["synthetic_100"] = b
    print(json.dumps(res, indent=1, default=str))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()
