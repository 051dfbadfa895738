"""ps_depth_maps and ps_depth_filter on two workloads:
  A. test_pose's rendered scene, its six views at 1280 x 960 as references, each with the other five as sources, 192
     planes, r = 3, top_k = 3 (the true depth ranges widened x0.8 / x1.25);
  B. 20 synthetic 1920 x 1080 references (smoothed noise), 5 sources each among 25 images, 192 planes.
Each call is timed with CUDA events (median and spread over --reps calls after a warm-up), then the sweep and filter kernels
by torch.profiler in a separate run.  Prints ms per reference, (pixel, plane, source) evaluations per second, the
sweep's algorithmic bytes (the u8 gathers L2 serves: four bytes per bilinear sample of the halo tile; HBM: the images
and the 9-byte outputs), the accuracy of A against the truth, the card name and power limit, and the float64 oracle on
one core for one 160 x 120 reference as context.

    python tools/depth_bench.py [--reps N] [out.json]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from popsift_b200 import api        # noqa: E402

KERNELS = ("dp_sweep_kernel", "dp_filter_kernel", "dp_compact_kernel", "scan_block_kernel", "scan_add_kernel")
N_DEPTHS, R = 192, 3


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


def _profile(fn, out_dir, tag):
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
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "depth_%s.pt.trace.json" % tag))
    return per


def _bytes(shapes, n_src, r=R):
    """the sweep's gathers (4 bytes per bilinear sample of each 32 x 16 tile's halo, per plane and source) and its HBM
    traffic (each reference and source image once per reference, the outputs)"""
    l2 = hbm = 0
    for (h, w), ns in zip(shapes, n_src):
        tiles = -(-w // 32) * -(-h // 16)
        l2 += tiles * (32 + 2 * r) * (16 + 2 * r) * 4 * N_DEPTHS * ns
        hbm += w * h * (1 + ns) + w * h * 9
    return l2, hbm


def _run(imgs, cams, poses, refs, sources, ranges, reps, out_dir, tag):
    import torch
    dev = [torch.from_numpy(im).cuda() for im in imgs]
    fprm = dict(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2)
    kw = dict(n_depths=N_DEPTHS, radius=R, top_k=3, max_cost=0.5)
    res = api.depth_maps(dev, cams, poses, refs, sources, ranges, filter=fprm, **kw)
    t_maps = _time(lambda: api.depth_maps(dev, cams, poses, refs, sources, ranges, **kw), reps)
    t_both = _time(lambda: api.depth_maps(dev, cams, poses, refs, sources, ranges, filter=fprm, **kw), reps)
    per = _profile(lambda: api.depth_maps(dev, cams, poses, refs, sources, ranges, filter=fprm, **kw), out_dir, tag)
    shapes = [imgs[r].shape for r in refs]
    n_src = [len(s) for s in sources]
    evals = sum(h * w * N_DEPTHS * ns for (h, w), ns in zip(shapes, n_src))
    l2, hbm = _bytes(shapes, n_src)
    sweep = per.get("dp_sweep_kernel", float("nan"))
    out = dict(refs=len(refs), size=list(shapes[0]), planes=N_DEPTHS, sources=n_src[0], call_ms=t_maps, call_with_filter_ms=t_both,
               ms_per_ref=t_maps[0] / len(refs), kernels_ms=per, evals=evals, evals_per_s=evals / (sweep / 1e3),
               sweep_gather_bytes=l2, sweep_gather_TBps=l2 / (sweep / 1e3) / 1e12, sweep_hbm_bytes=hbm,
               sweep_hbm_TBps=hbm / (sweep / 1e3) / 1e12, report=res.report, filter_report=res.filter_report)
    return out, res


def main():
    reps = 10
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    out_dir = os.path.dirname(os.path.abspath(out_path)) if out_path else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    import test_depth as td
    # A: the rendered views at full size
    imgs, cams, poses, truth = td._rendered(1.0)
    refs = list(range(6))
    sources = [[s for s in range(6) if s != r] for r in refs]
    ranges = [td._true_range(truth[r]) for r in refs]
    a, res = _run(imgs, cams, poses, refs, sources, ranges, reps, out_dir, "rendered")
    rel = np.concatenate([np.abs(res.depth[j][res.depth[j] > 0] / truth[r][res.depth[j] > 0] - 1) for j, r in enumerate(refs)])
    a["accuracy"] = dict(with_depth=float(np.mean([(d > 0).mean() for d in res.depth])), median=float(np.median(rel)),
                         p90=float(np.percentile(rel, 90)), above_5pct=float((rel > 0.05).mean()))
    # B: 20 synthetic 1920 x 1080 references
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(0)
    n = 25
    simgs = []
    for _ in range(n):
        x = gaussian_filter(rng.normal(size=(1080, 1920)).astype(np.float32), 1.0)
        simgs.append(np.clip(np.rint(x / x.std() * 50 + 128), 0, 255).astype(np.uint8))
    scams = [np.array([1500.0, 1500.0, 960.0, 540.0], np.float32)] * n
    sposes = [(np.eye(3), np.array([0.05 * k, 0.01 * (k % 3), 0.0])) for k in range(n)]
    srefs = list(range(20))
    ssrc = [[(r + d) % n for d in (1, 2, 3, 4, 5)] for r in srefs]
    b, _ = _run(simgs, scams, sposes, srefs, ssrc, [(2.0, 50.0)] * 20, reps, out_dir, "synthetic")
    # the float64 oracle on one core, one 160 x 120 reference with five sources and 32 planes, as context
    import depth_oracle as do
    s_imgs, s_cams, s_poses, s_truth = td._rendered(0.125)
    t0 = time.perf_counter()
    do.depth_map(s_imgs[0], s_cams[0], s_poses[0], [(s_imgs[k], s_cams[k], s_poses[k]) for k in range(1, 6)],
                 *td._true_range(s_truth[0]), n_depths=32, radius=R, top_k=3)
    t_or = time.perf_counter() - t0
    result = dict(gpu=q.stdout.strip(), rendered=a, synthetic=b,
                  oracle_context=dict(size=[120, 160], planes=32, sources=5, s=t_or, evals_per_s=120 * 160 * 32 * 5 / t_or))
    print(json.dumps(result, indent=1))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
