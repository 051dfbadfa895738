"""ps_relative_pose_batch on 240 planted calibrated pairs of about 2 000 correspondences with 50 % inliers (the pair
count and size of verify_bench.py), at 1 024 and 4 096 samples: median ms per call and per stage (torch.profiler kernel
times), the fraction of valid hypothesis slots, the FP32 rate of the scoring (33 flops per Sampson test, as
verify_bench.py counts) against the 67 TFLOP/s of the H100 SXM data sheet, card name and power limit; cv2's
findEssentialMat + recoverPose per pair on one core as context.

    python tools/pose_bench.py [--reps N] [out.json]
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
import pose_oracle as po            # noqa: E402
from popsift_b200 import api        # noqa: E402

STAGES = {"calibrate": ("pose_calibrate_kernel",), "solve": ("pose_solve_kernel",),
          "score": ("pose_compact_kernel", "pose_score_kernel"), "select_pose": ("pose_select_kernel",)}


def main():
    import torch
    reps = 5
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    rng = np.random.default_rng(0)
    sc = [po.planted_pose(rng, int(rng.integers(1800, 2200)), 0.5, 0.3) for _ in range(240)]
    corrs, cams = [s[0] for s in sc], [s[1] for s in sc]
    res = {"card": q.stdout.strip(), "pairs": 240, "rows": int(sum(len(c) for c in corrs))}
    for ns in (1024, 4096):
        r, (tc, _) = api.relative_pose_correspondences(corrs, cams, threshold=2.0, n_samples=ns, taps=True)
        valid = float((tc >= 0).mean())
        tests = float(sum(int((tc[p] >= 0).sum()) * len(corrs[p]) for p in range(len(corrs))))
        rot = max(po.rot_angle(x.R, s[2]) for x, s in zip(r, sc))
        times = []
        for _ in range(reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            api.relative_pose_correspondences(corrs, cams, threshold=2.0, n_samples=ns)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            api.relative_pose_correspondences(corrs, cams, threshold=2.0, n_samples=ns)
            torch.cuda.synchronize()
        stage = {k: 0.0 for k in STAGES}
        for e in prof.key_averages():
            for k, names in STAGES.items():
                if any(n in e.key for n in names):
                    stage[k] += e.device_time_total / 1e3
        score_ms = stage["score"]
        res["n%d" % ns] = {"ms_call_median_incl_h2d_d2h": float(np.median(times[1:])), "stage_ms": stage, "valid_slot_fraction": valid,
                           "score_tflops": 33 * tests / (score_ms * 1e-3) / 1e12 if score_ms > 0 else None,
                           "score_share_of_67": 33 * tests / (score_ms * 1e-3) / 67e12 if score_ms > 0 else None,
                           "worst_rotation_error_deg": rot}
        print(ns, json.dumps(res["n%d" % ns]), flush=True)
    try:
        import cv2
        t0 = time.perf_counter()
        for c, (kl, kr) in zip(corrs[:24], cams[:24]):
            xl = (c[:, :2] - kl[2:]) / kl[:2]; xr = (c[:, 2:] - kr[2:]) / kr[:2]
            E, m = cv2.findEssentialMat(xl.astype(np.float64), xr.astype(np.float64), np.eye(3), cv2.RANSAC, 0.999,
                                        2.0 / float(np.mean([kl[0], kl[1], kr[0], kr[1]])), maxIters=1024)
            cv2.recoverPose(E[:3], xl.astype(np.float64), xr.astype(np.float64), np.eye(3), mask=m)
        res["cv2_ms_per_pair_1024"] = (time.perf_counter() - t0) * 1e3 / 24
    except ImportError:
        res["cv2_ms_per_pair_1024"] = None
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
