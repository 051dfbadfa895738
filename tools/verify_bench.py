#!/usr/bin/env python
"""Times geometric verification on the GPU: 16 seeded affine views (synth.affine_warp) of one 1920x1080 make_frame, so that
pairs share content, extracted under MatchingMode; all 240 ordered pairs matched with ps_match_batch and turned into
correspondences with ps_match_correspondences; then ps_verify_batch with a homography (1024 samples) and a fundamental
matrix (4096 samples).

    python tools/verify_bench.py [--reps N] [out.json]

Reports the median ms per call after a warm-up (host clock around calls that end in a device synchronise), the gather's
time, the achieved FP32 rate of the scoring (error evaluations counted from shapes: n_corr x k x n_samples per pair, FMA =
2 flops) against the 67 TFLOP/s FP32 of the H100 SXM data sheet, the card name and power limit read in the same run, and,
as context, cv2.findHomography / cv2.findFundamentalMat (RANSAC, same threshold, maxIters = the same sample count,
confidence 1 - 1e-9 so that they rarely stop before the cap) per pair on one CPU core, on the same correspondences."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import affine_warp, make_frame  # noqa: E402

FP32_SHEET = 67.0               # H100 SXM data sheet, TFLOP/s FP32 (700 W)
FLOPS_PER_EVAL = {0: 21, 1: 33}  # the inlier tests of k_verify.cu (inlier_h / inlier_f), FMA = 2
CV2_CONFIDENCE = 1.0 - 1e-9      # OpenCV refuses 1.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [v.strip() for v in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # noqa: BLE001 -- the numbers are still worth printing
        return {"error": str(e)}


def views(n=16, w=1920, h=1080, seed=3):
    base = make_frame(w, h, seed)
    rng = np.random.default_rng(seed)
    cx, cy = (w - 1) / 2, (h - 1) / 2
    out = [base]
    for _ in range(n - 1):
        th, sc = np.deg2rad(rng.uniform(-12, 12)), rng.uniform(0.85, 1.15)
        L = sc * np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.array([[1, rng.uniform(-0.1, 0.1)], [0, 1]])
        t = np.array([cx, cy]) - L @ np.array([cx, cy]) + rng.uniform(-40, 40, 2)
        out.append(affine_warp(base, np.hstack([L, t[:, None]])))
    return out


def median_ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), [round(v, 4) for v in ts]


def main():
    args = sys.argv[1:]
    reps = 20
    if "--reps" in args:
        i = args.index("--reps")
        reps = int(args[i + 1])
        del args[i:i + 2]
    out_path = args[0] if args else None
    info = {"card": card()}
    lib = api.load_library()
    w, h = 1920, 1080
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    sets = [ps.enqueue(w, h, im).getDev() for im in views()]
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    counts = [s.getDescriptorCount() for s in sets]
    rows = sum(counts[l] for l, _ in pairs)
    bufs = api._DevBuffers(lib)
    try:
        d_match = bufs.alloc(rows * 12)
        c_pairs = (C.c_int32 * (2 * len(pairs)))(*[v for pq in pairs for v in pq])
        c_n = (C.c_int32 * len(sets))(*counts)
        c_sets = (C.c_void_p * len(sets))(*[s.getDescriptors() for s in sets])
        assert lib.ps_match_batch(0, len(sets), c_sets, c_n, len(pairs), c_pairs, d_match, 0) == 0
        d_corr, d_src = bufs.alloc(rows * 16), bufs.alloc(rows * 4)
        n_corr = np.zeros(len(pairs), np.int32)
        c_feat = (C.c_void_p * len(sets))(*[s.getFeatures() for s in sets])
        c_rev = (C.c_void_p * len(sets))(*[s.getReverseMap() for s in sets])

        def gather():
            rc = lib.ps_match_correspondences(0, len(sets), c_feat, c_rev, c_n, len(pairs), c_pairs, d_match, d_corr, d_src,
                                              n_corr.ctypes.data)
            assert rc == 0, rc
        info["gather_ms"], info["gather_ms_all"] = median_ms(gather, reps)
        start = np.concatenate([[0], np.cumsum([counts[l] for l, _ in pairs])])[:-1].astype(np.int32)
        info.update(frames=len(sets), pairs=len(pairs), descriptors=int(sum(counts)), match_rows=int(rows),
                    correspondences=int(n_corr.sum()), corr_per_pair_median=float(np.median(n_corr)))
        corr_host = np.zeros((rows, 4), np.float32)
        lib.ps_dev_to_host(corr_host.ctypes.data, d_corr, corr_host.nbytes)
        d_models, d_n, d_mask = bufs.alloc(len(pairs) * 36), bufs.alloc(len(pairs) * 4), bufs.alloc(rows)
        for model, ns, name in ((0, 1024, "homography"), (1, 4096, "fundamental")):
            prm = api._verify_params(model, 4.0, ns, 0, True)

            def verify():
                rc = lib.ps_verify_batch(0, len(pairs), d_corr, start.ctypes.data, n_corr.ctypes.data, C.byref(prm), d_models, d_n, d_mask, None)
                assert rc == 0, rc
            ms, all_ms = median_ms(verify, reps)
            k = 1 if model == 0 else 3
            m = 4 if model == 0 else 7
            evals = float(sum(int(n) for n in n_corr if n >= m)) * k * ns
            n_in = np.zeros(len(pairs), np.int32)
            lib.ps_dev_to_host(n_in.ctypes.data, d_n, n_in.nbytes)
            r = {"n_samples": ns, "ms": ms, "ms_all": all_ms, "error_evaluations": evals,
                 "fp32_tflops": evals * FLOPS_PER_EVAL[model] / (ms * 1e-3) / 1e12,
                 "inlier_fraction_median": float(np.median(n_in / np.maximum(n_corr, 1)))}
            r["fp32_fraction_of_sheet"] = r["fp32_tflops"] / FP32_SHEET
            # context: OpenCV's RANSAC on one CPU core, same correspondences, same iteration cap
            try:
                import cv2
                cv2.setNumThreads(1)
                sel = list(range(0, len(pairs), max(1, len(pairs) // 24)))
                t0 = time.perf_counter()
                for p in sel:
                    c = corr_host[start[p]:start[p] + n_corr[p]]
                    if len(c) < 8:
                        continue
                    if model == 0:
                        cv2.findHomography(c[:, :2], c[:, 2:], cv2.RANSAC, 4.0, maxIters=ns, confidence=CV2_CONFIDENCE)
                    else:
                        cv2.findFundamentalMat(c[:, :2], c[:, 2:], cv2.FM_RANSAC, 4.0, CV2_CONFIDENCE, ns)
                r["cv2_ms_per_pair_one_core"] = (time.perf_counter() - t0) * 1e3 / len(sel)
                r["cv2_pairs_timed"] = len(sel)
            except ImportError:
                r["cv2_ms_per_pair_one_core"] = None
            info[name] = r
    finally:
        bufs.free()
        ps.uninit()
    info["card_after"] = card()
    line = json.dumps(info)
    print(line)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
