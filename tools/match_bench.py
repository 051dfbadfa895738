#!/usr/bin/env python
"""Times the brute-force matcher on the GPU and reports its tensor-core roofline: 3 tf32 products x 2 x n_left x n_right
x 128 flops per pair against dense TF32 (the measured bf16 peak of MEASURED_PEAKS.json / 2 when present, else the
H100 SXM data sheet's 989 TFLOP/s dense BF16 / 2 = 495 TFLOP/s).

    python tools/match_bench.py [out.json]              ps_match on the descriptors of two 4K benchmark frames
    python tools/match_bench.py --batch N [out.json]    N 1920x1080 frames, all N (N - 1) ordered pairs: a Python loop of
                                                        ps_match against one ps_match_batch call

Every result records the card name, power limit and maximum SM clock (nvidia-smi).  Set POPSIFT_B200_LIB to time
another build of the library (the 4K leg only needs ps_match).

Also writes the two 4K frames as PGMs when `--pgm DIR` is given, so that the same pair can be fed to the reference
(`ref_dump --match`, timed under ncu: its compute_distance kernel is the like-for-like number)."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import make_frame, write_pgm  # noqa: E402

TF32_DENSE_SHEET = 989.0 / 2        # H100 SXM data sheet: 989 TFLOP/s dense BF16; tf32 issues at half that rate


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [v.strip() for v in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # noqa: BLE001 -- the numbers are still worth printing
        return {"error": str(e)}


def tf32_peak():
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks):
        return float(json.load(open(peaks))["bf16_tflops"]) / 2, "MEASURED_PEAKS.json bf16_tflops / 2 (tf32 issues at half the bf16 rate)"
    return TF32_DENSE_SHEET, "H100 SXM data sheet, 989 TFLOP/s dense BF16 / 2"


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()                                    # ends in a synchronisation (ps_match / ps_match_batch return when done)
        b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def four_k(pgm_dir):
    frames = bench.synth_frames(2, 0)
    if pgm_dir:
        os.makedirs(pgm_dir, exist_ok=True)
        for k, f in enumerate(frames):
            write_pgm(os.path.join(pgm_dir, "m%d.pgm" % k), f)
    cfg = api.Config()
    cfg.setOctaves(bench.OCTAVES); cfg.setLevels(bench.LEVELS)
    pm = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=bench.W, max_height=bench.H, slots=2)
    fds = [pm.enqueue(bench.W, bench.H, f).getDev() for f in frames]
    nl, nr = fds[0].getDescriptorCount(), fds[1].getDescriptorCount()
    L = api.load_library()
    d_out = L.ps_dev_alloc(12 * nl)
    res = {"n_left": nl, "n_right": nr}
    for name, flag in (("tensor", api.FeaturesDev.MATCH_TENSOR), ("exact", api.FeaturesDev.MATCH_EXACT)):
        call = lambda: L.ps_match(0, fds[0].getDescriptors(), nl, fds[1].getDescriptors(), nr, d_out, flag)  # noqa: E731
        for _ in range(3):
            call()
        ts = timed(call, 10)
        res[name + "_ms"] = float(np.median(ts))
        res[name + "_ms_min_max"] = [float(min(ts)), float(max(ts))]
    m_t = fds[0].match(fds[1], api.FeaturesDev.MATCH_TENSOR)
    m_e = fds[0].match(fds[1], api.FeaturesDev.MATCH_EXACT)
    res["rows_differing_tensor_vs_exact"] = int((m_t != m_e).any(1).sum())
    res["accepted"] = int(m_e[:, 2].sum())
    flops = 3 * 2.0 * nl * nr * 128
    res["tensor_tflops"] = flops / (res["tensor_ms"] * 1e-3) / 1e12
    res["useful_tflops"] = res["tensor_tflops"] / 3          # one fp32-accurate product per three tf32 products
    peak, src = tf32_peak()
    res["roofline"] = {"bound": "tensor", "achieved": res["tensor_tflops"], "peak": peak, "unit": "TFLOP/s",
                       "frac": res["tensor_tflops"] / peak, "peak_source": src,
                       "note": "whole ps_match call (split + wgmma pass + re-rank)"}
    L.ps_dev_free(d_out)
    pm.uninit()
    return res


def batch(n):
    w, h = 1920, 1080
    cfg = api.Config()
    pm = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=2)
    fds = [pm.enqueue(w, h, make_frame(w, h, 100 + k)).getDev() for k in range(n)]
    counts = [fd.getDescriptorCount() for fd in fds]
    pairs = [(i, j) for i in range(n) for j in range(n) if i != j]
    L = api.load_library()
    rows = sum(counts[i] for i, _ in pairs)
    d_out = L.ps_dev_alloc(12 * max(rows, 1))
    offs = np.concatenate([[0], np.cumsum([counts[i] for i, _ in pairs])]).astype(np.int64)
    ptrs = [fd.getDescriptors() for fd in fds]
    flag = api.FeaturesDev.MATCH_AUTO

    def loop():
        for p, (i, j) in enumerate(pairs):
            L.ps_match(0, ptrs[i], counts[i], ptrs[j], counts[j], C.c_void_p(d_out + 12 * int(offs[p])), flag)
    c_sets = (C.c_void_p * n)(*ptrs)
    c_n = (C.c_int32 * n)(*counts)
    c_pairs = (C.c_int32 * (2 * len(pairs)))(*[v for pq in pairs for v in pq])

    def one_call():
        rc = L.ps_match_batch(0, n, c_sets, c_n, len(pairs), c_pairs, d_out, flag)
        assert rc == 0, L.ps_last_error(None)
    res = {"frames": n, "size": "%dx%d" % (w, h), "pairs": len(pairs), "descriptors_per_frame_mean": float(np.mean(counts)),
           "descriptors_per_frame_min_max": [int(min(counts)), int(max(counts))]}
    flops = 3 * 2.0 * 128 * sum(counts[i] * counts[j] for i, j in pairs)
    peak, src = tf32_peak()
    outs = {}
    for name, fn in (("loop_ps_match", loop), ("ps_match_batch", one_call)):
        fn()                                    # warm-up of the same shapes
        ts = timed(fn, 5)
        ms = float(np.median(ts))
        res[name] = {"ms": ms, "ms_min_max": [float(min(ts)), float(max(ts))], "pairs_per_s": len(pairs) / (ms * 1e-3),
                     "tf32_tflops": flops / (ms * 1e-3) / 1e12, "frac_of_dense_tf32": flops / (ms * 1e-3) / 1e12 / peak}
        out = np.zeros((rows, 3), np.int32)
        L.ps_dev_to_host(out.ctypes.data, d_out, out.nbytes)
        outs[name] = out
    res["rows_differing_batch_vs_loop"] = int((outs["loop_ps_match"] != outs["ps_match_batch"]).any(1).sum())
    res["speedup"] = res["loop_ps_match"]["ms"] / res["ps_match_batch"]["ms"]
    res["peak"] = {"tf32_tflops": peak, "source": src}
    L.ps_dev_free(d_out)
    pm.uninit()
    return res


def main():
    args = sys.argv[1:]
    pgm_dir, n_batch = None, 0
    if "--pgm" in args:
        i = args.index("--pgm"); pgm_dir = args[i + 1]; del args[i:i + 2]
    if "--batch" in args:
        i = args.index("--batch"); n_batch = int(args[i + 1]); del args[i:i + 2]
    out = args[0] if args else None
    res = batch(n_batch) if n_batch else four_k(pgm_dir)
    res["card"] = card()
    res["library"] = api.LIB_PATH
    print(json.dumps(res))
    if out:
        json.dump(res, open(out, "w"), indent=1)


if __name__ == "__main__":
    main()
