#!/usr/bin/env python
"""Times the brute-force matcher (ps_match) on the descriptors of two 4K benchmark frames and reports its tensor-core
roofline: 3 tf32 products x 2 x n_left x n_right x 128 flops per call against the measured bf16 peak of
MEASURED_PEAKS.json (tf32 runs at half the bf16 rate on this part).

    python tools/match_bench.py [out.json]

Also writes the two frames as PGMs next to the JSON when `--pgm DIR` is given, so that the same pair can be fed to the
reference (`ref_dump --match`, timed under ncu: its compute_distance kernel is the like-for-like number)."""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import write_pgm  # noqa: E402


def main():
    import torch
    args = sys.argv[1:]
    pgm_dir = None
    if "--pgm" in args:
        i = args.index("--pgm"); pgm_dir = args[i + 1]; del args[i:i + 2]
    out = args[0] if args else None
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
        for _ in range(3):
            L.ps_match(0, fds[0].getDescriptors(), nl, fds[1].getDescriptors(), nr, d_out, flag)
        ts = []
        for _ in range(10):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            L.ps_match(0, fds[0].getDescriptors(), nl, fds[1].getDescriptors(), nr, d_out, flag)
            b.record(); b.synchronize()
            ts.append(a.elapsed_time(b))
        res[name + "_ms"] = float(np.median(ts))
    m_t = fds[0].match(fds[1], api.FeaturesDev.MATCH_TENSOR)
    m_e = fds[0].match(fds[1], api.FeaturesDev.MATCH_EXACT)
    res["rows_differing_tensor_vs_exact"] = int((m_t != m_e).any(1).sum())
    res["accepted"] = int(m_e[:, 2].sum())
    flops = 3 * 2.0 * nl * nr * 128
    res["tensor_tflops"] = flops / (res["tensor_ms"] * 1e-3) / 1e12
    res["useful_tflops"] = res["tensor_tflops"] / 3          # one fp32-accurate product per three tf32 products
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    bf16 = float(json.load(open(peaks))["bf16_tflops"]) if os.path.exists(peaks) else 1658.3
    res["roofline"] = {"bound": "tensor", "achieved": res["tensor_tflops"], "peak": bf16 / 2, "unit": "TFLOP/s",
                       "frac": res["tensor_tflops"] / (bf16 / 2),
                       "peak_source": "MEASURED_PEAKS.json bf16_tflops / 2 (tf32 issues at half the bf16 rate)",
                       "note": "whole ps_match call (split + wgmma pass + re-rank, one CTA per 128 left descriptors: %d CTAs)" % ((nl + 127) // 128)}
    L.ps_dev_free(d_out)
    pm.uninit()
    print(json.dumps(res))
    if out:
        json.dump(res, open(out, "w"), indent=1)


if __name__ == "__main__":
    main()
