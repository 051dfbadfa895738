#!/usr/bin/env python
"""Times the brute-force matcher on the GPU and reports its tensor-core roofline: 3 tf32 products x 2 x n_left x n_right
x 128 flops per pair against dense TF32 (the measured bf16 peak of MEASURED_PEAKS.json / 2 when present, else the
H100 SXM data sheet's 989 TFLOP/s dense BF16 / 2 = 495 TFLOP/s).

    python tools/match_bench.py [out.json]              ps_match on the descriptors of two 4K benchmark frames
    python tools/match_bench.py --batch N [out.json]    N 1920x1080 frames, all N (N - 1) ordered pairs: a Python loop of
                                                        ps_match against one ps_match_batch call

    python tools/match_bench.py --u8 [--batch N] [out.json]
                                                        the same workloads extracted with norm_multi = 9 and quantised
                                                        with ps_descriptors_to_u8: ps_match_u8_batch against the float
                                                        ps_match_batch on the same frames, alternating.  Integer TOPS count
                                                        2 x 128 x n_left x n_right per pair against dense INT8
                                                        (MEASURED_PEAKS.json int8_tops when present, else the H100 SXM data
                                                        sheet's 1979 TOPS)

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
INT8_DENSE_SHEET = 1979.0           # H100 SXM data sheet: 1979 TOPS dense INT8


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


def int8_peak():
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks):
        v = json.load(open(peaks)).get("int8_tops")
        if v:
            return float(v), "MEASURED_PEAKS.json int8_tops"
    return INT8_DENSE_SHEET, "H100 SXM data sheet, 1979 TOPS dense INT8"


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


def u8_vs_float(fds, pairs, reps):
    """ps_match_u8_batch on the quantised sets against the float ps_match_batch on the same sets, timed alternately"""
    L = api.load_library()
    n = len(fds)
    counts = [fd.getDescriptorCount() for fd in fds]
    rows = sum(counts[i] for i, _ in pairs)
    d_f, d_q = L.ps_dev_alloc(12 * max(rows, 1)), L.ps_dev_alloc(12 * max(rows, 1))
    fptrs = [fd.getDescriptors() for fd in fds]
    qptrs = [L.ps_dev_alloc(max(128 * c, 16)) for c in counts]
    quant = lambda: [L.ps_descriptors_to_u8(0, fp, c, qp) for fp, c, qp in zip(fptrs, counts, qptrs)]  # noqa: E731
    assert all(rc == 0 for rc in quant())
    c_f, c_q = (C.c_void_p * n)(*fptrs), (C.c_void_p * n)(*qptrs)
    c_n = (C.c_int32 * n)(*counts)
    c_pairs = (C.c_int32 * (2 * len(pairs)))(*[v for pq in pairs for v in pq])
    flag = api.FeaturesDev.MATCH_AUTO

    def f32(flags=flag, out=d_f):
        rc = L.ps_match_batch(0, n, c_f, c_n, len(pairs), c_pairs, out, flags)
        assert rc == 0, L.ps_last_error(None)

    def u8(flags=flag, out=d_q):
        rc = L.ps_match_u8_batch(0, n, c_q, c_n, len(pairs), c_pairs, out, flags)
        assert rc == 0, L.ps_last_error(None)

    def fetch(d):
        out = np.zeros((rows, 3), np.int32)
        L.ps_dev_to_host(out.ctypes.data, d, out.nbytes)
        return out
    f32(); u8()                                 # warm-up of the same shapes
    tf, tq = [], []
    for _ in range(reps):                       # alternating, so that clock and thermal drift hit both alike
        tf += timed(f32, 1)
        tq += timed(u8, 1)
    ops = 2.0 * 128 * sum(counts[i] * counts[j] for i, j in pairs)
    peak, src = int8_peak()
    res = {"pairs": len(pairs), "descriptors_per_set_min_max": [int(min(counts)), int(max(counts))]}
    for name, ts in (("float_ps_match_batch", tf), ("u8_ps_match_u8_batch", tq)):
        ms = float(np.median(ts))
        res[name] = {"ms": ms, "ms_min_max": [float(min(ts)), float(max(ts))]}
    res["u8_ps_match_u8_batch"]["int_tops"] = ops / (res["u8_ps_match_u8_batch"]["ms"] * 1e-3) / 1e12
    res["u8_ps_match_u8_batch"]["frac_of_dense_int8"] = res["u8_ps_match_u8_batch"]["int_tops"] / peak
    res["speedup_u8_vs_float"] = res["float_ps_match_batch"]["ms"] / res["u8_ps_match_u8_batch"]["ms"]
    res["peak"] = {"int8_tops": peak, "source": src}
    res["quantise_ms"] = float(np.median(timed(quant, 5)))
    m_q = fetch(d_q)
    f32(); m_f = fetch(d_f)
    u8(api.FeaturesDev.MATCH_EXACT); m_e = fetch(d_q)
    res["rows_differing_u8_vs_u8_exact"] = int((m_q != m_e).any(1).sum())
    # informational: quantisation may change matches
    res["rows_differing_u8_vs_float"] = int((m_q != m_f).any(1).sum())
    res["accepted_u8"], res["accepted_float"] = int(m_q[:, 2].sum()), int(m_f[:, 2].sum())
    res["accepted_differing_u8_vs_float"] = int(((m_q[:, 2] == 1) != (m_f[:, 2] == 1)).sum() +
                                                ((m_q[:, 2] == 1) & (m_f[:, 2] == 1) & (m_q[:, 0] != m_f[:, 0])).sum())
    for p in qptrs + [d_f, d_q]:
        L.ps_dev_free(p)
    return res


def u8_four_k():
    frames = bench.synth_frames(2, 0)
    cfg = api.Config()
    cfg.setOctaves(bench.OCTAVES); cfg.setLevels(bench.LEVELS); cfg.setNormalizationMultiplier(9)
    pm = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=bench.W, max_height=bench.H, slots=2)
    fds = [pm.enqueue(bench.W, bench.H, f).getDev() for f in frames]
    res = {"workload": "one 4K pair (0, 1)", "norm_multi": 9}
    res.update(u8_vs_float(fds, [(0, 1)], 10))
    del fds
    pm.uninit()
    return res


def u8_batch(n):
    w, h = 1920, 1080
    cfg = api.Config()
    cfg.setNormalizationMultiplier(9)
    pm = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=2)
    fds = [pm.enqueue(w, h, make_frame(w, h, 100 + k)).getDev() for k in range(n)]
    res = {"workload": "%d 1920x1080 frames, all ordered pairs" % n, "norm_multi": 9}
    res.update(u8_vs_float(fds, [(i, j) for i in range(n) for j in range(n) if i != j], 5))
    del fds
    pm.uninit()
    return res


def main():
    args = sys.argv[1:]
    pgm_dir, n_batch = None, 0
    u8 = "--u8" in args
    if u8:
        args.remove("--u8")
    if "--pgm" in args:
        i = args.index("--pgm"); pgm_dir = args[i + 1]; del args[i:i + 2]
    if "--batch" in args:
        i = args.index("--batch"); n_batch = int(args[i + 1]); del args[i:i + 2]
    out = args[0] if args else None
    if u8:
        res = u8_batch(n_batch) if n_batch else u8_four_k()
    else:
        res = batch(n_batch) if n_batch else four_k(pgm_dir)
    res["card"] = card()
    res["library"] = api.LIB_PATH
    print(json.dumps(res))
    if out:
        json.dump(res, open(out, "w"), indent=1)


if __name__ == "__main__":
    main()
