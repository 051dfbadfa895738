#!/usr/bin/env python
"""Times image retrieval on the GPU (popsift_b200_retrieval.h).

    python tools/retrieval_bench.py [--reps N] [out.json]

1. ps_retrieve_pairs on seeded unit vectors, dim = 8 192, m = 20, at n = 1 000 and n = 10 000 (the two sizes alternate):
   median ms per call and the FP32 rate against the 67 TFLOP/s of the H100 SXM data sheet, counting the FMAs needed
   (n (n - 1) / 2 x dim: every unordered pair once, FMA = 2 flops) and, beside it, the FMAs the kernel issues (tiles on
   and above the diagonal, 128 x 128 x dim each).
2. 64 frames of 1920x1080 (16 make_frame scenes x 4 affine views), extracted under MatchingMode: ps_vlad_train (k = 64
   and k = 1 024, 10 iterations) and ps_vlad_encode, ms per frame.
3. What retrieval buys on those frames: ps_match_u8_batch over all 4 032 ordered pairs, against ps_vlad_encode +
   ps_retrieve_pairs (m = 5) + ps_match_u8_batch on the selected unordered pairs (one direction each), with the share of
   the selected pairs whose views show the same scene.  The 8-bit copies of the sets are made once, outside the timings.

Every time is the median of --reps calls after a warm-up, host clock around calls that end in a device synchronise; the
card's name and power limit are read in the same run."""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [v.strip() for v in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # noqa: BLE001 -- the numbers are still worth printing
        return {"error": str(e)}


def scenes(n_scenes=16, views=4, w=1920, h=1080):
    rng = np.random.default_rng(11)
    out = []
    for s in range(n_scenes):
        base = make_frame(w, h, 200 + s)
        out.append(base)
        for _ in range(views - 1):
            a = np.deg2rad(rng.uniform(-20, 20))
            sc = rng.uniform(0.8, 1.25)
            sh = rng.uniform(-0.15, 0.15)
            L = sc * np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]) @ np.array([[1, sh], [0, 1]])
            c = np.array([w / 2, h / 2])
            out.append(affine_warp(base, np.c_[L, c - L @ c + rng.uniform(-60, 60, 2)]))
    return out


def check(lib, rc, name):
    if rc != 0:
        raise RuntimeError("%s error %d: %s" % (name, rc, lib.ps_last_error(None).decode()))


def main(argv):
    reps = 5
    if "--reps" in argv:
        i = argv.index("--reps")
        reps = int(argv[i + 1])
        argv = argv[:i] + argv[i + 2:]
    out_path = argv[0] if argv else None
    lib = api.load_library()
    bufs = api._DevBuffers(lib)
    res = {"card": card(), "reps": reps}
    try:
        # 1. similarity + top-m
        dim, m = 8192, 20
        rng = np.random.default_rng(1)
        legs = {}
        for n in (1000, 10000):
            v = rng.normal(size=(n, dim)).astype(np.float32)
            v /= np.linalg.norm(v, axis=1, keepdims=True)
            legs[n] = (bufs.upload(v), bufs.alloc(n * m * 4), bufs.alloc(n * m * 4))
        times = {n: [] for n in legs}
        for n, (d_v, d_n, d_s) in legs.items():
            check(lib, lib.ps_retrieve_pairs(0, n, d_v, dim, m, d_n, d_s), "ps_retrieve_pairs")      # warm-up
        for _ in range(reps):
            for n, (d_v, d_n, d_s) in legs.items():
                t0 = time.perf_counter()
                check(lib, lib.ps_retrieve_pairs(0, n, d_v, dim, m, d_n, d_s), "ps_retrieve_pairs")
                times[n].append((time.perf_counter() - t0) * 1e3)
        for n in legs:
            ms = float(np.median(times[n]))
            T = (n + 127) // 128
            need = n * (n - 1) / 2 * dim
            issued = T * (T + 1) / 2 * 128 * 128 * dim
            res["retrieve_n%d" % n] = {"ms": ms, "tflops_needed": 2 * need / ms / 1e9, "share_needed": 2 * need / ms / 1e9 / FP32_SHEET,
                                       "tflops_issued": 2 * issued / ms / 1e9, "share_issued": 2 * issued / ms / 1e9 / FP32_SHEET}
        bufs.free()

        # 2. codebook and encoding on 64 extracted 1080p frames
        imgs = scenes()
        w, h = 1920, 1080
        ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
        sets = [ps.enqueue(w, h, im).getDev() for im in imgs]
        n_img = len(sets)
        counts = [s.getDescriptorCount() for s in sets]
        res["frames"] = {"n": n_img, "descriptors_mean": float(np.mean(counts))}
        k = 64
        c_sets = (C.c_void_p * n_img)(*[s.getDescriptors() for s in sets])
        c_n = (C.c_int32 * n_img)(*counts)
        d_c, d_v = bufs.alloc(k * 512), bufs.alloc(n_img * k * 512)
        d_nb, d_sc = bufs.alloc(n_img * 5 * 4), bufs.alloc(n_img * 5 * 4)
        train = lambda: check(lib, lib.ps_vlad_train(0, n_img, c_sets, c_n, k, 10, 0, d_c, 0), "ps_vlad_train")  # noqa: E731
        encode = lambda: check(lib, lib.ps_vlad_encode(0, n_img, c_sets, c_n, k, d_c, d_v, None, 0), "ps_vlad_encode")  # noqa: E731
        t_train, t_enc = [], []
        train(); encode()
        for _ in range(reps):
            t0 = time.perf_counter(); train(); t_train.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); encode(); t_enc.append((time.perf_counter() - t0) * 1e3)
        res["train_k64_10it_ms_per_frame"] = float(np.median(t_train)) / n_img
        res["encode_k64_ms_per_frame"] = float(np.median(t_enc)) / n_img
        # the largest codebook: the aggregation rescans a chunk's assignments once per centroid (O(N k) reads)
        kb = 1024
        d_cb = bufs.alloc(kb * 512)
        d_vb = bufs.alloc(n_img * kb * 512)
        train_b = lambda: check(lib, lib.ps_vlad_train(0, n_img, c_sets, c_n, kb, 10, 0, d_cb, 0), "ps_vlad_train")  # noqa: E731
        encode_b = lambda: check(lib, lib.ps_vlad_encode(0, n_img, c_sets, c_n, kb, d_cb, d_vb, None, 0), "ps_vlad_encode")  # noqa: E731
        t_train, t_enc = [], []
        train_b(); encode_b()
        for _ in range(max(1, reps // 2)):
            t0 = time.perf_counter(); train_b(); t_train.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); encode_b(); t_enc.append((time.perf_counter() - t0) * 1e3)
        res["train_k1024_10it_ms_per_frame"] = float(np.median(t_train)) / n_img
        res["encode_k1024_ms_per_frame"] = float(np.median(t_enc)) / n_img

        # 3. all ordered pairs against retrieval + the selected pairs
        q = [api._to_u8_dev(lib, s.getDescriptors(), s.getDescriptorCount(), 0) for s in sets]
        bufs.ptrs += q
        c_q = (C.c_void_p * n_img)(*q)
        all_pairs = [(i, j) for i in range(n_img) for j in range(n_img) if i != j]
        d_out = bufs.alloc(sum(counts[i] for i, _ in all_pairs) * 12)

        def match(pairs):
            flat = (C.c_int32 * max(2 * len(pairs), 1))(*[v for pq in pairs for v in pq])
            check(lib, lib.ps_match_u8_batch(0, n_img, c_q, c_n, len(pairs), flat, d_out, 0), "ps_match_u8_batch")

        sel = []

        def retrieve_and_match():
            encode()
            check(lib, lib.ps_retrieve_pairs(0, n_img, d_v, k * 128, 5, d_nb, d_sc), "ps_retrieve_pairs")
            nbr = bufs.download(d_nb, (n_img, 5), np.int32)
            sel[:] = api.select_pairs(nbr)
            match(sel)

        t_all, t_ret = [], []
        match(all_pairs); retrieve_and_match()
        for _ in range(reps):
            t0 = time.perf_counter(); match(all_pairs); t_all.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); retrieve_and_match(); t_ret.append((time.perf_counter() - t0) * 1e3)
        scene = np.arange(n_img) // 4
        res["all_pairs"] = {"pairs": len(all_pairs), "ms": float(np.median(t_all))}
        res["retrieval_m5"] = {"pairs": len(sel), "ms": float(np.median(t_ret)),
                               "same_scene_share": float(np.mean([scene[i] == scene[j] for i, j in sel])),
                               "same_scene_pairs_found": int(sum(scene[i] == scene[j] for i, j in sel)), "same_scene_pairs": 16 * 6}
        ps.uninit()
    finally:
        bufs.free()
    txt = json.dumps(res, indent=1)
    print(txt)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(txt)


if __name__ == "__main__":
    main(sys.argv[1:])
