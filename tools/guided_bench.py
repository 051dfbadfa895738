#!/usr/bin/env python
"""Times guided matching on the GPU against the unguided matchers, on the workload of tools/verify_bench.py: 16 seeded affine
views (synth.affine_warp) of one 1920x1080 make_frame, extracted under MatchingMode with norm_multi = 9 (so that the 8-bit
descriptors are meaningful; the float matcher's ranking does not depend on the scale), all 240 ordered pairs.  The models
come from ps_verify_batch (homography: 1024 samples, fundamental matrix: 4096, t = 4 px) on the correspondences of
ps_match_batch, and stay on the device.

    python tools/guided_bench.py [--reps N] [out.json]

Variants, timed alternately (one call of each per round) after a warm-up, median ms per call (host clock around calls
that end in a device synchronise):
    match_f32      ps_match_batch
    guided_f32_h   ps_match_guided_batch, homographies, t = 4 px
    guided_f32_f   ps_match_guided_batch, fundamental matrices, t = 4 px
    match_u8       ps_match_u8_batch
    guided_u8_h    ps_match_u8_guided_batch, homographies, t = 4 px
For each: accepted rows and correspondences (ps_match_correspondences), and the fraction of correspondences within t of the
views' true affine map -- for the unguided float matcher also that of its verified (homography) inliers.  The card name and
power limit are read in the same run."""
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

T = 4.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [v.strip() for v in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                      # noqa: BLE001 -- the numbers are still worth printing
        return {"error": str(e)}


def views(n=16, w=1920, h=1080, seed=3):
    """the views of tools/verify_bench.py (same seed, same draws) and their 3x3 maps from the base frame"""
    base = make_frame(w, h, seed)
    rng = np.random.default_rng(seed)
    cx, cy = (w - 1) / 2, (h - 1) / 2
    out, maps = [base], [np.eye(3)]
    for _ in range(n - 1):
        th, sc = np.deg2rad(rng.uniform(-12, 12)), rng.uniform(0.85, 1.15)
        L = sc * np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ np.array([[1, rng.uniform(-0.1, 0.1)], [0, 1]])
        t = np.array([cx, cy]) - L @ np.array([cx, cy]) + rng.uniform(-40, 40, 2)
        A = np.hstack([L, t[:, None]])
        out.append(affine_warp(base, A))
        maps.append(np.vstack([A, [0, 0, 1.0]]))
    return out, maps


def main():
    args = sys.argv[1:]
    reps = 20
    if "--reps" in args:
        i = args.index("--reps")
        reps = int(args[i + 1])
        del args[i:i + 2]
    out_path = args[0] if args else None
    info = {"card": card(), "threshold_px": T}
    lib = api.load_library()
    w, h = 1920, 1080
    cfg = api.Config()
    cfg.setNormalizationMultiplier(9)
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    images, maps = views()
    sets = [ps.enqueue(w, h, im).getDev() for im in images]
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if i != j]
    P = len(pairs)
    counts = [s.getDescriptorCount() for s in sets]
    rows = sum(counts[l] for l, _ in pairs)
    start = np.concatenate([[0], np.cumsum([counts[l] for l, _ in pairs])])[:-1].astype(np.int32)
    bufs = api._DevBuffers(lib)
    try:
        c_pairs = (C.c_int32 * (2 * P))(*[v for pq in pairs for v in pq])
        c_n = (C.c_int32 * len(sets))(*counts)
        c_sets = (C.c_void_p * len(sets))(*[s.getDescriptors() for s in sets])
        c_feat = (C.c_void_p * len(sets))(*[s.getFeatures() for s in sets])
        c_rev = (C.c_void_p * len(sets))(*[s.getReverseMap() for s in sets])
        q = [api._to_u8_dev(lib, s.getDescriptors(), s.getDescriptorCount(), 0) for s in sets]
        bufs.ptrs += q
        c_sets8 = (C.c_void_p * len(sets))(*q)
        d_out = {k: bufs.alloc(rows * 12) for k in ("match_f32", "guided_f32_h", "guided_f32_f", "match_u8", "guided_u8_h")}
        d_corr, d_src = bufs.alloc(rows * 16), bufs.alloc(rows * 4)
        d_models = {0: bufs.alloc(P * 36), 1: bufs.alloc(P * 36)}
        d_n, d_mask = bufs.alloc(P * 4), bufs.alloc(rows)
        n_corr = np.zeros(P, np.int32)

        def gather(d_match):
            assert lib.ps_match_correspondences(0, len(sets), c_feat, c_rev, c_n, P, c_pairs, d_match, d_corr, d_src,
                                                n_corr.ctypes.data) == 0

        # the models: verification of the unguided float matches
        assert lib.ps_match_batch(0, len(sets), c_sets, c_n, P, c_pairs, d_out["match_f32"], 0) == 0
        gather(d_out["match_f32"])
        nc_match = n_corr.copy()
        masks = {}
        for model, ns in ((0, 1024), (1, 4096)):
            prm = api._verify_params(model, T, ns, 0, True)
            assert lib.ps_verify_batch(0, P, d_corr, start.ctypes.data, n_corr.ctypes.data, C.byref(prm), d_models[model], d_n,
                                       d_mask, None) == 0
            masks[model] = bufs.download(d_mask, rows, np.uint8).astype(bool)
        corr_match = bufs.download(d_corr, (rows, 4), np.float32)

        calls = {
            "match_f32": lambda: lib.ps_match_batch(0, len(sets), c_sets, c_n, P, c_pairs, d_out["match_f32"], 0),
            "guided_f32_h": lambda: lib.ps_match_guided_batch(0, len(sets), c_sets, c_feat, c_rev, c_n, P, c_pairs, d_models[0], 0, T,
                                                              d_out["guided_f32_h"], 0),
            "guided_f32_f": lambda: lib.ps_match_guided_batch(0, len(sets), c_sets, c_feat, c_rev, c_n, P, c_pairs, d_models[1], 1, T,
                                                              d_out["guided_f32_f"], 0),
            "match_u8": lambda: lib.ps_match_u8_batch(0, len(sets), c_sets8, c_n, P, c_pairs, d_out["match_u8"], 0),
            "guided_u8_h": lambda: lib.ps_match_u8_guided_batch(0, len(sets), c_sets8, c_feat, c_rev, c_n, P, c_pairs, d_models[0], 0, T,
                                                                d_out["guided_u8_h"], 0),
        }
        for _ in range(2):
            for fn in calls.values():
                assert fn() == 0
        times = {k: [] for k in calls}
        for _ in range(reps):
            for k, fn in calls.items():
                t0 = time.perf_counter()
                assert fn() == 0
                times[k].append((time.perf_counter() - t0) * 1e3)

        def true_err(corr, lr):
            l, r = lr
            M = maps[r] @ np.linalg.inv(maps[l])
            pr = corr[:, :2].astype(np.float64) @ M[:2, :2].T + M[:2, 2]
            return np.linalg.norm(pr - corr[:, 2:].astype(np.float64), axis=1)

        info.update(frames=len(sets), pairs=P, descriptors=int(sum(counts)), match_rows=int(rows), reps=reps)
        for k in calls:
            m = bufs.download(d_out[k], (rows, 3), np.int32)
            gather(d_out[k])
            corr = bufs.download(d_corr, (rows, 4), np.float32)
            within = total = 0
            for p in range(P):
                e = true_err(corr[start[p]:start[p] + n_corr[p]], pairs[p])
                within += int((e < T).sum()); total += len(e)
            info[k] = {"ms": float(np.median(times[k])), "ms_all": [round(v, 4) for v in times[k]], "accepted_rows": int(m[:, 2].sum()),
                       "correspondences": int(n_corr.sum()), "within_t_of_true_map": within,
                       "fraction_within_t": within / max(total, 1)}
        for model, name in ((0, "verified_h"), (1, "verified_f")):
            within = total = 0
            for p in range(P):
                sl = slice(start[p], start[p] + nc_match[p])
                c = corr_match[sl][masks[model][sl]]
                e = true_err(c, pairs[p])
                within += int((e < T).sum()); total += len(e)
            info["match_f32"][name + "_inliers"] = total
            info["match_f32"][name + "_within_t"] = within
            info["match_f32"][name + "_fraction_within_t"] = within / max(total, 1)
        for g, u in (("guided_f32_h", "match_f32"), ("guided_f32_f", "match_f32"), ("guided_u8_h", "match_u8")):
            info[g]["time_vs_unguided"] = info[g]["ms"] / info[u]["ms"]
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
