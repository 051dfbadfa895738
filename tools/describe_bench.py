#!/usr/bin/env python
"""Times the describe path (ps_describe_u8) against extraction (ps_submit_u8) on 3840x2160 make_frame frames, per frame:

    extract        ps_submit_u8 + ps_counts + ps_download
    given          ps_describe_u8(PS_DESCRIBE_GIVEN) at the frame's own keypoints (one per descriptor, its angle)
    orient         ps_describe_u8(PS_DESCRIBE_ORIENT) at the frame's own keypoints (one per Feature)
    dense          ps_describe_u8(PS_DESCRIBE_GIVEN) on an upright grid: step 8 px, image sigma 3.2 (~130 000 keypoints)

The four run alternating, frame after frame, after a warm-up of every case; each time is a host clock around the call and
the download of its results (which end in a device synchronise).  Prints one JSON object with the medians and the card's
name and power limit.

    python tools/describe_bench.py [--frames N] [--warmup W] [out.json]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from match_bench import card  # noqa: E402
from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import make_frame  # noqa: E402

W, H = 3840, 2160


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("out", nargs="?")
    a = ap.parse_args()
    frames = [make_frame(W, H, 100 + i) for i in range(3)]
    ps = api.PopSift(api.Config(), max_width=W, max_height=H, slots=1)
    # each frame's own keypoints, from one extraction
    own = []
    for img in frames:
        f = ps.enqueue(W, H, img).get()
        ext = ps.extrema(0)
        n = f.feat["num_ori"].astype(np.int64)
        idx = np.repeat(np.arange(len(n)), n)
        k = np.arange(len(idx)) - np.repeat(np.cumsum(n) - n, n)
        given = np.zeros(len(idx), api.KEYPOINT_DTYPE)
        for c in ("x", "y", "sigma"):
            given[c] = f.feat[c][idx]
        given["ori"] = f.feat["ori"][idx, k]
        given["octave"], given["level"] = ext["octave"][idx], ext["lpos"][idx]
        per_feat = np.zeros(len(n), api.KEYPOINT_DTYPE)
        for c in ("x", "y", "sigma"):
            per_feat[c] = f.feat[c]
        per_feat["octave"], per_feat["level"] = ext["octave"], ext["lpos"]
        own.append((given, per_feat))
    ys, xs = np.mgrid[0:H:8, 0:W:8]
    dense = np.zeros(xs.size, api.KEYPOINT_DTYPE)
    dense["x"], dense["y"], dense["sigma"] = xs.ravel(), ys.ravel(), 3.2
    dense["octave"] = dense["level"] = -1

    cases = {
        "extract": lambda i: ps.enqueue(W, H, frames[i]),
        "given": lambda i: ps.describe(W, H, frames[i], own[i][0]),
        "orient": lambda i: ps.describe(W, H, frames[i], own[i][1], orientations=True),
        "dense": lambda i: ps.describe(W, H, frames[i], dense),
    }
    times = {c: [] for c in cases}
    counts = {}
    for it in range(a.warmup + a.frames):
        i = it % len(frames)
        for c, fn in cases.items():
            t0 = time.perf_counter()
            f = fn(i).get()
            dt = (time.perf_counter() - t0) * 1e3
            counts[c] = (f.getFeatureCount(), f.getDescriptorCount())
            if it >= a.warmup:
                times[c].append(dt)
    ps.uninit()
    res = {"card": card(), "size": [W, H], "frames": a.frames,
           "ms_median": {c: float(np.median(v)) for c, v in times.items()},
           "ms_min": {c: float(np.min(v)) for c, v in times.items()},
           "last_counts": counts, "dense_keypoints": int(len(dense))}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
