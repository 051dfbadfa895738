#!/usr/bin/env python
"""Where do the last-bit differences of orientation angles come from?  (runs on a GPU machine)

Four 4K benchmark frames through the reference (5 octaves, twice; and 2 octaves: the same octave-0/1 data in a different
launch context) and through this library with the orientation kernel in several launch shapes (environment toggles of
k_orient.cu).  For every pair of runs: keypoints (bit-equal octave/x/y/sigma) whose angle lists differ in any bit, per octave.

    python tools/ori_experiment.py OUT.json
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_FRAMES = 4
VARIANTS = {
    "default": {},
    "one_warp_per_cta": {"POPSIFT_B200_ORI_WARPS": "1"},
    "one_warp_per_cta_148_ctas": {"POPSIFT_B200_ORI_WARPS": "1", "POPSIFT_B200_ORI_GRID": "148"},
    "four_warps_148_ctas": {"POPSIFT_B200_ORI_GRID": "148"},
    "lane_sums": {"POPSIFT_B200_ORI_LANESUM": "1"},
}


def child(out):
    import bench
    from popsift_b200 import api
    frames = bench.synth_frames(N_FRAMES, 0)
    cfg = api.Config(); cfg.setOctaves(5); cfg.setLevels(3)
    ps = api.PopSift(cfg, max_width=bench.W, max_height=bench.H, slots=1)
    res = {}
    for i, f in enumerate(frames):
        r = ps.enqueue(bench.W, bench.H, f).get()
        res["f%d" % i] = r.feat.copy()
    ps.uninit()
    np.savez(out, **res)


def keyed(feat):
    k = np.stack([feat["octave"].astype(np.int64), feat["x"].view(np.int32).astype(np.int64),
                  feat["y"].view(np.int32).astype(np.int64), feat["sigma"].view(np.int32).astype(np.int64)], axis=1)
    return {tuple(r): i for i, r in enumerate(k.tolist())}


def diff(fa, fb, octaves=5):
    ka, kb = keyed(fa), keyed(fb)
    per = [[0, 0] for _ in range(octaves)]           # [common keypoints, keypoints with a differing angle list]
    for k, i in ka.items():
        j = kb.get(k)
        if j is None:
            continue
        o = int(k[0])
        per[o][0] += 1
        a = np.sort(fa[i]["ori"][: int(fa[i]["num_ori"])]); b = np.sort(fb[j]["ori"][: int(fb[j]["num_ori"])])
        if len(a) != len(b) or not np.array_equal(a.view(np.int32), b.view(np.int32)):
            per[o][1] += 1
    return per


def main(out):
    import bench
    import oracle_lib as ol
    from popsift_b200.synth import write_pgm
    REF = os.path.join(ROOT, "oracle", "_ref", "ref_dump")
    frames = bench.synth_frames(N_FRAMES, 0)
    runs = {}
    with tempfile.TemporaryDirectory() as td:
        ins = []
        for i, f in enumerate(frames):
            p = os.path.join(td, "f%d.pgm" % i); write_pgm(p, f); ins += ["-i", p]
        subprocess.run([REF, "--octaves", "5", "--levels", "3", "-o", os.path.join(td, "ref5"), "--repeat", "2"] + ins, check=True, capture_output=True)
        subprocess.run([REF, "--octaves", "2", "--levels", "3", "-o", os.path.join(td, "ref2")] + ins, check=True, capture_output=True)
        runs["ref_5oct_a"] = [ol.read_ref_features(os.path.join(td, "ref5.%d.r0" % i))[0] for i in range(N_FRAMES)]
        runs["ref_5oct_b"] = [ol.read_ref_features(os.path.join(td, "ref5.%d.r1" % i))[0] for i in range(N_FRAMES)]
        runs["ref_2oct"] = [ol.read_ref_features(os.path.join(td, "ref2.%d" % i))[0] for i in range(N_FRAMES)]
        for name, env in VARIANTS.items():
            o = os.path.join(td, name + ".npz")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", o], check=True, env={**os.environ, **env})
            z = np.load(o)
            runs["ours_" + name] = [z["f%d" % i] for i in range(N_FRAMES)]
    res = {}
    pairs = [("ref_5oct_a", "ref_5oct_b"), ("ref_5oct_a", "ref_2oct")] + [("ours_" + v, "ref_5oct_a") for v in VARIANTS] + \
            [("ours_default", "ours_one_warp_per_cta"), ("ours_default", "ours_one_warp_per_cta_148_ctas")]
    for a, b in pairs:
        tot = [[0, 0] for _ in range(5)]
        for i in range(N_FRAMES):
            for o, (c, d) in enumerate(diff(runs[a][i], runs[b][i])):
                tot[o][0] += c; tot[o][1] += d
        res["%s vs %s" % (a, b)] = tot
        print("%-55s" % ("%s vs %s" % (a, b)), " ".join("o%d:%d/%d" % (o, d, c) for o, (c, d) in enumerate(tot)), flush=True)
    json.dump(res, open(out, "w"), indent=1)


if __name__ == "__main__":
    if sys.argv[1] == "--child":
        child(sys.argv[2])
    else:
        main(sys.argv[1])
