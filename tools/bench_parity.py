#!/usr/bin/env python
"""Parity of the BENCHMARK workload itself (runs on a GPU machine): the 32 synthetic 3840x2160 frames of
bench.py, default Config (PopSift mode, RootSift, octaves=5, levels=3), through
  * the unmodified reference (oracle/_ref/ref_dump), TWICE  -> its own run-to-run jitter,
  * this library.
Writes a compact JSON: per-frame feature / descriptor counts of the three runs, and for every keypoint
whose orientation set differs (reference run A vs run B, and ours vs reference run A) the keypoint and
both orientation lists.  Descriptors are compared for the keypoints whose orientations agree.

    python tools/bench_parity.py OUT.json [n_frames]
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

import bench  # noqa: E402
import oracle_lib as ol  # noqa: E402
from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import write_pgm  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "ref_dump")


def keyed(feat):
    """(octave, x bits, y bits, sigma bits) -> feature row"""
    k = np.stack([feat["octave"].astype(np.int64), feat["x"].view(np.int32).astype(np.int64),
                  feat["y"].view(np.int32).astype(np.int64), feat["sigma"].view(np.int32).astype(np.int64)], axis=1)
    return {tuple(r): i for i, r in enumerate(k.tolist())}


def ori_list(f):
    return sorted(float(v) for v in f["ori"][: int(f["num_ori"])])


def diff_runs(fa, da, ia, fb, db, ib, tol=1e-6):
    """features of run a vs run b: keypoints only in one, keypoints whose orientation sets differ, and the
    descriptor L2 over the (keypoint, orientation) pairs that agree"""
    ka, kb = keyed(fa), keyed(fb)
    only_a = [k for k in ka if k not in kb]
    only_b = [k for k in kb if k not in ka]
    ori_diffs, l2 = [], []
    for k, i in ka.items():
        j = kb.get(k)
        if j is None:
            continue
        oa, ob = ori_list(fa[i]), ori_list(fb[j])
        same = len(oa) == len(ob) and all(abs(x - y) < tol for x, y in zip(oa, ob))
        if not same:
            ori_diffs.append({"octave": int(fa[i]["octave"]), "x": float(fa[i]["x"]), "y": float(fa[i]["y"]),
                              "sigma": float(fa[i]["sigma"]), "a": oa, "b": ob})
            continue
        for r in range(int(fa[i]["num_ori"])):
            # orientations are stored in the same (descending peak) order when the sets agree
            rb = int(np.argmin(np.abs(fb[j]["ori"][: int(fb[j]["num_ori"])] - fa[i]["ori"][r])))
            va, vb = da[ia[i][r]], db[ib[j][rb]]
            l2.append(float(np.linalg.norm(va.astype(np.float64) - vb.astype(np.float64))))
    l2 = np.array(l2) if l2 else np.zeros(1)
    return {"only_a": len(only_a), "only_b": len(only_b), "ori_diffs": ori_diffs, "pairs": int(len(l2)),
            "desc_l2_max": float(l2.max()), "desc_l2_p999": float(np.percentile(l2, 99.9)), "desc_l2_median": float(np.median(l2))}


def main(out, n_frames):
    frames = bench.synth_frames(n_frames, 0)
    res = {"workload": "bench.py frames (3840x2160, seed 7 variants), default Config, octaves=5 levels=3", "frames": []}
    with tempfile.TemporaryDirectory() as td:
        cmd = [REF, "--octaves", "5", "--levels", "3", "-o", os.path.join(td, "ref"), "--repeat", "2"]
        for i, f in enumerate(frames):
            p = os.path.join(td, "f%d.pgm" % i)
            write_pgm(p, f)
            cmd += ["-i", p]
        subprocess.run(cmd, check=True, capture_output=True)
        cfg = api.Config()
        cfg.setOctaves(5)
        cfg.setLevels(3)
        ps = api.PopSift(cfg, max_width=bench.W, max_height=bench.H, slots=2)
        tot = {"ours": [0, 0], "ref_a": [0, 0], "ref_b": [0, 0]}
        for i, f in enumerate(frames):
            r = ps.enqueue(bench.W, bench.H, f).get()
            of, od, oi = r.feat.copy(), r.desc.copy(), r.desc_idx.copy()
            suffix = (".%d" % i) if len(frames) > 1 else ""
            fa, da = ol.read_ref_features(os.path.join(td, "ref%s.r0" % suffix))
            fb, db = ol.read_ref_features(os.path.join(td, "ref%s.r1" % suffix))
            row = {"frame": i, "ours": [len(of), len(od)], "ref_a": [len(fa), len(da)], "ref_b": [len(fb), len(db)]}
            for k in tot:
                tot[k][0] += row[k][0]; tot[k][1] += row[k][1]
            row["ref_a_vs_ref_b"] = diff_runs(fa, da, fa["desc_idx"], fb, db, fb["desc_idx"])
            row["ours_vs_ref_a"] = diff_runs(of, od, oi, fa, da, fa["desc_idx"])
            res["frames"].append(row)
            print(i, row["ours"], row["ref_a"], row["ref_b"], len(row["ref_a_vs_ref_b"]["ori_diffs"]),
                  len(row["ours_vs_ref_a"]["ori_diffs"]), row["ours_vs_ref_a"]["desc_l2_max"], flush=True)
            os.remove(os.path.join(td, "ref%s.r0" % suffix)); os.remove(os.path.join(td, "ref%s.r1" % suffix))
        ps.uninit()
        res["totals"] = tot
    json.dump(res, open(out, "w"), indent=1)
    print(json.dumps(res["totals"]))


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 32)
