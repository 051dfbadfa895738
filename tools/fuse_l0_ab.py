"""A/B of the fused level-0/1 launch of octave 0 (POPSIFT_B200_FUSE_L0=1) against the two separate launches (=0).

    python tools/fuse_l0_ab.py [--runs N] [--steps K] [--warmup W] [out_dir]

Alternates the two settings, N runs each, of `bench.py --gpus 1 --steps K --warmup W --dump-outputs DIR`; reports the median
and range of `value`, `ms_per_step` and `roofline.ms` per setting and whether the dumped outputs of all runs are
byte-identical; then runs tools/stage_profile.py once per setting for the device time of the octave-0 level-0 and level-1
launches against the fused launch.  Card name and power limit are recorded with the numbers."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, clock = [x.strip() for x in q.split(",")]
    return {"name": name, "power_limit": power, "sm_max_clock": clock}


def digest(d):
    h = hashlib.sha256()
    for fn in sorted(os.listdir(d)):
        h.update(fn.encode())
        with open(os.path.join(d, fn), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def env_for(fuse):
    return dict(os.environ, POPSIFT_B200_FUSE_L0="1" if fuse else "0")


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": xs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("out", nargs="?", default=None)
    args = ap.parse_args()

    out = {"card": card(), "bench": {}, "profile": {}}
    print(json.dumps(out["card"]), flush=True)
    res = {1: [], 0: []}
    digests = []
    with tempfile.TemporaryDirectory() as td:
        for i in range(args.runs):
            for fuse in (1, 0):
                d = os.path.join(td, "dump_%d_%d" % (fuse, i))
                cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
                       "--warmup", str(args.warmup), "--dump-outputs", d]
                p = subprocess.run(cmd, env=env_for(fuse), capture_output=True, text=True, cwd=td)
                if p.returncode != 0:
                    raise SystemExit("bench.py failed (FUSE_L0=%d):\n%s" % (fuse, p.stderr[-3000:]))
                line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1]
                j = json.loads(line)
                res[fuse].append(j)
                digests.append(digest(d))
                print("FUSE_L0=%d run %d: value %.1f ms_per_step %.3f roofline.ms %.4f launches %d"
                      % (fuse, i, j["value"], j["ms_per_step"], j["roofline"]["ms"], j["gpu_launches"]), flush=True)
        for fuse in (1, 0):
            prof = os.path.join(td, "stage_%d.json" % fuse)
            p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "stage_profile.py"), prof], env=env_for(fuse),
                               capture_output=True, text=True, cwd=td)
            if p.returncode != 0:
                raise SystemExit("stage_profile.py failed (FUSE_L0=%d):\n%s" % (fuse, p.stderr[-3000:]))
            with open(prof) as f:
                sp = json.load(f)
            out["profile"]["fuse_%d" % fuse] = {
                "pyramid_ms_per_frame": sp["stages_ms_per_frame"]["pyramid"],
                "octave0_level01_kernels": {k: v for k, v in sp["kernels"].items()
                                            if "level0" in k or "level01" in k or "R=5 next=false cand=false" in k},
            }
    for fuse in (1, 0):
        rs = res[fuse]
        out["bench"]["fuse_%d" % fuse] = {"value": summary([r["value"] for r in rs]),
                                          "ms_per_step": summary([r["ms_per_step"] for r in rs]),
                                          "roofline_ms": summary([r["roofline"]["ms"] for r in rs]),
                                          "gpu_launches": rs[0]["gpu_launches"]}
    a, b = out["bench"]["fuse_1"]["value"], out["bench"]["fuse_0"]["value"]
    out["value_gain"] = a["median"] / b["median"] - 1.0
    out["value_ranges_overlap"] = not (a["min"] > b["max"] or b["min"] > a["max"])
    out["dumps_identical"] = len(set(digests)) == 1
    txt = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fuse_l0_ab.json"), "w") as f:
            f.write(txt)
    print(txt)


if __name__ == "__main__":
    main()
