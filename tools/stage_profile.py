"""Per-kernel device time of the benchmark workload, from torch.profiler (CUDA activities), in a run of its own.

    python tools/stage_profile.py [--frames N] [--warmup W] [out.json]

N 3840x2160 frames of bench.py's workload (octaves 5, levels 3, default Config) go through ps_submit_dev_u8 / ps_counts on
ONE slot, so that kernels of different frames do not overlap and each kernel's duration is its own.  The first W frames
(run directly, captured, replayed) are not profiled.  Kernels are grouped by instantiation (march_level_kernel by radius,
NEXT and CAND flags); the JSON gives the device time per frame of each group and of each stage, the card name and power
limit, and the pyramid's algorithmic bytes per frame under the 68 B and 48 B per octave-pixel models (the level kernels
with and without DoG plane stores)."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, OCTAVES, LEVELS = 3840, 2160, 5, 3


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        out["power_limit"], out["sm_max_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:
        out["power_limit"] = "unavailable: %s" % e
    return out


def group(name: str):
    """(stage, group key) of one kernel name"""
    m = re.search(r"march_level_kernel<(\d+), (\w+), (\w+)>", name)
    if m:
        return "pyramid", "march_level_kernel R=%s next=%s cand=%s" % m.groups()
    m = re.search(r"(march_level01x2_kernel|march_level0x2_kernel|march_level0_kernel|level0_kernel|level0_generic_kernel)<([^>]*)>", name)
    if m:
        return "pyramid", "level0 %s<%s>" % (m.group(1), m.group(2))
    m = re.search(r"(cand_extrema_kernel|find_extrema_kernel)<([^>]*)>", name)
    if m:
        return "extrema", "%s<%s>" % (m.group(1), m.group(2))
    base = re.sub(r"^void\s+", "", name.replace("(anonymous namespace)::", "").split("(")[0])
    base = base.split("::")[-1]
    low = base.lower()
    for stage, keys in (("pyramid", ("blur", "decimate", "dog_planes", "interp", "fixed_")),
                        ("orientation", ("ori",)), ("descriptors", ("desc",)), ("prep", ("prep", "fix_feature"))):
        if any(k in low for k in keys):
            return stage, base
    return "other", base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("out", nargs="?", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("stage_profile.py: no CUDA device")
    import bench
    from popsift_b200 import api

    L = api.load_library()
    cfg = api.Config()
    cfg.setOctaves(OCTAVES)
    cfg.setLevels(LEVELS)
    ctx = L.ps_create(0, C.byref(cfg._c), W, H, 1)
    if not ctx:
        raise SystemExit("ps_create failed: " + L.ps_last_error(None).decode())
    frames = [torch.from_numpy(f).cuda() for f in bench.synth_frames(max(args.frames, args.warmup), 0)]
    nf, nd = C.c_int32(), C.c_int32()

    def run(i):
        f = frames[i % len(frames)]
        if L.ps_submit_dev_u8(ctx, 0, f.data_ptr(), W, W, H) != 0 or L.ps_counts(ctx, 0, C.byref(nf), C.byref(nd)) != 0:
            raise SystemExit("popsift_b200: " + L.ps_last_error(ctx).decode())
        return nf.value, nd.value

    for i in range(args.warmup):
        run(i)
    torch.cuda.synchronize()
    counts = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.frames):
            counts.append(run(i))
        torch.cuda.synchronize()
    L.ps_destroy(ctx)
    with tempfile.TemporaryDirectory() as td:
        tr = os.path.join(td, "trace.json")
        prof.export_chrome_trace(tr)
        events = json.load(open(tr))["traceEvents"]

    kernels = defaultdict(lambda: {"stage": "", "launches": 0, "us": 0.0})
    for e in events:
        if e.get("cat") != "kernel":
            continue
        stage, key = group(e["name"])
        k = kernels[key]
        k["stage"] = stage
        k["launches"] += 1
        k["us"] += float(e["dur"])
    n = args.frames
    per_kernel = {key: {"stage": v["stage"], "launches_per_frame": v["launches"] / n, "ms_per_frame": v["us"] / n / 1e3}
                  for key, v in sorted(kernels.items(), key=lambda kv: -kv[1]["us"])}
    stages = defaultdict(float)
    for v in per_kernel.values():
        stages[v["stage"]] += v["ms_per_frame"]
    geo = cfg.geometry(W, H)
    sum_wh = sum(w * h for w, h in geo)
    w0, h0 = geo[0]
    out = {
        "card": card(),
        "workload": "%d frames %dx%d u8, octaves %d, levels %d, default Config, one slot (+%d warm-up frames)" % (n, W, H, OCTAVES, LEVELS, args.warmup),
        "features_per_frame": [c[0] for c in counts],
        "kernels": per_kernel,
        "stages_ms_per_frame": dict(stages),
        "pyramid_plus_extrema_ms_per_frame": stages["pyramid"] + stages["extrema"],
        "pyramid_bytes_per_frame": {
            "octave_pixels": sum_wh,
            "model_68B": 68 * sum_wh,
            "model_48B": 48 * sum_wh,
            "note": "68 B per octave-pixel: level kernels read G[l-1], write G[l] and DoG[l-1]; 48 B: no DoG plane stores",
        },
        "octave0_level_launch_bytes": {"with_dog_12B": 12 * w0 * h0, "without_dog_8B": 8 * w0 * h0},
    }
    txt = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt)
    print(txt)


if __name__ == "__main__":
    main()
