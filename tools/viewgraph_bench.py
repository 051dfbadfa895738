"""ps_view_graph_filter on global_bench.py's co-visibility graph, with card name and power limit.

  The graph: triangulate_bench's 1 000 cameras and 2 M tracks, pairs = the distinct pairs of consecutive members of the
  tracks (240 015), n_front = the tracks they share; relative rotations with 0.5 degree noise, 10 % replaced by random
  rotations that keep their real n_front (global_bench.py's draws, the same seed).  Reported: median ms per call over the
  reps (inputs on the device, a host clock ending in a synchronise), the kernel split (adjacency build / enumeration /
  decision, torch.profiler, a run of its own), triangles per second of the enumeration, the enumeration's algorithmic
  bytes against 3.35 TB/s (the H100 SXM data sheet), and rotation averaging with global_bench.py's parameters on all
  pairs and on the kept pairs (median and largest error against the truth after alignment).

    python tools/viewgraph_bench.py [--reps N] [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bundle_oracle as bo          # noqa: E402
import global_oracle as go          # noqa: E402
import triangulate_bench as tb      # noqa: E402
from popsift_b200 import api        # noqa: E402

PEAK_BW = 3.35e12


def covisibility(rng):
    """global_bench.py's rotation-averaging input: (R_true, pairs, records, is_outlier)"""
    g = tb.make_graph(rng)
    n = len(g["n_feat"])
    Rt = np.stack([np.asarray(R) for R, _ in g["poses"]])
    np.stack([bo.small_rotation(rng, 0.1) @ R for R in Rt])       # global_bench draws the positioning rotations here
    st = np.asarray(g["start"], np.int64)
    off = np.concatenate([[0], np.cumsum(g["n_feat"])])
    mem_set = np.searchsorted(off, np.asarray(g["members"], np.int64), side="right") - 1
    same = np.ones(len(mem_set) - 1, bool)
    same[st[1:-1] - 1] = False
    key = mem_set[:-1][same].astype(np.int64) * n + mem_set[1:][same]
    keys, nf = np.unique(key, return_counts=True)
    pairs = [(int(k // n), int(k % n)) for k in keys]
    out_pair = rng.random(len(pairs)) < 0.1
    rec = np.zeros(len(pairs), api.TWO_VIEW_DTYPE)
    for p, (l, r) in enumerate(pairs):
        rec[p]["R"] = go.random_rotation(rng) if out_pair[p] else bo.small_rotation(rng, 0.5) @ Rt[r] @ Rt[l].T
    rec["n_front"] = nf
    return Rt, pairs, rec, out_pair


def enumeration_bytes(n, pairs):
    """the bytes vg_enum_kernel reads, from the oriented CSR rebuilt on the host: per oriented entry its pair id, ends and
    the two out-list bounds (4 + 8 + 16), the shorter list once (4 per entry) and one binary search of the longer per entry
    (4 per probe); per triangle the two other pair ids (8), three rotations (216) and three ends (24).  Returns
    (adjacency bytes, triangle bytes per triangle)"""
    e = np.asarray(pairs, np.int64)
    deg = np.bincount(e.reshape(-1), minlength=n)
    low = (deg[e[:, 0]] < deg[e[:, 1]]) | ((deg[e[:, 0]] == deg[e[:, 1]]) & (e[:, 0] < e[:, 1]))
    u = np.where(low, e[:, 0], e[:, 1])
    v = np.where(low, e[:, 1], e[:, 0])
    out = np.bincount(u, minlength=n)
    un, vn = out[u], out[v]
    sn, ln = np.minimum(un, vn), np.maximum(un, vn)
    probes = np.ceil(np.log2(ln + 1.0))
    adj = int((28 + 4 * sn + 4 * sn * probes).sum())
    return adj, 8 + 216 + 24


def main():
    import torch
    reps = 3
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"card": q.stdout.strip()}
    print("card", res["card"], flush=True)
    torch.zeros(1, device="cuda")
    lib = api.load_library()
    Rt, pairs, rec, out_pair = covisibility(np.random.default_rng(0))
    n, P = len(Rt), len(pairs)
    print("graph: %d cameras, %d pairs" % (n, P), flush=True)
    bufs = api._DevBuffers(lib)
    try:
        d_rec = bufs.upload(rec)
        d_kept = bufs.alloc(P * 128)
        prm = api._view_graph_params(max_cycle_error=3.0, min_inliers=0)
        keep = np.zeros(P, np.uint8)
        st = np.zeros(P, api.CYCLE_STATS_DTYPE)
        rep = api.PsViewGraphReport()
        c_pairs = api._c_pairs(pairs)

        def call():
            rc = lib.ps_view_graph_filter(0, n, P, c_pairs, d_rec, C.byref(prm), keep.ctypes.data, st.ctypes.data, d_kept, C.byref(rep))
            api._check(lib, rc, "ps_view_graph_filter")

        ms, times = tb.timed(call, reps)
        names = {"adjacency": ("vg_used_kernel", "vg_orient_kernel", "vg_gather_kernel", "radix_", "scan_"),
                 "enumeration": ("vg_enum_kernel",), "decision": ("vg_decide_kernel", "vg_compact_kernel")}
        kern = tb.kernel_ms(call, names)
        adj_bytes, per_tri = enumeration_bytes(n, pairs)
        enum_bytes = adj_bytes + per_tri * rep.n_triangles
        k = keep.astype(bool)
        res["filter"] = {"cameras": n, "pairs": P, "outlier_pairs": int(out_pair.sum()), "triangles": rep.n_triangles,
                         "consistent_triangles": rep.n_consistent_triangles, "kept": rep.n_kept, "untested": rep.n_untested,
                         "outliers_kept": int(k[out_pair].sum()), "inliers_dropped": int((~k[~out_pair]).sum()),
                         "ms_per_call_median": ms, "ms_all": times, "kernel_ms": kern,
                         "triangles_per_s_enumeration": rep.n_triangles / (kern["enumeration"] * 1e-3) if kern["enumeration"] else None,
                         "enumeration_adjacency_bytes": adj_bytes, "enumeration_bytes_with_triangles": enum_bytes,
                         "enumeration_share_of_hbm": enum_bytes / (kern["enumeration"] * 1e-3) / PEAK_BW if kern["enumeration"] else None}
        print(json.dumps(res["filter"]), flush=True)
        # rotation averaging with global_bench.py's parameters, on all pairs and on the kept ones
        rprm = api._rotation_params(loss="cauchy", loss_scale=2.0, max_iters=5, step_tol=0.0, cg_max_iters=50, cg_tol=1e-10, min_inliers=0)
        R0 = api._rotation_dev(lib, 0, n, pairs, d_rec, rprm)[0]
        R1 = api._rotation_dev(lib, 0, n, [pairs[p] for p in np.flatnonzero(k)], d_kept, rprm)[0]
        e0, e1 = go.rotation_errors(R0, Rt), go.rotation_errors(R1, Rt)
        res["rotation_averaging"] = {"all_pairs_err_deg_median_max": [float(np.median(e0)), float(e0.max())],
                                     "kept_pairs_err_deg_median_max": [float(np.median(e1)), float(e1.max())]}
        print(json.dumps(res["rotation_averaging"]), flush=True)
    finally:
        bufs.free()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
