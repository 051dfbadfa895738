"""ps_global_positioning and ps_rotation_averaging on triangulate_bench's SfM-scale graph, with card name and power limit.

  Positioning: the graph's 1 000 cameras, 2 M tracks and about 7.4 M observations (0.5 px noise, 10 % outlier
  observations) under the true rotations turned by 0.1 degree, every set registered; a fixed number of iterations
  (function_tol = 0) with a fixed CG budget.  Rotation averaging: the co-visibility graph of the same cameras (the
  distinct pairs of consecutive members of the tracks, n_front = the tracks they share), relative rotations with 0.5
  degree noise and 10 % replaced by random rotations.  Reported: median ms per call (inputs on the device, ending in a
  synchronise) and per iteration, kernel time per pass (torch.profiler), the matvec pass's algorithmic bytes against
  3.35 TB/s (the H100 SXM data sheet), accuracy against the truth after alignment; as labelled context, the numpy oracle
  with dense solves on a small problem on one core.

    python tools/global_bench.py [--reps N] [--iters K] [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

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
# one CG matvec pass, counted from gl_point_kernel<1> and gl_cam_kernel<1>: per member, on each side, its weight (8), its
# ends (8) and the other node's p (24), and the camera side's list entry (4); per node p and D read, q written (56)
MATVEC_PER_MEMBER, MATVEC_PER_NODE = 2 * (8 + 8 + 24) + 4, 24 + 8 + 24


def main():
    import torch
    reps, iters, cg_iters = 3, 5, 50
    args = sys.argv[1:]
    if "--reps" in args:
        i = args.index("--reps"); reps = int(args[i + 1]); del args[i:i + 2]
    if "--iters" in args:
        i = args.index("--iters"); iters = int(args[i + 1]); del args[i:i + 2]
    out_path = args[0] if args else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"card": q.stdout.strip()}
    print("card", res["card"], flush=True)
    torch.zeros(1, device="cuda")
    lib = api.load_library()
    rng = np.random.default_rng(0)
    t0 = time.perf_counter()
    g = tb.make_graph(rng)
    print("graph built in %.1f s" % (time.perf_counter() - t0), flush=True)
    truth = g["poses"]
    n = len(g["n_feat"])
    Rt = np.stack([np.asarray(R) for R, _ in truth])
    Rn = np.ascontiguousarray(np.stack([bo.small_rotation(rng, 0.1) @ R for R in Rt]))
    reg = np.ones(n, np.uint8)
    # the co-visibility graph of the tracks
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
    bufs = api._DevBuffers(lib)
    try:
        dev = tb.Device(lib, g, bufs)
        d_X = bufs.alloc(dev.T * 24)
        prm = api._position_params(loss="huber", loss_scale=0.1, max_iters=iters, function_tol=0.0, cg_max_iters=cg_iters, cg_tol=1e-10)
        poses = (api.PsRigid * n)()
        pos = np.zeros(n, np.uint8)
        rep = api.PsPositionReport()

        def call():
            rc = lib.ps_global_positioning(0, n, dev.c_nf, dev.c_feat, dev.cams.ctypes.data, Rn.ctypes.data, reg.ctypes.data, dev.T, dev.d_st,
                                           dev.d_mem, dev.M, C.byref(prm), poses, pos.ctypes.data, d_X, C.byref(rep))
            api._check(lib, rc, "ps_global_positioning")

        ms, times = tb.timed(call, reps)
        names = {"matvec": ("gl_point_kernel<1>", "gl_cam_kernel<1>"), "cg_other": ("gl_cg_",), "rhs": ("gl_point_kernel<0>", "gl_cam_kernel<0>"),
                 "lin": ("gp_lin_kernel",), "setup": ("gp_check_kernel", "gp_track_kernel", "radix_", "scan_", "gp_iota_kernel"),
                 "other": ("gp_move_kernel", "gp_out_kernel", "gl_cost_kernel")}
        kern = tb.kernel_ms(call, names)
        C_est = np.stack([-np.asarray(poses[i].R[:]).reshape(3, 3).T @ np.asarray(poses[i].t[:]) for i in range(n)])
        C_true = np.stack([-np.asarray(R).T @ np.asarray(t) for R, t in truth])
        err = np.linalg.norm(go.align_centres(C_est, C_true) - C_true, axis=1) / np.linalg.norm(C_true - C_true.mean(0), axis=1).max()
        solves = rep.iterations + 1
        matvec_bytes = MATVEC_PER_MEMBER * dev.M + MATVEC_PER_NODE * (n + dev.T)
        mv_ms = kern.get("matvec", 0.0) / max(rep.cg_iterations, 1)
        res["positioning"] = {"cameras": n, "tracks": dev.T, "members": dev.M, "observations": rep.n_obs, "iterations": rep.iterations,
                              "solves": solves, "cg_iterations": rep.cg_iterations, "ms_per_call_median": ms, "ms_all": times,
                              "ms_per_iteration": ms / solves, "kernel_ms": kern, "kernel_ms_per_cg_iteration":
                              (kern.get("matvec", 0.0) + kern.get("cg_other", 0.0)) / max(rep.cg_iterations, 1),
                              "matvec_bytes_per_pass": matvec_bytes, "matvec_ms_per_pass": mv_ms,
                              "matvec_share_of_hbm": matvec_bytes / (mv_ms * 1e-3) / PEAK_BW if mv_ms else None,
                              "cost": [rep.initial_cost, rep.final_cost], "centre_err_over_scene_median_max": [float(np.median(err)), float(err.max())]}
        print(json.dumps(res["positioning"]), flush=True)
        d_rec = bufs.upload(rec)
        rprm = api._rotation_params(loss="cauchy", loss_scale=2.0, max_iters=iters, step_tol=0.0, cg_max_iters=cg_iters, cg_tol=1e-10, min_inliers=0)
        rep_r = []

        def rcall():
            rep_r[:] = [api._rotation_dev(lib, 0, n, pairs, d_rec, rprm)]

        rms, rtimes = tb.timed(rcall, reps)
        rkern = tb.kernel_ms(rcall, {"matvec": ("gl_cam_kernel<1>",), "cg_other": ("gl_cg_",), "lin": ("gl_rot_",)})
        R_est, _, _, rrep = rep_r[0]
        rerr = go.rotation_errors(R_est, Rt)
        res["rotation_averaging"] = {"cameras": n, "pairs": len(pairs), "outlier_pairs": int(out_pair.sum()), "iterations": rrep.iterations,
                                     "cg_iterations": rrep.cg_iterations, "ms_per_call_median": rms, "ms_all": rtimes,
                                     "ms_per_iteration": rms / max(rrep.iterations, 1), "kernel_ms": rkern,
                                     "rotation_err_deg_median_max": [float(np.median(rerr)), float(rerr.max())]}
        print(json.dumps(res["rotation_averaging"]), flush=True)
    finally:
        bufs.free()
    # context: the numpy oracle with dense solves on a 6-camera, 300-track problem, one core
    sc = bo.planted(np.random.default_rng(1), 6, list(np.random.default_rng(2).integers(2, 7, size=300)), noise=0.5)
    P = go.Positioning(sc["feats"], sc["cams"], np.stack([np.asarray(R) for R, _ in sc["poses_true"]]), np.ones(6, bool), sc["start"],
                       sc["members"])
    t0 = time.perf_counter()
    P.run(max_iters=iters, function_tol=0.0)
    res["context_numpy_dense_oracle_one_core"] = {"cameras": 6, "tracks": 300, "iterations": iters, "s": time.perf_counter() - t0}
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
