"""ps_bundle_adjust on triangulate_bench's SfM-scale graph, with card name and power limit.

  The graph: 1 000 posed cameras, 2 M tracks, about 7.4 M observations (0.5 px noise, 10 % outliers).  Poses 1 .. 999 are
  turned by 0.1 degree and moved by 0.02 (0.2 % of the camera distance); ps_triangulate_tracks gives the points and masks;
  then ps_bundle_adjust (Huber loss, s = 2 px, camera 0 fixed, t[2] of camera 1 held) runs a fixed number of LM
  iterations (function_tol = 0) with a fixed CG budget.  Reported: median ms per call (inputs on the device, ending in a
  synchronise), ms per LM iteration and per CG iteration, kernel time per pass (torch.profiler), the passes' algorithmic
  bytes and FP64 operations counted here against 3.35 TB/s and 34 TFLOP/s FP64 (the H100 SXM data sheet) with the bound
  that is nearer, the cost and termination; and, as labelled context, the numpy oracle's dense LM on a sub-problem of 20
  cameras on one core.

    python tools/bundle_bench.py [--reps N] [--iters K] [out.json]
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
import triangulate_bench as tb      # noqa: E402
from popsift_b200 import api        # noqa: E402

PEAK_FP64 = 34e12
PEAK_BW = 3.35e12
OBS = 160            # bytes of one stored observation (sqrt(w) Jc, Jp, e in double)

# Per used observation and pass, (bytes, FP64 operations) counted from the kernels: the stored record is read once per
# pass that uses it; the gathers (a camera's 6-vector, a point's 3-vector, the index) are counted once per observation.
PASSES = {
    "linearize": (OBS + 4 * 4 + 8 + 24 + 8, 160),                  # writes the record; reads indices, pixel, point
    "cam_grad": (OBS + 4, 27 * 4),                                  # U (21) and g (6): 2 mul + 2 add each
    "point": (6 * 8 + 8 * 2 + 8, 9 * 4),                           # Jp, e; V (6), g (3)
    "cam_precond": (OBS + 4 + 4 + 72, 6 * 3 * 4 + 12 * 4 + 21 * 4 + 12 + 6 * 4),
    "point_matvec": (OBS - 16 + 48 + 4, 12 * 2 + 6 * 4),           # Jc, Jp; p_set gather
    "cam_matvec": (OBS - 16 + 24 + 8, 12 + 6 * 4),                 # Jc, Jp; y_track gather
    "point_back": (2 * (OBS - 16) + 2 * 48 + 8, 2 * 24 + 6 * 4 + 12),
    "cost": (4 * 3 + 8 + 24 + 8, 40),
}


def main():
    import torch
    reps, iters, cg_iters = 3, 5, 25
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
    pert = [truth[0]]
    for R, t in truth[1:]:
        pert.append((bo.small_rotation(rng, 0.1) @ R, t + rng.normal(scale=0.02 / np.sqrt(3), size=3)))
    t1 = np.array(pert[1][1]); t1[2] = truth[1][1][2]
    pert[1] = (pert[1][0], t1)
    g["poses"] = pert
    n = len(g["n_feat"])
    fixed = (C.c_uint8 * n)(*([1] + [0] * (n - 1)))
    bufs = api._DevBuffers(lib)
    try:
        dev = tb.Device(lib, g, bufs)
        dev.call(api._tri_params(max_error=4.0, min_angle=1.5, n_samples=256, refine_iters=10))
        counts = dict(zip(api.TRI_STATUS, [int(v) for v in dev.cnt.n_status]))
        print("triangulated", counts, flush=True)
        pts0 = bufs.download(dev.d_pts, dev.T, api.TRACK_POINT_DTYPE)
        d_pts = bufs.alloc(dev.T * 40)
        d_err = bufs.alloc(dev.M * 4)
        prm = api._bundle_params(loss="huber", loss_scale=2.0, max_iters=iters, function_tol=0.0, cg_max_iters=cg_iters, cg_tol=1e-8,
                                 scale_set=1, scale_axis=2)
        out = (api.PsRigid * n)()
        rep = api.PsBundleReport()

        def call():
            if lib.ps_host_to_dev(d_pts, pts0.ctypes.data, pts0.nbytes) != 0:
                raise RuntimeError("upload")
            rc = lib.ps_bundle_adjust(0, n, dev.c_nf, dev.c_feat, dev.cams.ctypes.data, dev.rig, dev.T, dev.d_st, dev.d_mem, dev.M,
                                      d_pts, dev.d_mask, fixed, C.byref(prm), out, d_err, C.byref(rep))
            api._check(lib, rc, "ps_bundle_adjust")

        ms, times = tb.timed(call, reps)
        report = api._bundle_report(rep)._asdict()
        print(json.dumps(report), flush=True)
        names = {k: ("ba_%s_kernel" % k,) for k in PASSES}
        names.update(cg_update=("ba_cg_update_kernel",), setup=("ba_check_kernel", "ba_flag_kernel", "ba_compact_kernel", "radix_", "scan_",
                                                                  "ba_iota_kernel"), other=("ba_cg_init_kernel", "ba_cam_update_kernel",
                                                                                            "ba_reduce_kernel", "ba_final_kernel"))
        kern = tb.kernel_ms(call, names)
        rot0, cen0 = bo.pose_errors(pert, truth)
        rot1, cen1 = bo.pose_errors([(np.array(out[i].R[:]).reshape(3, 3), np.array(out[i].t[:])) for i in range(n)], truth)
    finally:
        bufs.free()
    U, T = report["n_obs"], dev.T
    n_lin = report["accepted"] + 1 if report["accepted"] < report["iterations"] else report["accepted"]
    calls = {"linearize": n_lin, "cam_grad": n_lin, "point": report["iterations"], "cam_precond": report["iterations"],
             "point_matvec": report["cg_iterations"], "cam_matvec": report["cg_iterations"], "point_back": report["iterations"],
             "cost": report["iterations"] + 1}
    roof = {}
    for k, (b, f) in PASSES.items():
        tot_b, tot_f = float(b) * U * calls[k], float(f) * U * calls[k]
        s = kern.get(k, 0.0) * 1e-3
        roof[k] = {"launches": calls[k], "kernel_ms": kern.get(k, 0.0), "bytes": tot_b, "fp64_ops": tot_f,
                   "share_of_hbm": tot_b / s / PEAK_BW if s else None, "share_of_fp64": tot_f / s / PEAK_FP64 if s else None,
                   "nearer_bound": ("bytes" if tot_b / PEAK_BW > tot_f / PEAK_FP64 else "fp64")}
    cg_kernel_ms = kern["point_matvec"] + kern["cam_matvec"] + kern["cg_update"]
    res["synthetic"] = {"cameras": n, "tracks": T, "members": dev.M, "used_observations": U, "lm_iterations": report["iterations"],
                        "cg_iterations": report["cg_iterations"], "ms_per_call_median": ms, "ms_all": times,
                        "ms_per_lm_iteration": ms / max(report["iterations"], 1),
                        "kernel_ms_per_cg_iteration": cg_kernel_ms / max(report["cg_iterations"], 1), "kernel_ms": kern,
                        "passes": roof, "report": report, "triangulate_counts": counts,
                        "rotation_err_deg_before_after_median": [float(np.median(rot0[1:])), float(np.median(rot1[1:]))],
                        "centre_err_before_after_median": [float(np.median(cen0[1:])), float(np.median(cen1[1:]))]}
    print(json.dumps(res["synthetic"]), flush=True)
    # context: the dense numpy oracle on 20 cameras' tracks, one core
    sub_cams = 20
    sc = bo.planted(np.random.default_rng(1), sub_cams, list(np.random.default_rng(2).integers(2, 8, size=400)), noise=0.5, rot_deg=0.1,
                    trans=0.02)
    bo.gauge_to_truth(sc, 0, 1, 2)
    f = np.zeros(sub_cams, np.uint8); f[0] = 1
    prob = bo.problem(sc, f, loss_kind="huber", loss_scale=2.0, scale_set=1, scale_axis=2)
    t0 = time.perf_counter()
    _, _, orep = bo.lm(prob, sc["poses"], sc["X0"], max_iters=iters, function_tol=0.0)
    res["context_numpy_dense_oracle_one_core"] = {"cameras": sub_cams, "observations": int(len(prob.set)), "parameters": prob.n,
                                                  "lm_iterations": orep["iterations"], "s": time.perf_counter() - t0}
    print(json.dumps(res["context_numpy_dense_oracle_one_core"]), flush=True)
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
