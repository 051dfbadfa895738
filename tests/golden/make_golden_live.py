"""Fixtures of the reference runs the GPU parity tests compare against (tests/golden/live/*.npz).

Runs the UNMODIFIED reference (oracle/_ref/ref_dump, built by `make -C oracle ref` from the reference's sources) on
the same seeded frames and options as the tests and keeps, per run, what the tests compare with -- small enough to
commit:
  feat          every feature (ol.REF_FEATURE_DTYPE), all orientations
  desc_rows     a fixed, seeded sample of MAX_DESC descriptor rows (all rows for the affine set) and `desc`, their values
  n_desc        the reference's descriptor count
  planes        JSON {"o_l": [rows, cols, sha256]} of the --log plane dumps the test compares bit for bit
bench32.npz holds the 32 benchmark frames (octaves=5, levels=3): per frame the counts and the sha256 of the sorted
keypoint keys, orientation counts and angles, and a sample of 16 descriptors per frame.

stress_*.npz / knob_*.npz are runs on the adversarial images of tests/stress_images.py (STRESS_RUNS), with the octave-0
planes of their --log dumps.

    python tests/golden/make_golden_live.py OUTDIR [--only 'stress_*']   (on a GPU machine, with oracle/_ref/ref_dump built)
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import oracle_lib as ol  # noqa: E402
from popsift_b200.synth import affine_set, make_frame, write_pgm  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "ref_dump")
MAX_DESC = 256            # descriptor rows kept per run (the affine runs keep all: their test matches descriptors)


def vlc(*extra):
    return ["--mode", "vlfeat", "--norm", "classic"] + list(extra)


def prs(*extra):
    return ["--mode", "popsift", "--norm", "rootsift"] + list(extra)


# name -> (w, h, seed, ref_dump arguments, octaves whose --log planes are kept)
RUNS = {
    # test_live_against_reference_library
    "lib_1920x1080_101": (1920, 1080, 101, vlc(), 0),
    "lib_1920x1080_102": (1920, 1080, 102, prs(), 0),
    "lib_800x600_21": (800, 600, 21, vlc("--downsampling", "0"), 0),
    "lib_3840x2160_7": (3840, 2160, 7, vlc("--octaves", "5"), 0),
    "lib_800x600_22": (800, 600, 22, vlc("--gauss-mode", "opencv"), 0),
    "lib_640x480_23": (640, 480, 23, prs("--gauss-mode", "opencv", "--sigma", "1.2", "--levels", "4"), 0),
    "lib_700x500_24": (700, 500, 24, vlc("--downsampling", "-0.5"), 0),
    "lib_640x480_25": (640, 480, 25, prs("--downsampling", "0.5"), 0),
    "lib_641x479_26": (641, 479, 26, vlc("--downsampling", "1"), 0),
    # test_descriptor_modes_vs_reference (default Config)
    "desc_iloop": (640, 480, 1, ["--desc-mode", "iloop"], 0),
    "desc_grid": (640, 480, 1, ["--desc-mode", "grid"], 0),
    "desc_igrid": (640, 480, 1, ["--desc-mode", "igrid"], 0),
    "desc_notile": (640, 480, 1, ["--desc-mode", "notile"], 0),
    # test_level0_planes_bit_exact_vs_live_reference (default Config, octaves=2)
    "l0_700x500_24": (700, 500, 24, ["--octaves", "2", "--downsampling", "-0.5"], 2),
    "l0_640x480_27": (640, 480, 27, ["--octaves", "2", "--downsampling", "-1.5"], 2),
    "l0_641x479_26": (641, 479, 26, ["--octaves", "2", "--downsampling", "1"], 2),
    "l0_5000x96_28": (5000, 96, 28, ["--octaves", "2"], 2),
    "l0_4096x64_29": (4096, 64, 29, ["--octaves", "2"], 2),
    "l0_1000x700_30": (1000, 700, 30, ["--octaves", "2", "--downsampling", "0"], 2),
    # the other scaling / Gauss modes
    "direct_scaling": (640, 480, 31, vlc("--direct-scaling"), 3),
    "gauss_vlfeat_direct": (640, 480, 33, vlc("--gauss-mode", "vlfeat-direct"), 2),
    "gauss_relative": (640, 480, 35, vlc("--gauss-mode", "relative"), 3),
    "gauss_fixed9": (640, 480, 37, vlc("--gauss-mode", "fixed9"), 3),
    "gauss_fixed15": (640, 480, 37, vlc("--gauss-mode", "fixed15"), 3),
    "direct_relative": (512, 384, 39, vlc("--gauss-mode", "relative", "--direct-scaling"), 3),
    "direct_fixed9": (512, 384, 39, vlc("--gauss-mode", "fixed9", "--direct-scaling"), 3),
    "direct_fixed15": (512, 384, 39, vlc("--gauss-mode", "fixed15", "--direct-scaling"), 3),
    "direct_vlfeat-direct": (512, 384, 39, vlc("--gauss-mode", "vlfeat-direct", "--direct-scaling"), 3),
}


def ocv(*extra):
    return ["--mode", "opencv", "--norm", "classic"] + list(extra)


# name -> (tests/stress_images.py image, ref_dump arguments): test_stress_parity.py::test_stress_vs_reference_runs
STRESS_RUNS = {
    "stress_checker_p8_prs": ("checker_p8", prs()),
    "stress_checker_p8_ocv": ("checker_p8", ocv()),
    "stress_checker_rot30_p6_prs": ("checker_rot30_p6", prs()),
    "stress_checker_rot30_p6_vlc": ("checker_rot30_p6", vlc()),
    "stress_block_noise_4_prs": ("block_noise_4", prs()),
    "stress_block_noise_4_ocv": ("block_noise_4", ocv()),
    "stress_block_noise_4_vlc": ("block_noise_4", vlc()),
    "stress_binary_noise_vlc": ("binary_noise", vlc()),
    "stress_saturated_prs": ("saturated", prs()),
    "stress_dark_prs": ("dark", prs("--threshold", "0.001")),
    "stress_border_impulses_prs": ("border_impulses", prs()),
    "stress_border_impulses_ocv": ("border_impulses", ocv()),
    "stress_step_edges_vlc": ("step_edges", vlc()),
    # the Config knobs structure-from-motion callers set
    "knob_threshold_0.005": ("saturated", prs("--threshold", "0.005")),
    "knob_threshold_0.1": ("saturated", prs("--threshold", "0.1")),
    "knob_edge_2": ("saturated", prs("--edge-limit", "2")),
    "knob_edge_50": ("saturated", prs("--edge-limit", "50")),
    "knob_iblur_0": ("saturated", prs("--initial-blur", "0")),
    "knob_iblur_1": ("saturated", prs("--initial-blur", "1")),
    "knob_iblur_1_block_noise_4": ("block_noise_4", prs("--initial-blur", "1")),
    "knob_nm9_rs": ("block_noise_4", prs("--norm-multi", "9")),
    "knob_nm3_classic": ("block_noise_4", vlc("--norm-multi", "3")),
    "knob_sigma2_l2": ("checker_rot30_p6", prs("--sigma", "2.0", "--levels", "2")),
}


def sample_rows(n, seed, keep_all=False):
    if keep_all or n <= MAX_DESC:
        return np.arange(n, dtype=np.int64)
    return np.sort(np.random.default_rng(seed).choice(n, MAX_DESC, replace=False)).astype(np.int64)


def save_run(path, feat, desc, planes, seed, keep_all=False):
    rows = sample_rows(len(desc), seed, keep_all)
    np.savez_compressed(path, feat=feat, desc_rows=rows, desc=desc[rows], n_desc=np.array([len(desc)]),
                        planes=np.frombuffer(json.dumps(planes, sort_keys=True).encode(), np.uint8))


def run_one(td, img, args, log_octaves):
    pgm = os.path.join(td, "f.pgm")
    write_pgm(pgm, img)
    subprocess.run([REF, "-i", "f.pgm", "-o", "f.bin"] + args + (["--log"] if log_octaves else []), cwd=td, check=True,
                   capture_output=True)
    feat, desc = ol.read_ref_features(os.path.join(td, "f.bin"))
    planes = {}
    for oc in range(log_octaves):
        for lv in range(6):
            fn = os.path.join(td, "dir-octave-dump", "pyramid-o-%d-l-%d.dump" % (oc, lv))
            if lv == 5 and not os.path.exists(fn):         # levels = 2: five Gaussian planes per octave
                break
            p = ol.read_ref_dump(fn)
            planes["%d_%d" % (oc, lv)] = [p.shape[0], p.shape[1], hashlib.sha256(p.tobytes()).hexdigest()]
    return feat, desc, planes


def bench32(out):
    import bench
    frames = bench.synth_frames(32, 0)
    rec = {k: [] for k in ("counts", "keys_sha", "num_ori_sha", "ori_sha")}
    skeys, sori, sdesc = [], [], []
    with tempfile.TemporaryDirectory() as td:
        cmd = [REF, "--octaves", "5", "--levels", "3", "-o", os.path.join(td, "ref")]
        for i, f in enumerate(frames):
            write_pgm(os.path.join(td, "f%d.pgm" % i), f)
            cmd += ["-i", os.path.join(td, "f%d.pgm" % i)]
        subprocess.run(cmd, check=True, capture_output=True)
        for i in range(len(frames)):
            rf, rd = ol.read_ref_features(os.path.join(td, "ref.%d" % i))
            keys = bench32_keys(rf)
            order = np.lexsort(keys.T[::-1])
            rec["counts"].append([len(rf), len(rd)])
            rec["keys_sha"].append(hashlib.sha256(keys[order].tobytes()).hexdigest())
            rec["num_ori_sha"].append(hashlib.sha256(rf["num_ori"][order].astype("<i4").tobytes()).hexdigest())
            rec["ori_sha"].append(hashlib.sha256(rf["ori"][order].astype("<f4").tobytes()).hexdigest())
            # 16 (keypoint, orientation 0) descriptors per frame
            pick = np.random.default_rng(1000 + i).choice(len(rf), 16, replace=False)
            skeys.append(np.concatenate([np.full((16, 1), i, np.int64), keys[pick]], axis=1))
            sori.append(rf["ori"][pick, 0])
            sdesc.append(rd[rf["desc_idx"][pick, 0]])
    np.savez_compressed(os.path.join(out, "bench32.npz"), sample_keys=np.concatenate(skeys), sample_desc=np.concatenate(sdesc),
                        meta=np.frombuffer(json.dumps(rec).encode(), np.uint8))


def bench32_keys(feat):
    """(octave, x bits, y bits, sigma bits) per keypoint, int64 -- the identity the bench32 test pairs keypoints by"""
    return np.stack([feat["octave"].astype(np.int64), feat["x"].view(np.int32).astype(np.int64),
                     feat["y"].view(np.int32).astype(np.int64), feat["sigma"].view(np.int32).astype(np.int64)], axis=1)


def main():
    import argparse
    import fnmatch
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--only", default="*", help="make only the runs whose name matches this shell pattern, e.g. 'stress_*'")
    a = ap.parse_args()
    out = a.out
    os.makedirs(out, exist_ok=True)
    want = lambda name: fnmatch.fnmatchcase(name, a.only)   # noqa: E731
    # the sample seed of a run is its index in the sorted table: the stress / knob runs are numbered separately so that
    # adding them left the earlier fixtures unchanged
    for k, (name, (w, h, seed, args, log_oc)) in enumerate(sorted(RUNS.items())):
        if not want(name):
            continue
        with tempfile.TemporaryDirectory() as td:
            feat, desc, planes = run_one(td, make_frame(w, h, seed), args, log_oc)
        save_run(os.path.join(out, name + ".npz"), feat, desc, planes, k)
        print(name, len(feat), len(desc), flush=True)
    import stress_images
    for k, (name, (img_name, args)) in enumerate(sorted(STRESS_RUNS.items())):
        if not want(name):
            continue
        with tempfile.TemporaryDirectory() as td:
            feat, desc, planes = run_one(td, stress_images.image(img_name), args, 1)
        save_run(os.path.join(out, name + ".npz"), feat, desc, planes, 500 + k)
        print(name, len(feat), len(desc), flush=True)
    for k, (im, _A) in enumerate(affine_set(), 1):
        if not want("aff%d" % k):
            continue
        with tempfile.TemporaryDirectory() as td:
            feat, desc, planes = run_one(td, im, vlc(), 0)
        save_run(os.path.join(out, "aff%d.npz" % k), feat, desc, planes, 100 + k, keep_all=True)
        print("aff%d" % k, len(feat), len(desc), flush=True)
    if want("bench32"):
        bench32(out)
        print("bench32 done", flush=True)


if __name__ == "__main__":
    main()
