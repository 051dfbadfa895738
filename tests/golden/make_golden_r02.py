"""Round-2 fixtures: turns the raw outputs of the UNMODIFIED reference (run on a B200 by
tools/gpu_ref_golden_r02.sh through oracle/_ref/ref_dump and oracle/_ref/texprobe, results in
ref_out/ref2/) into the small committed files in tests/golden/.

    bash tools/gpu_ref_golden_r02.sh                   (on a GPU machine)
    python tests/golden/make_golden_r02.py ref_out/ref2

Fixtures:
  texture_float.npz            what the B200 texture unit returns for the reference's FLOAT input texture
                               (ImageFloat): a random 64x64 float image, 2x2 blends at a 16x16 grid of
                               fractions for 16x32 texels, and the fraction quantisation of one texel row
  texture_u8_general.npz       the 8-bit input texture at a 16x16 grid of general fractions (`texprobe upairs`)
  planes_f256_float.npz        sha256 (+ data of two) of the planes the float-mode reference run dumped
  feat_*_opencv_*.npz          Config::OpenCV SiftMode
  feat_*_float_*.npz           PopSift::FloatImages (pixels = u8 / 256)
  feat_aff{1..6}_vlfeat_classic.npz   synthetic affine set (BASELINE configs[4] stand-in); descriptors for 1, 2
  feat_f256_desc_*.npz, feat_f256_direct.npz   descriptor modes / direct scaling (for when they are built)
  match_*.npz                  FeaturesDev::match: device-resident features, descriptors, reverse maps of both
                               images and the parsed "accept/reject" lines of the reference's device printf
  filter_*.npz                 grid filter runs (when present)
  bench32_parity.json          the 32 benchmark frames: per-frame counts of two reference runs (its run-to-run
                               jitter: none) and of this library at the time the fixture was made
"""
import glob
import hashlib
import json
import os
import re
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as ol  # noqa: E402

LINE = re.compile(r"(accept|reject) feat\s*(\d+) \[\s*(\d+)\] matches feat\s*(\d+) \[\s*(\d+)\] \( 2nd feat\s*(\d+) \[\s*(\d+)\] \) dist ([0-9.eE+-]+|inf|nan) vs ([0-9.eE+-]+|inf|nan)")


def save_feat(src, name, key, with_desc=True):
    fn = os.path.join(src, name)
    if not os.path.exists(fn):
        return False
    feat, desc = ol.read_ref_features(fn)
    d = {"feat": feat}
    if with_desc:
        d["desc"] = desc.astype(np.float32)
    else:
        d["n_desc"] = np.array([len(desc)])
    np.savez_compressed(os.path.join(HERE, "feat_%s.npz" % key), **d)
    return True


def main(src):
    # ---- float texture probe
    fn = os.path.join(src, "tex_fpairs.bin")
    if os.path.exists(fn):
        data = open(fn, "rb").read()
        W, H, n1, n2 = struct.unpack_from("4i", data, 0)
        img = np.frombuffer(data, np.float32, W * H, 16).reshape(H, W)
        o = np.frombuffer(data, np.float32, n1 + n2, 16 + 4 * W * H)
        grid = o[:n1].reshape(32, 32, 16, 16)[:16]              # texel rows j = 8..23, i = 8..39; [j, i, b, a]
        quant = o[n1:].reshape(4, 32, 1024)[0]                  # j = 8, i = 8..39, a/1024
        np.savez_compressed(os.path.join(HERE, "texture_float.npz"), img=img, grid=grid, quant=quant)
    # ---- 8-bit texture at general fractions
    fn = os.path.join(src, "tex_upairs.bin")
    if os.path.exists(fn):
        data = open(fn, "rb").read()
        W, H, n1, _ = struct.unpack_from("4i", data, 0)
        img = np.frombuffer(data, np.uint8, W * H, 16).reshape(H, W)
        o = np.frombuffer(data, np.float32, n1, 16 + W * H).reshape(32, 32, 16, 16)[:16]
        np.savez_compressed(os.path.join(HERE, "texture_u8_general.npz"), img=img, grid=o)
    # ---- float-mode planes
    meta, keep = {}, {}
    for fn in sorted(glob.glob(os.path.join(src, "logf256", "dir-octave-dump", "*.dump"))):
        b = os.path.basename(fn)
        oc, l = int(b.split("-o-")[1].split("-")[0]), int(b.split("-l-")[1].split(".")[0])
        p = ol.read_ref_dump(fn)
        meta["g_%d_%d" % (oc, l)] = {"shape": list(p.shape), "sha256": hashlib.sha256(p.tobytes()).hexdigest()}
        if oc == 1:
            keep["g_%d_%d" % (oc, l)] = p
    if meta:
        keep["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(HERE, "planes_f256_float.npz"), **keep)
    # ---- features
    for name, key, wd in (("f256_opencv_classic.bin", "f256_opencv_classic", True), ("f640_opencv_rs.bin", "f640_opencv_rs", True),
                          ("logf256/feat.bin", "f256_float_vlfeat_classic", True),
                          ("f640_float_vlfeat_classic.bin", "f640_float_vlfeat_classic", True),
                          ("f640_float_ds0.bin", "f640_float_ds0", True), ("f256_direct.bin", "f256_direct", True)):
        save_feat(src, name, key, wd)
    for dm in ("iloop", "grid", "igrid", "notile"):
        save_feat(src, "f256_desc_%s.bin" % dm, "f256_desc_%s" % dm)
    for k in range(1, 7):
        save_feat(src, "aff%d_vlfeat_classic.bin" % k, "aff%d_vlfeat_classic" % k, with_desc=(k <= 2))
    # ---- grid filter
    for fn in sorted(glob.glob(os.path.join(src, "*_filter_*.bin"))):
        save_feat(src, os.path.basename(fn), os.path.basename(fn)[:-4], with_desc=False)
    # ---- matcher
    for stem in ("match_640", "match_aff12"):
        if not os.path.exists(os.path.join(src, stem + ".txt")):
            continue
        out = {}
        for k in (0, 1):
            feat, desc, rev = ol.read_ref_features(os.path.join(src, "%s.%d" % (stem, k)), with_rev=True)
            out["feat%d" % k], out["desc%d" % k], out["rev%d" % k] = feat, desc, rev
        rows = []
        for ln in open(os.path.join(src, stem + ".txt")):
            m = LINE.search(ln)
            if m:
                rows.append((m.group(1) == "accept", int(m.group(2)), int(m.group(3)), int(m.group(4)), int(m.group(5)),
                             int(m.group(6)), int(m.group(7)), float(m.group(8)), float(m.group(9))))
        out["lines"] = np.array(rows, dtype=[("accept", "?"), ("l_feat", "<i4"), ("l", "<i4"), ("r1_feat", "<i4"), ("r1", "<i4"),
                                             ("r2_feat", "<i4"), ("r2", "<i4"), ("d1", "<f4"), ("d2", "<f4")])
        assert len(rows) == len(out["desc0"]), (stem, len(rows), len(out["desc0"]))
        np.savez_compressed(os.path.join(HERE, "%s.npz" % stem), **out)
    # ---- benchmark-workload parity
    fn = os.path.join(src, "bench_parity.json")
    if os.path.exists(fn):
        r = json.load(open(fn))
        small = {"workload": r["workload"], "totals": r["totals"],
                 "frames": [{"frame": f["frame"], "ours": f["ours"], "ref_a": f["ref_a"], "ref_b": f["ref_b"],
                             "ref_a_vs_ref_b": {k: (len(v) if k == "ori_diffs" else v) for k, v in f["ref_a_vs_ref_b"].items()},
                             "ours_vs_ref_a": {k: (len(v) if k == "ori_diffs" else v) for k, v in f["ours_vs_ref_a"].items()}}
                            for f in r["frames"]]}
        json.dump(small, open(os.path.join(HERE, "bench32_parity.json"), "w"), indent=1)
    # ---- texture coordinates at non-integer scale factors (`texprobe coords 700 500 0.5`, `coords 640 480 1.5`)
    probes = (("a", "tex_c700_up05.bin", 0.5), ("b", "tex_c640_up15.bin", 1.5))
    if all(os.path.exists(os.path.join(src, fn)) for _, fn, _ in probes):
        import struct
        out = {}
        for tag, fn, up in probes:
            data = open(os.path.join(src, fn), "rb").read()
            w, h, W0, H0, nrows, maxoff = struct.unpack_from("6i", data, 0)
            rows = np.frombuffer(data, np.int32, nrows, 24)
            off = 24 + 4 * nrows
            img = np.frombuffer(data, np.uint8, w * h, off).reshape(h, w).copy()
            o = np.frombuffer(data, np.float32, nrows * W0 * (2 * maxoff + 1), off + w * h).reshape(nrows, W0, 2 * maxoff + 1)
            r16 = np.rint(o.astype(np.float64) * 65535).astype(np.int64)          # the unit returns r16 / 65535
            assert ((r16.astype(np.float32) / np.float32(65535)) == o).all()
            sel, xs = [0, 3, 7, 8, 12, 15, 16, 17], np.arange(0, W0, 7)
            out[tag + "_img"], out[tag + "_rows"], out[tag + "_xs"] = img, rows[sel], xs.astype(np.int32)
            out[tag + "_r16"] = r16[sel][:, xs, :].astype(np.uint16)
            out[tag + "_meta"], out[tag + "_up"] = np.array([w, h, W0, H0, maxoff], np.int32), np.float32(up)
        np.savez_compressed(os.path.join(HERE, "texture_coords.npz"), **out)
    # ---- Config::ScaleDirect (ref_dump --direct-scaling --log on the 256x192 frame and on the 640x480 frame of
    # tests/test_gpu_parity.py::test_direct_scaling_vs_oracle_and_live_reference)
    save_feat(src, "ref_direct_f256.bin", "f256_direct")
    save_feat(os.path.dirname(src.rstrip("/")), "ref_direct_640.bin", "f640_direct")
    # --gauss-mode relative, the unnormalized linear float texture probe (`texprobe lcoords`)
    save_feat(src, "ref_relative_f256.bin", "f256_relative")
    save_feat(os.path.dirname(src.rstrip("/")), "ref_vlfeat_direct_640.bin", "f640_vlfeat_direct")
    fn = os.path.join(src, "ref_relative_f256_planes.json")
    if os.path.exists(fn):
        json.dump(json.load(open(fn)), open(os.path.join(HERE, "planes_f256_relative.json"), "w"), indent=0)
    fn = os.path.join(src, "tex_lcoords.bin")
    if os.path.exists(fn):
        import struct
        data = open(fn, "rb").read()
        W, H, n, _ = struct.unpack_from("4i", data, 0)
        q = np.frombuffer(data, np.float32, 2 * n, 16).reshape(n, 2)
        o = np.frombuffer(data, np.float32, n, 16 + 8 * n)
        sel = np.r_[np.arange(0, 17 * 8192, 5), np.arange(17 * 8192, n, 3)]
        np.savez_compressed(os.path.join(HERE, "texture_lcoords.npz"), W=np.int32(W), H=np.int32(H), xy=q[sel], out=o[sel])
    # --gauss-mode fixed9 / fixed15
    for m in ("fixed9", "fixed15"):
        save_feat(src, "ref_%s_f256.bin" % m, "f256_%s" % m)
        fn = os.path.join(src, "ref_%s_f256_planes.json" % m)
        if os.path.exists(fn):
            json.dump(json.load(open(fn)), open(os.path.join(HERE, "planes_f256_%s.json" % m), "w"), indent=0)
    # --gauss-mode vlfeat-direct
    save_feat(src, "ref_vlfeat_direct_f256.bin", "f256_vlfeat_direct")
    fn = os.path.join(src, "ref_vlfeat_direct_f256_planes.json")
    if os.path.exists(fn):
        json.dump(json.load(open(fn)), open(os.path.join(HERE, "planes_f256_vlfeat_direct.json"), "w"), indent=0)
    fn = os.path.join(src, "ref_direct_f256_planes.json")
    if os.path.exists(fn):
        json.dump(json.load(open(fn)), open(os.path.join(HERE, "planes_f256_direct.json"), "w"), indent=0)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "ref_out/ref2")
