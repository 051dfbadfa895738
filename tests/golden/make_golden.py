"""Turns the raw outputs of the UNMODIFIED reference (run on a B200 by
tools/gpu_ref_golden.sh through oracle/_ref/ref_dump and oracle/_ref/texprobe,
results in ref_out/ref1/) into the small committed fixtures in tests/golden/.

    bash tools/gpu_ref_golden.sh                       (on a GPU machine)
    python tests/golden/make_golden.py ref_out/ref1

Fixtures:
  planes_f256.npz     sha256 of every Gaussian / DoG plane of the 256x192 frame (seed 3), full
                      planes of octaves >= 2, geometry
  feat_*.npz          reference features (+descriptors) for the named frame / config
  texture_pairs.npz   what the B200 texture unit returns for the reference's input texture
                      configuration: fraction-0 for 256 values, fraction-0.5 for all (a,b) pairs
"""
import hashlib
import json
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as ol  # noqa: E402


def main(src):
    # planes
    out = {}
    meta = {}
    for kind, sub, pat in (("g", "dir-octave-dump", "pyramid-o-%d-l-%d.dump"), ("d", "dir-dog-dump", "d-pyramid-o-%d-l-%d.dump")):
        for o in range(20):
            for l in range(12):
                fn = os.path.join(src, "log256", sub, pat % (o, l))
                if not os.path.exists(fn):
                    continue
                p = ol.read_ref_dump(fn)
                meta["%s_%d_%d" % (kind, o, l)] = {"shape": list(p.shape), "sha256": hashlib.sha256(p.tobytes()).hexdigest(),
                                                   "sum": float(p.astype(np.float64).sum())}
                if o >= 2:
                    out["%s_%d_%d" % (kind, o, l)] = p
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "planes_f256.npz"), **out)
    # features
    for name, with_desc in (("f256_popsift_rs", True), ("log256/feat_vl_classic", True), ("f640_popsift_rs_a", True),
                            ("f640_popsift_rs_b", False), ("f640_vlfeat_classic_a", True), ("f640_vlfeat_classic_b", False),
                            ("f640_ds0", True), ("f1080_popsift_rs", False), ("f1080_vlfeat_classic", False)):
        feat, desc = ol.read_ref_features(os.path.join(src, name + ".bin"))
        key = name.replace("log256/feat_vl_classic", "f256_vlfeat_classic")
        d = {"feat": feat}
        if with_desc:
            d["desc"] = desc.astype(np.float32)
        else:
            d["n_desc"] = np.array([len(desc)])
        np.savez_compressed(os.path.join(HERE, "feat_%s.npz" % key), **d)
    # texture pairs
    data = open(os.path.join(src, "tex_pairs.bin"), "rb").read()
    n = struct.unpack_from("i", data, 0)[0]
    x = np.frombuffer(data, np.float32, n, 4)
    n2 = struct.unpack_from("i", data, 4 + 4 * n)[0]
    y = np.frombuffer(data, np.float32, n2, 8 + 4 * n)
    np.savez_compressed(os.path.join(HERE, "texture_pairs.npz"), x_half=x[:65536].reshape(256, 256),
                        frac0=x[65536:], y_half=y.reshape(256, 256))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "ref_out/ref1")
