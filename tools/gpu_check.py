"""Verbose parity + timing report (diagnostics, not a test; needs a GPU):
    python tools/gpu_check.py > check.txt 2>&1
Compares the CUDA path with the CPU oracle plane by plane, extremum by extremum, and with the
reference library itself (oracle/_ref/ref_dump) when present."""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import compare  # noqa: E402
import oracle_lib as ol  # noqa: E402
from popsift_b200 import api  # noqa: E402
from popsift_b200.synth import make_frame, write_pgm  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref", "ref_dump")


def mk_cfg(mode="popsift", norm="rootsift", downsampling=None, octaves=None):
    c = api.Config()
    c.setMode(mode)
    c.setNormMode("RootSift" if norm == "rootsift" else "classic")
    if downsampling is not None:
        c.setDownsampling(downsampling)
    if octaves is not None:
        c.setOctaves(octaves)
    return c


def planes_report(ps, o):
    bad = 0
    for oc in range(o.num_octaves):
        for l in range(6):
            a, b = ps.plane(0, oc, l), o.gauss(oc, l)
            n = int((a != b).sum())
            if n:
                bad += 1
                yy, xx = np.argwhere(a != b)[0]
                print("   G o%d l%d: %d/%d differ, max|d|=%g first (y=%d,x=%d) gpu=%r cpu=%r" %
                      (oc, l, n, a.size, np.abs(a - b).max(), yy, xx, a[yy, xx], b[yy, xx]))
        for l in range(5):
            a, b = ps.plane(0, oc, l, dog=True), o.dog(oc, l)
            n = int((a != b).sum())
            if n:
                bad += 1
                yy, xx = np.argwhere(a != b)[0]
                print("   D o%d l%d: %d/%d differ, max|d|=%g first (y=%d,x=%d)" % (oc, l, n, a.size, np.abs(a - b).max(), yy, xx))
    print("   planes with differences: %d" % bad)
    return bad


def run_case(w, h, seed, mode, norm, downsampling=None, octaves=None, planes=True, ref=True):
    print("=== %dx%d seed %d mode=%s norm=%s ds=%s oct=%s" % (w, h, seed, mode, norm, downsampling, octaves))
    img = make_frame(w, h, seed)
    cfg = mk_cfg(mode, norm, downsampling, octaves)
    ps = api.PopSift(cfg, max_width=w, max_height=h, slots=1)
    ps.set_timing(True)
    job = ps.enqueue(w, h, img)
    feats = job.get()
    print("   gpu: %d features, %d descriptors; stages ms %s" % (feats.getFeatureCount(), feats.getDescriptorCount(),
                                                                {k: round(v, 3) for k, v in ps.stage_ms(0).items()}))
    kw = dict(mode=mode, norm=norm)
    if downsampling is not None:
        kw["downsampling"] = downsampling
    if octaves is not None:
        kw["octaves"] = octaves
    o = ol.Oracle(ol.make_config(**kw), w, h)
    t = time.time(); o.run(img); print("   oracle: %.2fs" % (time.time() - t))
    if planes:
        planes_report(ps, o)
    # extrema
    ge = ps.extrema(0)
    oe = o.extrema()
    gs = set((int(e["octave"]), float(e["x"]), float(e["y"]), int(e["lpos"])) for e in ge)
    os_ = set((int(e[4]), float(e[0]), float(e[1]), int(e[3])) for e in oe)
    print("   extrema gpu %d oracle %d ; exact common %d only-gpu %d only-oracle %d" % (len(ge), len(oe), len(gs & os_), len(gs - os_), len(os_ - gs)))
    for t_ in sorted(gs - os_)[:5]:
        print("      only gpu   ", t_)
    for t_ in sorted(os_ - gs)[:5]:
        print("      only oracle", t_)
    of, od = o.features()
    ka, da = feats.keypoints()
    kb, db = ol.flatten(of, od)
    print("   vs oracle :", compare.report(ka, da, kb, db))
    if ref and os.path.exists(REF):
        with tempfile.TemporaryDirectory() as td:
            pgm = os.path.join(td, "f.pgm"); out = os.path.join(td, "f.bin")
            write_pgm(pgm, img)
            cmd = [REF, "-i", pgm, "-o", out, "--mode", mode, "--norm", norm]
            if downsampling is not None:
                cmd += ["--downsampling", str(downsampling)]
            if octaves is not None:
                cmd += ["--octaves", str(octaves)]
            subprocess.run(cmd, check=True, capture_output=True)
            rf, rd = ol.read_ref_features(out)
            kr, dr = ol.flatten(rf, rd)
            print("   reference : %d features %d descriptors" % (len(rf), len(rd)))
            print("   vs ref    :", compare.report(ka, da, kr, dr))
    ps.uninit()


def main():
    run_case(256, 192, 3, "vlfeat", "classic")
    run_case(640, 480, 1, "popsift", "rootsift")
    run_case(640, 480, 1, "vlfeat", "classic")
    run_case(640, 480, 1, "popsift", "rootsift", downsampling=0)
    run_case(641, 479, 5, "vlfeat", "classic")
    run_case(1920, 1080, 100, "popsift", "rootsift", planes=False)
    run_case(1920, 1080, 100, "vlfeat", "classic", planes=False)
    run_case(3840, 2160, 7, "popsift", "rootsift", octaves=5, planes=False)
    # timing loop at 1080p and 4K
    for (w, h, seed, kw) in [(1920, 1080, 100, {}), (3840, 2160, 7, dict(octaves=5))]:
        img = make_frame(w, h, seed)
        cfg = mk_cfg(**kw)
        ps = api.PopSift(cfg, max_width=w, max_height=h, slots=2)
        ps.set_timing(True)
        for _ in range(3):
            ps.enqueue(w, h, img).get()
        t = time.time()
        n = 10
        jobs = [ps.enqueue(w, h, img) for _ in range(2)]
        for i in range(n):
            jobs[i % 2].get()
            if i + 2 < n:
                jobs[i % 2] = ps.enqueue(w, h, img)
        dt = time.time() - t
        print("timing %dx%d: %.2f ms/frame wall (2 slots), %.1f Mpix/s; stages %s" %
              (w, h, dt / n * 1e3, w * h * n / dt / 1e6, {k: round(v, 3) for k, v in ps.stage_ms(0).items()}))
        ps.uninit()


if __name__ == "__main__":
    main()
