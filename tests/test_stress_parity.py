"""The extraction path (pyramid -> extrema -> orientation -> descriptor -> normalisation) on adversarial content
(tests/stress_images.py) and with the Config knobs structure-from-motion callers set, against
  (1) the CPU oracle: planes bit-identical, extrema identical, same counts, F1 >= 0.99, descriptor L2 < 1e-3;
  (2) the reference's stored runs of the same bytes (tests/golden/live/stress_*.npz, knob_*.npz): identical keypoints,
      orientation counts and angles, sampled descriptors within 1e-3;
and the paths no make_frame image reaches: the candidate extrema kernel's stage-3 queue overflow, the fallback pyramid /
extrema kernels on stress frames, input from device memory with a pitch, and frames of several sizes through one
context."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import compare
import oracle_lib as ol
import stress_images as si
from popsift_b200 import api
from popsift_b200.synth import make_frame

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = os.path.join(HERE, "golden")
sys.path.insert(0, G)
import make_golden_live as mgl  # noqa: E402

F1_MIN, L2_MAX = 0.99, 1e-3
MAX_EXTREMA = 100000
MODES = (("popsift", "rootsift"), ("vlfeat", "classic"), ("opencv", "classic"))
PARITY_IMAGES = [n for n in si.NAMES if n != "checker_p3_4k"]
IMAGE_KW = {"dark": dict(threshold=0.001)}       # DoG values of a 0..3 image stay below the default threshold


def gpu_config(mode="popsift", norm="rootsift", **kw):
    c = api.Config()
    c.setMode(mode)
    c.setNormMode("RootSift" if norm == "rootsift" else "classic")
    setters = {"threshold": c.setThreshold, "edge_limit": c.setEdgeLimit, "initial_blur": c.setInitialBlur,
               "norm_multi": c.setNormalizationMultiplier, "sigma": c.setSigma, "levels": c.setLevels,
               "octaves": c.setOctaves}
    for k, v in kw.items():
        if k == "max_extrema":
            c._c.max_extrema = int(v)          # ps_config::max_extrema (popsift::Config has no setter for it)
        else:
            setters[k](v)
    return c


def oracle_config(mode="popsift", norm="rootsift", **kw):
    kw = dict(kw)
    if "initial_blur" in kw:
        kw["has_initial_blur"] = 0 if kw["initial_blur"] == 0.0 else 1
    return ol.make_config(mode=mode, norm=norm, **kw)


def run_gpu(img, cfg, slots=1):
    h, w = img.shape
    imode = api.PopSift.FloatImages if img.dtype == np.float32 else api.PopSift.ByteImages
    ps = api.PopSift(cfg, imode=imode, max_width=w, max_height=h, slots=slots)
    return ps, ps.enqueue(w, h, img).get()


def sorted_extrema(ge):
    return sorted((int(e["octave"]), float(e["x"]), float(e["y"]), int(e["lpos"])) for e in ge)


def sorted_oracle_extrema(oe):
    return sorted((int(e[4]), float(e[0]), float(e[1]), int(e[3])) for e in oe)


def check_descriptors(desc, norm, nm, label):
    """finite; unit norm (classic) or unit sum of squares (RootSift), after scaling by 2^-norm_multi"""
    d = desc.astype(np.float64) * 2.0 ** -nm
    assert np.isfinite(d).all(), (label, "non-finite descriptor")
    if len(d):
        ss = (d * d).sum(1)
        bad = np.abs(ss - 1.0).max() if norm == "rootsift" else np.abs(np.sqrt(ss) - 1.0).max()
        assert bad < 1e-3, (label, norm, float(bad))


def _num_ori_by_key(feat):
    d = {}
    for f in feat:
        d.setdefault((int(f["octave"]), float(f["x"]), float(f["y"])), []).append(int(f["num_ori"]))
    return {k: sorted(v) for k, v in d.items()}


# Keypoints (input-image x, y) whose number of orientations differs between this library and the oracle because the
# ratio of a secondary histogram peak to the highest one is 0.8 to within the difference between the CUDA math library
# (expf, atan2f, hypotf in the reference and here) and libm (the oracle).  The reference decides: its stored run of each
# listed (image, initial_blur, mode) -- named below -- has this library's orientations at every one of them, bit for bit
# (test_stress_vs_reference_runs).  x, y rounded to 1e-3:
#   block_noise_4, PopSift (stress_block_noise_4_prs) and VLFeat (stress_block_noise_4_vlc) mode: (41.499, 473.501) 2
#       orientations, the oracle 3; (185.392, 245.390) and (621.391, 53.391) 1, the oracle 2
#   block_noise_4, OpenCV mode (stress_block_noise_4_ocv): (185.654, 245.652) 2, the oracle 1
#   block_noise_4, initial_blur 1.0, PopSift mode (knob_iblur_1_block_noise_4): (13.619, 185.381) 2, the oracle 4;
#       (225.501, 325.508) 3 / 4; (237.385, 385.614) 4 / 3; (377.241, 21.549) 2 / 1; (377.497, 121.499) 4 / 3.
#       VLFeat mode has the same five: the orientation stage does not depend on the mode, and these extrema are the
#       same (octave, x, y, sigma) in both modes, so the PopSift-mode run decides for them too.
_BN4_TIES = {(41.499, 473.501), (185.392, 245.390), (621.391, 53.391)}
_BN4_IBLUR1_TIES = {(13.619, 185.381), (225.501, 325.508), (237.385, 385.614), (377.241, 21.549), (377.497, 121.499)}
ORI_COUNT_TIES = {
    ("block_noise_4", 0.5, "popsift"): _BN4_TIES,
    ("block_noise_4", 0.5, "vlfeat"): _BN4_TIES,
    ("block_noise_4", 0.5, "opencv"): {(185.654, 245.652)},
    ("block_noise_4", 1.0, "popsift"): _BN4_IBLUR1_TIES,
    ("block_noise_4", 1.0, "vlfeat"): _BN4_IBLUR1_TIES,
}


def compare_with_oracle(img, mode, norm, label, **kw):
    """planes bit-identical, sorted (octave, x, y, lpos) identical, feature counts identical, orientation counts
    identical (but for ORI_COUNT_TIES), every descriptor within 1e-3 of the oracle's descriptor stage at the same
    keypoint and orientation, and the whole pipeline against the oracle's: F1 >= 0.99, descriptor L2 < 1e-3 where the
    orientations agree; returns (#extrema, None)"""
    h, w = img.shape
    ps, feats = run_gpu(img, gpu_config(mode, norm, **kw))
    o = ol.Oracle(oracle_config(mode, norm, **kw), w, h)
    o.run(img)
    try:
        L = max(kw.get("levels", 3), 2)
        assert len(ps.slot_geometry(0)) == o.num_octaves
        bad = []
        for oc in range(o.num_octaves):
            for lv in range(L + 3):
                if not np.array_equal(ps.plane(0, oc, lv), o.gauss(oc, lv)):
                    bad.append(("gauss", oc, lv))
            for lv in range(L + 2):
                if not np.array_equal(ps.plane(0, oc, lv, dog=True), o.dog(oc, lv)):
                    bad.append(("dog", oc, lv))
        assert not bad, (label, bad)
        oe = o.extrema()
        if len(oe):
            per_octave = np.bincount(oe[:, 4].astype(np.int64))
            # past max_extrema, which extrema are kept depends on arrival order in both libraries
            assert per_octave.max() < kw.get("max_extrema", MAX_EXTREMA), (label, per_octave)
        ge = ps.extrema(0)
        a, b = sorted_extrema(ge), sorted_oracle_extrema(oe)
        assert a == b, (label, len(a), len(b), len(set(a) ^ set(b)))
        of, od = o.features()
        assert feats.getFeatureCount() == len(of), (label, feats.getFeatureCount(), len(of))
        # orientation counts: identical except at the listed peak-ratio ties (see ORI_COUNT_TIES)
        mine, theirs = _num_ori_by_key(feats.feat), _num_ori_by_key(of)
        differ = {k for k in set(mine) | set(theirs) if mine.get(k) != theirs.get(k)}
        allowed = ORI_COUNT_TIES.get((label.split("/")[-1], kw.get("initial_blur", 0.5), mode), set())
        if differ:
            print("%s %s: orientation counts differ at %s" % (label, mode, sorted((round(k[1], 3), round(k[2], 3), mine.get(k), theirs.get(k)) for k in differ)))
        assert {(round(k[1], 3), round(k[2], 3)) for k in differ} <= allowed, (label, mode, sorted(differ))
        extra = sum(sum(theirs.get(k, [])) - sum(mine.get(k, [])) for k in differ)
        assert len(od) - feats.getDescriptorCount() == extra, (label, feats.getDescriptorCount(), len(od))
        nm = kw.get("norm_multi", 0)
        s = 2.0 ** -nm
        check_descriptors(feats.desc, norm, nm, label)
        # every descriptor against the oracle's descriptor stage at this library's keypoint and orientation
        n_ori = ge["num_ori"].astype(np.int64)
        idx = np.repeat(np.arange(len(ge)), n_ori)
        k = np.arange(len(idx)) - np.repeat(np.cumsum(n_ori) - n_ori, n_ori)
        assert np.array_equal(feats.feat["num_ori"], ge["num_ori"]) and len(idx) == feats.getDescriptorCount()
        didx = ge["idx_ori"][idx].astype(np.int64) + k
        assert np.array_equal(feats.desc_idx[idx, k], didx), label          # extremum i is feature i
        want = o.describe(ge["x"][idx], ge["y"][idx], ge["sigma"][idx], ge["ori"][idx, k], ge["octave"][idx], ge["lpos"][idx])
        l2 = np.linalg.norm((feats.desc[didx].astype(np.float64) - want) * s, axis=1) if len(idx) else np.zeros(1)
        if len(od):
            # the whole pipeline against the oracle's: keypoint / orientation F1, and the descriptor bar wherever the two
            # orientation stages agree (libm and the CUDA math library may move a peak of a near-flat histogram)
            ka, da = feats.keypoints()
            kb, db = ol.flatten(of, od)
            pairs, _, _, f1 = compare.match_keypoints(ka, kb)
            ia = np.array([p[0] for p in pairs]); ib = np.array([p[1] for p in pairs])
            dth = np.abs(np.angle(np.exp(1j * (ka[ia, 3] - kb[ib, 3]))))
            pl2 = np.linalg.norm((da[ia].astype(np.float64) - db[ib]) * s, axis=1)
            same = dth < 1e-5
            print("%-34s %-8s %6d ext %7d desc  L2 max %.3g p99 %.3g median %.3g  | pipeline F1 %.4f, L2 max %.3g "
                  "(%.3g where the angles agree, %d do not)" % (label, mode, len(a), len(idx), l2.max(), np.percentile(l2, 99),
                                                             np.median(l2), f1, pl2.max(), pl2[same].max(initial=0.0), (~same).sum()))
            assert f1 >= F1_MIN and pl2[same].max(initial=0.0) < L2_MAX, (label, mode, f1, pl2[same].max(initial=0.0))
            # the pairs left out of that bar are few (measured: at most 1.4 % on binary block noise, 4 of 193 on
            # border_impulses), and their descriptors are still held to 1e-3 at this library's angle above
            assert (~same).sum() <= 0.02 * len(pairs) + 4, (label, mode, int((~same).sum()), len(pairs))
            assert l2.max() < L2_MAX, (label, mode, float(l2.max()))
        else:
            print("%-34s %-8s %6d ext %7d desc" % (label, mode, len(a), 0))
        return len(a), None
    finally:
        ps.uninit()
        o.close()


# RootSift descriptors of the 0..3 "dark" image exceed the 1e-3 bar: the known limit of the descriptor's fixed-point
# bins documented in k_desc.cu and INTEGRATION.md (5e-3 from the oracle, 4.4e-3 from the reference; the classic modes
# pass, test_dark_classic_vs_oracle).  Strict: the test fails as soon as the limit is lifted and the marker is stale.
DARK_ROOTSIFT = pytest.mark.xfail(strict=True, reason="fixed-point resolution of RootSift descriptors on 0..3 grey-level content")


@pytest.mark.parametrize("name", [pytest.param(n, marks=DARK_ROOTSIFT) if n == "dark" else n for n in PARITY_IMAGES])
def test_stress_images_vs_oracle(name):
    """every stress image under popsift / RootSift, vlfeat / classic and opencv / classic"""
    img = si.image(name)
    n = {}
    for mode, norm in MODES[:1] if name == "dark" else MODES:     # dark: the classic modes in test_dark_classic_vs_oracle
        n[mode], _ = compare_with_oracle(img, mode, norm, name, **IMAGE_KW.get(name, {}))
    if name.startswith("const_"):
        assert n == {"popsift": 0, "vlfeat": 0, "opencv": 0}
    if name in ("checker_p3", "checker_p8", "checker_rot30_p6", "block_noise_4", "binary_noise", "saturated",
                "border_impulses", "binary_noise_f32", "checker_p8_f32"):
        assert n["popsift"] > 50, n          # the image is not trivially empty


def test_dark_classic_vs_oracle():
    img = si.image("dark")
    for mode, norm in MODES[1:]:
        assert compare_with_oracle(img, mode, norm, "dark", **IMAGE_KW["dark"])[0] > 50


def test_border_structure_reaches_the_clamps():
    """border_impulses places keypoints whose orientation window and descriptor support reach past the image edge:
    some keypoint lies within 3 sigma of the border of its octave, in every mode (opencv: outside its 5-pixel margin)"""
    img = si.image("border_impulses")
    for mode, norm in MODES:
        ps, feats = run_gpu(img, gpu_config(mode, norm))
        dims = ps.slot_geometry(0)
        e = ps.extrema(0)
        ps.uninit()
        W = np.array([dims[o][0] for o in e["octave"]], np.float64)
        H = np.array([dims[o][1] for o in e["octave"]], np.float64)
        x, y, s = e["x"].astype(np.float64), e["y"].astype(np.float64), e["sigma"].astype(np.float64)
        near = np.minimum(np.minimum(x, W - 1 - x), np.minimum(y, H - 1 - y)) < 3 * s
        assert near.sum() >= 5, (mode, int(near.sum()))


KNOBS = [
    ("threshold_0.005", dict(threshold=0.005), "rootsift"),
    ("threshold_0.1", dict(threshold=0.1), "rootsift"),
    ("edge_2", dict(edge_limit=2.0), "rootsift"),
    ("edge_50", dict(edge_limit=50.0), "rootsift"),
    ("iblur_0", dict(initial_blur=0.0), "rootsift"),
    ("iblur_1", dict(initial_blur=1.0), "rootsift"),
    ("nm3_rs", dict(norm_multi=3), "rootsift"),
    ("nm9_rs", dict(norm_multi=9), "rootsift"),
    ("nm3_classic", dict(norm_multi=3), "classic"),
    ("nm9_classic", dict(norm_multi=9), "classic"),
    # the largest descriptor support the configuration allows (sigma 2.0, levels 2: sigma up to 2 * 2^(4/2) per octave)
    ("sigma2_l2", dict(sigma=2.0, levels=2), "rootsift"),
]


@pytest.mark.parametrize("label,kw,norm", KNOBS, ids=[k[0] for k in KNOBS])
def test_config_knobs_vs_oracle(label, kw, norm):
    """threshold, edge_limit, initial_blur and norm_multi on a make_frame image and on full-contrast content; descriptors
    compared after scaling by 2^-norm_multi"""
    images = [("make_frame", make_frame(640, 480, 1)), ("block_noise_4", si.image("block_noise_4"))]
    if label == "sigma2_l2":
        images += [("checker_rot30_p6", si.image("checker_rot30_p6")), ("step_edges", si.image("step_edges"))]
    else:
        images.append(("saturated", si.image("saturated")))
    counts = []
    for iname, img in images:
        modes = [("popsift", norm)] if label.startswith("nm") or label == "sigma2_l2" else [("popsift", norm), ("vlfeat", "classic")]
        for mode, nrm in modes:
            n, _ = compare_with_oracle(img, mode, nrm, "%s/%s" % (label, iname), **kw)
            counts.append(n)
    assert max(counts) > 0
    if label.startswith("nm"):
        # the multiplier really is applied: descriptor components reach 2^nm * 0.2 and more
        ps, feats = run_gpu(images[1][1], gpu_config("popsift", norm, **kw))
        assert feats.desc.max() > 0.1 * 2 ** kw["norm_multi"]
        ps.uninit()


def _key_rows(feat):
    """(octave, x bits, y bits, sigma bits) per keypoint"""
    return np.stack([feat["octave"].astype(np.int64), feat["x"].view(np.int32).astype(np.int64),
                     feat["y"].view(np.int32).astype(np.int64), feat["sigma"].view(np.int32).astype(np.int64)], axis=1)


def _ordered(feat):
    """keypoint order by key, ties broken by the orientation angles"""
    keys = _key_rows(feat)
    ori = np.where(np.arange(4)[None, :] < feat["num_ori"][:, None], feat["ori"], np.float32(0)).view(np.int32)
    cols = np.concatenate([keys, ori.astype(np.int64)], axis=1)
    return np.lexsort(cols.T[::-1]), keys, ori


def _args_to_kw(args):
    opts = dict(zip(args[0::2], args[1::2]))
    kw = {}
    conv = {"--threshold": ("threshold", float), "--edge-limit": ("edge_limit", float), "--initial-blur": ("initial_blur", float),
            "--norm-multi": ("norm_multi", int), "--sigma": ("sigma", float), "--levels": ("levels", int)}
    for k, (name, f) in conv.items():
        if k in opts:
            kw[name] = f(opts[k])
    return opts["--mode"], opts["--norm"], kw


@pytest.mark.parametrize("name", [pytest.param(n, marks=DARK_ROOTSIFT) if n == "stress_dark_prs" else n for n in sorted(mgl.STRESS_RUNS)])
def test_stress_vs_reference_runs(name):
    """The reference's own run of the same bytes (tests/golden/live/<name>.npz, made on an H100 by
    tests/golden/make_golden_live.py --only 'stress_*' / 'knob_*'), to the bench32 standard: identical feature and
    descriptor counts, keypoints (octave, x, y, sigma) bit-identical, the same number of orientations per keypoint,
    orientation angles bit-identical, octave-0 planes bit-identical, sampled descriptors within 1e-3."""
    img_name, args = mgl.STRESS_RUNS[name]
    mode, norm, kw = _args_to_kw(args)
    img = si.image(img_name)
    rf, rd, planes = ol.ref_golden(name)
    ps, feats = run_gpu(img, gpu_config(mode, norm, **kw))
    try:
        L = max(kw.get("levels", 3), 2)
        for lv in range(L + 3):
            assert planes["0_%d" % lv] == ol.plane_id(ps.plane(0, 0, lv)), (name, "octave 0 plane", lv)
        assert (feats.getFeatureCount(), feats.getDescriptorCount()) == (len(rf), len(rd)), \
            (name, feats.getFeatureCount(), feats.getDescriptorCount(), len(rf), len(rd))
        go, gk, gori = _ordered(feats.feat)
        ro, rk, rori = _ordered(rf)
        assert np.array_equal(gk[go], rk[ro]), (name, int((gk[go] != rk[ro]).any(1).sum()), "keypoints differ")
        assert np.array_equal(feats.feat["num_ori"][go], rf["num_ori"][ro]), name
        assert np.array_equal(gori[go], rori[ro]), (name, int((gori[go] != rori[ro]).any(1).sum()), "orientations differ")
        s = 2.0 ** -kw.get("norm_multi", 0)
        l2 = []
        for j, i in zip(go.tolist(), ro.tolist()):
            for k in range(int(rf["num_ori"][i])):
                ref = rd[rf["desc_idx"][i, k]]
                if not np.isnan(ref).all():
                    mine = feats.desc[feats.desc_idx[j, k]]
                    l2.append(float(np.linalg.norm((mine.astype(np.float64) - ref.astype(np.float64)) * s)))
        if len(rd):
            assert l2, name
            l2 = np.array(l2)
            print("%-30s %6d feat %7d desc  vs reference: L2 max %.3g p99 %.3g median %.3g (%d sampled)"
                  % (name, len(rf), len(rd), l2.max(), np.percentile(l2, 99), np.median(l2), len(l2)))
            assert l2.max() < L2_MAX, (name, float(l2.max()))
        check_descriptors(feats.desc, norm, kw.get("norm_multi", 0), name)
    finally:
        ps.uninit()


def _stage2_survivors(planes, thr):
    """Voxels of levels 1 .. L, rows / columns 1 .. n-2, with |DoG| >= thr that are strictly greater or strictly
    smaller than all 26 neighbours: what stage 2 of cand_extrema_kernel queues for refinement.  planes: one
    (L + 2, H, W) array per octave."""
    total = 0
    for D in planes:
        P, Hh, Ww = D.shape
        if Hh < 3 or Ww < 3:
            continue
        for lv in range(1, P - 1):
            c = D[lv, 1:Hh - 1, 1:Ww - 1]
            mx = np.full(c.shape, -np.inf, np.float32)
            mn = np.full(c.shape, np.inf, np.float32)
            for dz in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        if dz or dy or dx:
                            n = D[lv + dz, 1 + dy:Hh - 1 + dy, 1 + dx:Ww - 1 + dx]
                            np.maximum(mx, n, out=mx)
                            np.minimum(mn, n, out=mn)
            total += int(((np.abs(c) >= thr) & ((c > mx) | (c < mn))).sum())
    return total


def test_stage3_queue_overflow_vs_oracle():
    """cand_extrema_kernel queues stage-2 survivors in a 1024-entry shared-memory queue per block and refines at once
    whatever does not fit.  A 3840x2160 checkerboard of period 3 has one blob per square at octave 0: counted from this
    library's own DoG planes, its 3x3x3 extrema exceed 1024 x the kernel's grid (3 blocks per SM), so at least one block
    takes the overflow path.  max_extrema is raised in library and oracle so that nothing is dropped; the extrema must be
    those of the oracle, and every one of them must become a feature (results stay on the device: Config::MatchingMode)."""
    import torch
    img = si.image("checker_p3_4k")
    h, w = img.shape
    kw = dict(octaves=3, max_extrema=1000000)
    ps = api.PopSift(gpu_config("popsift", "rootsift", **kw), mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    feats = ps.enqueue(w, h, img).getDev()
    o = ol.Oracle(oracle_config("popsift", "rootsift", **kw), w, h)
    o.run(img, 3)                      # pyramid + extrema
    try:
        L = 3
        dogs = [np.stack([ps.plane(0, oc, lv, dog=True) for lv in range(L + 2)]) for oc in range(len(ps.slot_geometry(0)))]
        for oc, D in enumerate(dogs):
            for lv in range(L + 2):
                assert np.array_equal(D[lv], o.dog(oc, lv)), (oc, lv)
        thr = np.float32(1.6) * np.float32(api.Config().getPeakThreshold())
        survivors = _stage2_survivors(dogs, thr)
        del dogs
        grid = 3 * torch.cuda.get_device_properties(0).multi_processor_count
        print("stage-3 overflow: %d stage-2 survivors, queue capacity 1024 x %d blocks = %d" % (survivors, grid, 1024 * grid))
        assert survivors > 1024 * grid
        ge, oe = ps.extrema(0), o.extrema()
        assert np.bincount(oe[:, 4].astype(np.int64)).max() < kw["max_extrema"]
        a = np.stack([ge["octave"].astype(np.float64), ge["x"], ge["y"], ge["lpos"].astype(np.float64)], 1)
        b = oe[:, [4, 0, 1, 3]].astype(np.float64)
        a, b = a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])]
        assert a.shape == b.shape and np.array_equal(a, b), (a.shape, b.shape)
        assert feats.getFeatureCount() == len(oe) == survivors
        assert feats.getDescriptorCount() >= feats.getFeatureCount()
        del feats
    finally:
        ps.uninit()
        o.close()


_SUBPROCESS_RUN = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import stress_images as si
from popsift_b200 import api
out = {}
for name, mode in (("block_noise_4", "popsift"), ("border_impulses", "opencv"), ("checker_rot30_p6", "vlfeat")):
    img = si.image(name)
    h, w = img.shape
    c = api.Config(); c.setMode(mode); c.setNormMode("classic")
    ps = api.PopSift(c, max_width=w, max_height=h, slots=1)
    f = ps.enqueue(w, h, img).get()
    e = ps.extrema(0)
    ex = np.stack([e["octave"].astype(np.float64), e["x"], e["y"], e["lpos"].astype(np.float64), e["sigma"]], 1)
    out[name + "_extrema"] = ex[np.lexsort(ex.T[::-1])]
    rows = []
    for i, ft in enumerate(f.feat):
        for k in range(int(ft["num_ori"])):
            rows.append(np.concatenate([[ft["octave"], ft["x"], ft["y"], ft["sigma"], ft["ori"][k]], f.desc[f.desc_idx[i, k]]]))
    rows = np.array(rows, np.float64).reshape(-1, 133)
    out[name + "_features"] = rows[np.lexsort(rows.T[::-1])]
    ps.uninit()
np.savez(sys.argv[3], **out)
"""


def _run_in_subprocess(env_extra, path):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, "-c", _SUBPROCESS_RUN, HERE, ROOT, str(path)], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return dict(np.load(str(path)))


def test_fallback_paths_give_the_same_extrema_on_stress_frames(tmp_path):
    """The dense DoG scan, the tile pyramid kernels and the uniform single-stream pyramid give the same sorted extrema
    and the same (keypoint, orientation, descriptor) rows as the default path, on full-contrast and border content."""
    base = _run_in_subprocess({}, tmp_path / "base.npz")
    assert all(len(v) > 10 for v in base.values())
    for env in ({"POPSIFT_B200_DENSE_SCAN": "1"}, {"POPSIFT_B200_TILE_KERNELS": "1"},
                {"POPSIFT_B200_UNIFORM": "1", "POPSIFT_B200_FORK": "0"}):
        got = _run_in_subprocess(env, tmp_path / "alt.npz")
        for k, v in base.items():
            assert got[k].shape == v.shape and np.array_equal(got[k], v), (env, k, got[k].shape, v.shape)


def _canonical(feats):
    rows = []
    for i, ft in enumerate(feats.feat):
        for k in range(int(ft["num_ori"])):
            rows.append(np.concatenate([[ft["octave"], ft["x"], ft["y"], ft["sigma"], ft["ori"][k]], feats.desc[feats.desc_idx[i, k]]]))
    rows = np.array(rows, np.float64).reshape(-1, 133)
    return rows[np.lexsort(rows.T[::-1])]


def _result(ps, slot, feats):
    return (feats.getFeatureCount(), feats.getDescriptorCount(), _canonical(feats),
            hashlib.sha256(ps.plane(slot, 1, 2).tobytes()).hexdigest())


def _same(a, b):
    return a[0] == b[0] and a[1] == b[1] and a[3] == b[3] and a[2].shape == b[2].shape and np.array_equal(a[2], b[2])


def test_submit_dev_u8_with_pitch_equals_host_submit():
    """ps_submit_dev_u8 (the input path bench.py measures): a 641x479 frame in device memory at pitch == w and at a
    padded pitch of 704 bytes (padding filled with 255) gives the planes, extrema and features of ps_submit_u8"""
    L = api.load_library()
    img = si.image("block_noise_4", 641, 479)
    h, w = img.shape
    cfg = gpu_config()
    ps_h, fh = run_gpu(img, cfg)
    want = _result(ps_h, 0, fh)
    want_planes = [(oc, lv, ps_h.plane(0, oc, lv)) for oc in range(len(ps_h.slot_geometry(0))) for lv in range(6)]
    want_ext = sorted_extrema(ps_h.extrema(0))
    ps_h.uninit()
    assert want[0] > 100
    for pitch in (w, 704):
        host = np.full((h, pitch), 255, np.uint8)
        host[:, :w] = img
        d = L.ps_dev_alloc(host.nbytes)
        assert d
        try:
            assert L.ps_host_to_dev(d, host.ctypes.data, host.nbytes) == 0
            ps = api.PopSift(cfg, max_width=w, max_height=h, slots=1)
            ps._check(L.ps_submit_dev_u8(ps._ctx, 0, d, pitch, w, h))
            fd = ps._collect(0)
            got = _result(ps, 0, fd)
            for oc, lv, p in want_planes:
                assert np.array_equal(ps.plane(0, oc, lv), p), (pitch, oc, lv)
            assert sorted_extrema(ps.extrema(0)) == want_ext, pitch
            assert _same(got, want), (pitch, got[:2], want[:2])
            ps.uninit()
        finally:
            L.ps_dev_free(d)


def test_mixed_geometries_through_one_context():
    """One 1920x1080 context with two slots takes 640x480, 97x61, 641x479 and 1920x1080 frames in an interleaved order in
    which every size is captured as a CUDA graph and later replayed after frames of other sizes.  Every result (features,
    descriptors, the hash of octave 1 / level 2) equals a dedicated context's result for that frame."""
    frames = {"a": si.image("block_noise_4", 640, 480), "b": si.image("checker_rot30_p6", 97, 61),
              "c": si.image("saturated", 641, 479), "d": si.image("border_impulses", 1920, 1080)}
    cfg = gpu_config()
    want = {}
    for key, img in frames.items():
        ps, f = run_gpu(img, cfg)
        want[key] = _result(ps, 0, f)
        ps.uninit()
    # per slot: three of a kind (direct, capture, replay), then other sizes and back to a captured one
    slot0 = "aaabacadddabbbdcc"
    slot1 = "bbbabdbcccaaadcdd"
    order = [s for pair in zip(slot0, slot1) for s in pair]
    for key in "abcd":
        assert order.count(key) >= 3
    ps = api.PopSift(cfg, max_width=1920, max_height=1080, slots=2)
    prev = None
    for i, key in enumerate(order):
        img = frames[key]
        job = ps.enqueue(img.shape[1], img.shape[0], img)
        if prev is not None:
            pj, pkey, pslot, pi = prev
            got = _result(ps, pslot, pj.get())
            assert _same(got, want[pkey]), (pi, pkey, got[:2], want[pkey][:2], got[3] == want[pkey][3])
        prev = (job, key, i % 2, i)
    pj, pkey, pslot, pi = prev
    assert _same(_result(ps, pslot, pj.get()), want[pkey]), (pi, pkey)
    ps.uninit()
