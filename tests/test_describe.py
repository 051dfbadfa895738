"""Describe path on the GPU (ps_describe_u8 / ps_describe_f32, PopSift.describe): orientations and descriptors at
caller-supplied keypoints.

  * round trips: a frame's own keypoints, described with their angles or with computed orientations, give back the
    extraction's orientations and descriptors bit for bit (in input order, also when permuted);
  * the octave / level rule (tests/describe_rule.py) for keypoints without hints;
  * foreign keypoints (dense grids, random positions and scales beyond the pyramid) against the oracle's orientation
    and descriptor stages (orc_orient of tests/orient_oracle.c, orc_describe);
  * rejected keypoints, argument errors, capacity growth, one slot shared with detection and its CUDA graph, the other
    descriptor modes, float images and MatchingMode."""
import os
import subprocess
import sys

import numpy as np
import pytest

import describe_rule as dr
import oracle_lib as ol
import orient_oracle as oo
import stress_images as si
from popsift_b200 import api
from popsift_b200.synth import make_frame

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MODES = (("popsift", "rootsift"), ("vlfeat", "classic"), ("opencv", "classic"))
L = 3
L2_MAX = 1e-3


def gpu_config(mode="popsift", norm="rootsift"):
    c = api.Config()
    c.setMode(mode)
    c.setNormMode("RootSift" if norm == "rootsift" else "classic")
    return c


def extract(ps, img):
    """features of one frame and the slot's extremum records (index = Feature index); ps has one slot"""
    h, w = img.shape
    f = ps.enqueue(w, h, img).get()
    return f, ps.extrema(0)


def describe(ps, img, kp, orient=False):
    h, w = img.shape
    return ps.describe(w, h, img, kp, orientations=orient).get()


def per_desc_keypoints(f, ext):
    """one keypoint per descriptor of an extraction: the Feature's x, y, sigma and angle, octave and lpos as hints"""
    n = f.feat["num_ori"].astype(np.int64)
    idx = np.repeat(np.arange(len(n)), n)
    k = np.arange(len(idx)) - np.repeat(np.cumsum(n) - n, n)
    kp = np.zeros(len(idx), api.KEYPOINT_DTYPE)
    for a in ("x", "y", "sigma"):
        kp[a] = f.feat[a][idx]
    kp["ori"] = f.feat["ori"][idx, k]
    kp["octave"] = ext["octave"][idx]
    kp["level"] = ext["lpos"][idx]
    return kp, f.desc_idx[idx, k]


def per_feature_keypoints(f, ext):
    kp = np.zeros(len(f.feat), api.KEYPOINT_DTYPE)
    for a in ("x", "y", "sigma"):
        kp[a] = f.feat[a]
    kp["octave"] = ext["octave"]
    kp["level"] = ext["lpos"]
    return kp


def feature_fields(f):
    """the Feature records as plain arrays (without the descriptor pointers, which differ from run to run)"""
    return {a: np.ascontiguousarray(f.feat[a]) for a in ("octave", "x", "y", "sigma", "num_ori", "ori")}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_in_order(f, kp, ext_octave=None):
    """one Feature per keypoint with the keypoint's own bits, descriptors contiguous in input order"""
    assert f.getFeatureCount() == len(kp)
    for a in ("x", "y", "sigma"):
        assert np.array_equal(bits(f.feat[a]), bits(kp[a])), a
    n = f.feat["num_ori"].astype(np.int64)
    first = np.cumsum(n) - n
    has = n > 0
    assert np.array_equal(f.desc_idx[has, 0], first[has])
    assert f.getDescriptorCount() == n.sum()
    if ext_octave is not None:
        assert np.array_equal(f.feat["octave"], ext_octave)


# ---------------------------------------------------------------------------------------------- round trips

ROUND_TRIP = [(m, n, w, h) for m, n in MODES for w, h in ((640, 480), (1920, 1080))] + [("popsift", "rootsift", 3840, 2160)]


@pytest.mark.parametrize("mode,norm,w,h", ROUND_TRIP)
def test_round_trip_given_and_orient(mode, norm, w, h):
    """A frame's own keypoints with octave and lpos hints: with the given angles (one keypoint per descriptor) the
    descriptors are the extraction's bit for bit; with computed orientations (one keypoint per Feature) num_ori, the
    angles and the descriptors are, also for the keypoints in a random order.  Without hints, where the rule gives back
    the detected (octave, lpos), debug_octave and the descriptors equal the hinted run."""
    img = make_frame(w, h, 11)
    ps = api.PopSift(gpu_config(mode, norm), max_width=w, max_height=h, slots=1)
    try:
        f, ext = extract(ps, img)
        assert f.getDescriptorCount() > 200
        # GIVEN
        kp, didx = per_desc_keypoints(f, ext)
        g = describe(ps, img, kp)
        check_in_order(g, kp)
        assert (g.feat["num_ori"] == 1).all()
        assert np.array_equal(bits(g.feat["ori"][:, 0]), bits(kp["ori"]))
        assert np.array_equal(g.feat["octave"], kp["octave"])
        assert np.array_equal(bits(g.desc), bits(f.desc[didx]))
        # ORIENT
        kf = per_feature_keypoints(f, ext)
        r = describe(ps, img, kf, orient=True)
        check_in_order(r, kf, ext["octave"])
        assert np.array_equal(r.feat["num_ori"], f.feat["num_ori"])
        assert np.array_equal(bits(r.feat["ori"]), bits(f.feat["ori"]))
        assert np.array_equal(bits(r.desc), bits(f.desc))
        perm = np.random.default_rng(5).permutation(len(kf))
        p = describe(ps, img, kf[perm], orient=True)
        check_in_order(p, kf[perm])
        assert np.array_equal(p.feat["num_ori"], f.feat["num_ori"][perm])
        assert np.array_equal(bits(p.feat["ori"]), bits(f.feat["ori"][perm]))
        n = f.feat["num_ori"][perm].astype(np.int64)
        i = np.repeat(np.arange(len(n)), n)
        k = np.arange(len(i)) - np.repeat(np.cumsum(n) - n, n)
        assert np.array_equal(bits(p.desc[p.desc_idx[i, k]]), bits(f.desc[f.desc_idx[perm[i], k]]))
        # derived octave and level
        kd = kp.copy()
        kd["octave"] = kd["level"] = -1
        d = describe(ps, img, kd)
        n_oct = len(ps.slot_geometry(0))
        o, lvl, S = dr.octave_level(kd["sigma"], ps._config.sigma, L, 1, n_oct)
        inside = (kp["level"] >= 1) & (kp["level"] <= L)
        clean = inside & ~dr.near_rounding_edge(S, kp["octave"], L)
        assert clean.sum() > 0.9 * len(kp)
        assert np.array_equal(o[clean], kp["octave"][clean]) and np.array_equal(lvl[clean], kp["level"][clean])
        assert np.array_equal(d.feat["octave"][clean], kp["octave"][clean])
        assert np.array_equal(bits(d.desc[clean]), bits(g.desc[clean]))
        other = (~clean).sum()
        print("%s %dx%d: %d descriptors, %d keypoints with lpos outside 1..L or S near a rounding edge (not compared)"
              % (mode, w, h, len(kp), other))
    finally:
        ps.uninit()


# ------------------------------------------------------------------------------------------- foreign keypoints

def grid_keypoints(w, h, step=8, sigmas=(1.6, 3.2, 6.4), offset=0.0):
    ys, xs = np.mgrid[0:h:step, 0:w:step] + np.float32(offset)
    kp = np.zeros(xs.size * len(sigmas), api.KEYPOINT_DTYPE)
    kp["x"] = np.tile(xs.ravel(), len(sigmas))
    kp["y"] = np.tile(ys.ravel(), len(sigmas))
    kp["sigma"] = np.repeat(np.float32(sigmas), xs.size)
    kp["octave"] = kp["level"] = -1
    return kp


def random_keypoints(w, h, n, seed):
    """positions over the whole frame with a fifth in the outer 2 px, log-uniform sigma from 0.2 to 400 (below octave 0
    and above the top octave), angles in [-pi, pi)"""
    rng = np.random.default_rng(seed)
    kp = np.zeros(n, api.KEYPOINT_DTYPE)
    x = rng.uniform(0, w - 1, n)
    y = rng.uniform(0, h - 1, n)
    edge = rng.random(n) < 0.2
    side = rng.integers(0, 4, n)
    t = rng.uniform(0, 2, n)
    x = np.where(edge & (side == 0), t, np.where(edge & (side == 1), w - 1 - t, x))
    y = np.where(edge & (side == 2), t, np.where(edge & (side == 3), h - 1 - t, y))
    kp["x"], kp["y"] = x, y
    kp["sigma"] = np.exp(rng.uniform(np.log(0.2), np.log(400.0), n))
    kp["ori"] = rng.uniform(-np.pi, np.pi, n)
    kp["octave"] = kp["level"] = -1
    return kp


# Keypoints (input-image x, y rounded to 1e-3) whose number of orientations differs between this library and the
# oracle's orientation stage: a secondary histogram peak is 0.8 of the highest to within the difference between the CUDA
# math library (expf, atan2f, hypotf) and libm, as for ORI_COUNT_TIES in test_stress_parity.py.
# Key: (image, mode, keypoint set).
DESCRIBE_ORI_TIES = {
}

FOREIGN_IMAGES = ("make_frame", "block_noise_4", "checker_rot30_p6")


def foreign_image(name):
    return make_frame(640, 480, 13) if name == "make_frame" else si.image(name)


def _l2_vs(got, want):
    got, want = got.astype(np.float64), want.astype(np.float64)
    assert np.array_equal(np.isnan(got).any(1), np.isnan(want).any(1))
    return np.linalg.norm(np.nan_to_num(got) - np.nan_to_num(want), axis=1)


# Low-contrast supports: the descriptor's 32-bit fixed-point bins take their scale from full-contrast gradients, so where
# every gradient of the support is a few grey levels the rounding shows, most through RootSift's square root (the known
# limit documented in k_desc.cu and INTEGRATION.md).  Random keypoints reach such supports far more often than detected
# ones: the top octave of checker_rot30_p6 (a period-6 checkerboard averaged to within 1.05 grey levels) and small
# supports on make_frame's smooth texture.  Measured on an H100: up to 9.2e-3 L2 (RootSift) and 1.9e-3 (classic) where
# the largest gradient in the support is below LOW_CONTRAST grey levels; those are held to LOW_CONTRAST_L2_MAX, all
# others to L2_MAX.
# Sub-pyramid scales: an octave-local sigma below sigma0 (a detected keypoint has at least sigma0 * 2^(0.5 / L)) gives a
# support of a few pixels and a dozen samples, where one sample entering or leaving the support between the two
# implementations (the support's edge, the polynomial atan2 and approximate exp of k_desc.cu) moves the descriptor a lot:
# up to 0.15 L2 measured on binary block noise, 1.1e-3 on make_frame.  Those are held to SUB_PYRAMID_P99 in the 99th
# percentile and printed.
LOW_CONTRAST = 4.0
LOW_CONTRAST_L2_MAX = 2e-2
SUB_PYRAMID_P99 = 2e-2


def support_max_gradient(o, oc, lvl, xl, yl, sl):
    """largest central-difference gradient magnitude of the oracle's plane (oc, lvl) over each keypoint's descriptor
    support (the square of half-width 2.5 * 3 * sigma * sqrt(2) around it, inside [1, W-2] x [1, H-2])"""
    out = np.zeros(len(oc))
    planes = {}
    for j in range(len(oc)):
        key = (int(oc[j]), int(lvl[j]))
        if key not in planes:
            planes[key] = o.gauss(*key)
        p = planes[key]
        H, W = p.shape
        r = int(np.ceil(7.5 * float(sl[j]) * 1.4143)) + 2
        x0, x1 = max(1, int(xl[j]) - r), min(W - 2, int(xl[j]) + r)
        y0, y1 = max(1, int(yl[j]) - r), min(H - 2, int(yl[j]) + r)
        if x1 >= x0 and y1 >= y0:
            gx = p[y0:y1 + 1, x0 + 1:x1 + 2] - p[y0:y1 + 1, x0 - 1:x1]
            gy = p[y0 + 1:y1 + 2, x0:x1 + 1] - p[y0 - 1:y1, x0:x1 + 1]
            out[j] = np.hypot(gx, gy).max()
    return out


def check_foreign_l2(l2, o, image, mode, kname, what, kp, oc, lvl, xl, yl, sl):
    sub = sl < np.float32(1.6)
    low = (support_max_gradient(o, oc, lvl, xl, yl, sl) < LOW_CONTRAST) & ~sub
    rest = ~sub & ~low
    worst = np.argsort(-l2)[:4]
    p99 = float(np.percentile(l2[sub], 99)) if sub.any() else 0.0
    print("%s %s %s %s: %d descriptors, L2 max %.3g, %.3g on low-contrast supports (%d), sub-pyramid scales (%d) p99 %.3g "
          "max %.3g; worst: %s" % (
        image, mode, kname, what, len(l2), l2[rest].max(initial=0), l2[low].max(initial=0), low.sum(), sub.sum(), p99,
        l2[sub].max(initial=0),
        [(round(float(l2[j]), 5), round(float(sl[j]), 3), int(oc[j]), int(lvl[j]), round(float(kp["x"][j]), 2), round(float(kp["y"][j]), 2)) for j in worst]))
    # all other descriptors within L2_MAX, but for at most 0.1 % + 2 below 5 L2_MAX (measured on an H100: one of 2744 at
    # 1.08e-3 under GIVEN and one of 3225 at 2.03e-3 under ORIENT, both RootSift on binary block noise; none in the
    # classic modes)
    over = int((l2[rest] >= L2_MAX).sum())
    assert over <= 1e-3 * rest.sum() + 2 and l2[rest].max(initial=0) < 5 * L2_MAX, (kname, what, over, float(l2[rest].max(initial=0)))
    assert l2[low].max(initial=0) < LOW_CONTRAST_L2_MAX, (kname, what, float(l2[low].max(initial=0)))
    assert p99 < SUB_PYRAMID_P99, (kname, what, p99)


@pytest.mark.parametrize("mode,norm", MODES)
@pytest.mark.parametrize("image", FOREIGN_IMAGES)
def test_foreign_keypoints_vs_oracle(image, mode, norm):
    """Dense upright grids and seeded random keypoints: under GIVEN every descriptor is within 1e-3 L2 of orc_describe at
    the kernel's octave and level (predicted by the rule, confirmed by debug_octave); under ORIENT num_ori equals
    orc_orient's but for listed peak-ratio ties, angles agree within 1e-3 rad where the counts agree (but for a few on
    flat-topped histograms, see below), and descriptors are within 1e-3 of orc_describe at the kernel's angles (low-contrast
    supports: LOW_CONTRAST_L2_MAX)."""
    img = foreign_image(image)
    h, w = img.shape
    ps = api.PopSift(gpu_config(mode, norm), max_width=w, max_height=h, slots=1)
    o = ol.Oracle(ol.make_config(mode=mode, norm=norm), w, h)
    try:
        o.run(img, stages=1)
        f0 = ps.enqueue(w, h, img).get()          # fixes the slot's geometry
        assert f0 is not None
        dims = ps.slot_geometry(0)
        assert len(dims) == o.num_octaves
        # The grid is offset by a quarter pixel: at integer positions and these sigmas the edge of the descriptor's support
        # (|r| < 2.5 SBP) passes exactly through pixel centres, and under computed angles the last bit of __sincosf against
        # libm's sincosf decides whether a whole row of samples is in or out (both are right; up to 1e-2 L2 measured on
        # block_noise_4).
        for kname, kp in (("grid", grid_keypoints(w, h, offset=0.25)), ("random", random_keypoints(w, h, 3000, 17))):
            # GIVEN
            ok, oc, lvl, xl, yl, sl, S = dr.place(kp, ps._config.sigma, L, 1, dims, orient=False)
            g = describe(ps, img, kp)
            check_in_order(g, kp)
            assert np.array_equal(g.feat["num_ori"], ok.astype(np.int32)), (kname, "rejections")
            assert np.array_equal(g.feat["octave"], np.where(ok, oc, -1)), (kname, "octaves")
            idx = np.nonzero(ok)[0]
            got = g.desc[g.desc_idx[idx, 0]]
            want = o.describe(xl[idx], yl[idx], sl[idx], kp["ori"][idx], oc[idx], lvl[idx])
            l2 = _l2_vs(got, want)
            edge = dr.near_rounding_edge(S[idx], oc[idx], L)
            if edge.any():      # the other rounding of the level
                alt = o.describe(xl[idx], yl[idx], sl[idx], kp["ori"][idx], oc[idx], np.clip(lvl[idx] + np.where(S[idx] - oc[idx] * L > lvl[idx], 1, -1), 0, L + 2))
                l2 = np.where(edge, np.minimum(l2, _l2_vs(got, alt)), l2)
            check_foreign_l2(l2, o, image, mode, kname, "GIVEN", kp[idx], oc[idx], lvl[idx], xl[idx], yl[idx], sl[idx])
            assert len(idx) > 0.5 * len(kp)
            # ORIENT
            ok, oc, lvl, xl, yl, sl, S = dr.place(kp, ps._config.sigma, L, 1, dims, orient=True)
            r = describe(ps, img, kp, orient=True)
            check_in_order(r, kp)
            assert np.array_equal(r.feat["octave"], np.where(ok, oc, -1))
            assert (r.feat["num_ori"][~ok] == 0).all() and (r.feat["num_ori"][ok] >= 1).all()
            idx = np.nonzero(ok & ~dr.near_rounding_edge(S, oc, L))[0]
            num, ori = oo.orient(o, xl[idx], yl[idx], sl[idx], oc[idx], lvl[idx])
            mine = r.feat["num_ori"][idx]
            differ = np.nonzero(mine != num)[0]
            listed = {(round(float(kp["x"][idx[j]]), 3), round(float(kp["y"][idx[j]]), 3)) for j in differ}
            if len(differ):
                print("%s %s %s: orientation counts differ at %s" % (image, mode, kname, sorted(
                    (round(float(kp["x"][idx[j]]), 3), round(float(kp["y"][idx[j]]), 3), int(mine[j]), int(num[j])) for j in differ)))
            assert listed <= DESCRIBE_ORI_TIES.get((image, mode, kname), set()), (image, mode, kname)
            same = np.nonzero(mine == num)[0]
            n = mine[same].astype(np.int64)
            rows = np.repeat(same, n)
            k = np.arange(len(rows)) - np.repeat(np.cumsum(n) - n, n)
            ang_gpu = r.feat["ori"][idx[rows], k].astype(np.float64)
            dth = np.abs(np.angle(np.exp(1j * (ang_gpu - ori[rows, k]))))
            # On binary block noise the smoothed histograms have flat tops where the parabola refinement follows the last
            # bits of expf / hypotf / atan2f (CUDA math library here, libm in the oracle): up to 3.3e-2 rad measured.  Like
            # the pipeline comparison of test_stress_parity.py, at most 2 % + 4 of the angles may exceed the bar.
            far = int((dth >= 1e-3).sum())
            print("%s %s %s ORIENT: %d angles, %d beyond 1e-3 rad (max %.3g)" % (image, mode, kname, len(dth), far, dth.max(initial=0)))
            assert far <= 0.02 * len(dth) + 4, (kname, far, len(dth), float(dth.max(initial=0)))
            # descriptors at the kernel's angles, for every described keypoint
            n = r.feat["num_ori"][idx].astype(np.int64)
            rows = np.repeat(np.arange(len(idx)), n)
            k = np.arange(len(rows)) - np.repeat(np.cumsum(n) - n, n)
            got = r.desc[r.desc_idx[idx[rows], k]]
            want = o.describe(xl[idx][rows], yl[idx][rows], sl[idx][rows], r.feat["ori"][idx[rows], k], oc[idx][rows], lvl[idx][rows])
            l2 = _l2_vs(got, want)
            check_foreign_l2(l2, o, image, mode, kname, "ORIENT", kp[idx][rows], oc[idx][rows], lvl[idx][rows], xl[idx][rows],
                             yl[idx][rows], sl[idx][rows])
    finally:
        ps.uninit()
        o.close()


# --------------------------------------------------------------------------------- rejections and arguments

def test_rejected_keypoints_keep_their_place():
    """NaN / infinite coordinates, sigma <= 0, a NaN angle (GIVEN), positions outside the octave and bad explicit
    octaves / levels give num_ori = 0 in place, zero angles and the keypoint's own bits; the keypoints around them are
    described as without them."""
    img = make_frame(640, 480, 3)
    ps = api.PopSift(gpu_config(), max_width=640, max_height=480, slots=1)
    try:
        good = grid_keypoints(640, 480, step=40, sigmas=(2.5,))
        good["ori"] = np.linspace(-3, 3, len(good))
        bad = np.zeros(12, api.KEYPOINT_DTYPE)
        bad["x"], bad["y"], bad["sigma"], bad["octave"], bad["level"] = 100, 100, 2.0, -1, -1
        bad["x"][0] = np.nan
        bad["y"][1] = np.inf
        bad["sigma"][2] = 0.0
        bad["sigma"][3] = -1.0
        bad["sigma"][4] = np.nan
        bad["x"][5] = -0.5
        bad["x"][6] = 700.0
        bad["octave"][7] = 99
        bad["octave"][8] = -2
        bad["level"][9] = L + 3
        bad["level"][10] = -5
        bad["ori"][11] = np.nan                        # rejected under GIVEN only
        pos = np.sort(np.random.default_rng(2).choice(len(good) + len(bad), len(bad), replace=False))
        mixed = np.zeros(len(good) + len(bad), api.KEYPOINT_DTYPE)
        is_bad = np.zeros(len(mixed), bool)
        is_bad[pos] = True
        mixed[is_bad] = bad
        mixed[~is_bad] = good
        for orient in (False, True):
            ref = describe(ps, img, good, orient)
            got = describe(ps, img, mixed, orient)
            check_in_order(got, mixed)
            rej = is_bad.copy()
            if orient:
                rej[pos[11]] = False
            assert (got.feat["num_ori"][rej] == 0).all() and (got.feat["ori"][rej] == 0).all()
            assert (got.feat["octave"][rej] == -1).all()
            keep = ~is_bad
            assert np.array_equal(got.feat["num_ori"][keep], ref.feat["num_ori"])
            assert np.array_equal(bits(got.feat["ori"][keep]), bits(ref.feat["ori"]))
            gi = np.nonzero(keep)[0]
            n = ref.feat["num_ori"].astype(np.int64)
            rows = np.repeat(np.arange(len(n)), n)
            k = np.arange(len(rows)) - np.repeat(np.cumsum(n) - n, n)
            assert np.array_equal(bits(got.desc[got.desc_idx[gi[rows], k]]), bits(ref.desc[ref.desc_idx[rows, k]]))
    finally:
        ps.uninit()


def test_describe_argument_errors():
    """n < 0, keypoints NULL with n > 0 and unknown flags give PS_ERR_ARG, an image beyond the context PS_ERR_TOO_LARGE;
    n = 0 is valid and gives zero features."""
    lib = api.load_library()
    img = make_frame(320, 240, 1)
    ps = api.PopSift(gpu_config(), max_width=320, max_height=240, slots=1)
    try:
        kp = api.keypoints_array([[10.0, 10.0, 2.0, 0.0]])
        ctx = ps._ctx
        assert lib.ps_describe_u8(ctx, 0, img.ctypes.data, 320, 240, kp.ctypes.data, -1, 0) == -1
        assert lib.ps_describe_u8(ctx, 0, img.ctypes.data, 320, 240, None, 1, 0) == -1
        assert lib.ps_describe_u8(ctx, 0, img.ctypes.data, 320, 240, kp.ctypes.data, 1, 2) == -1
        assert lib.ps_describe_u8(ctx, 0, img.ctypes.data, 320, 240, kp.ctypes.data, 1, -1) == -1
        assert lib.ps_describe_u8(ctx, 5, img.ctypes.data, 320, 240, kp.ctypes.data, 1, 0) == -1
        big = np.zeros((480, 640), np.uint8)
        assert lib.ps_describe_u8(ctx, 0, big.ctypes.data, 640, 480, kp.ctypes.data, 1, 0) == -3
        f = describe(ps, img, np.zeros(0, api.KEYPOINT_DTYPE), True)
        assert f.getFeatureCount() == 0 and f.getDescriptorCount() == 0
        f = describe(ps, img, kp)
        assert f.getFeatureCount() == 1 and f.getDescriptorCount() == 1
    finally:
        ps.uninit()


# ------------------------------------------------------------------------------------------------- capacity

def test_300k_keypoints_equal_three_calls_of_100k():
    """One ORIENT call with 300 000 keypoints (beyond the slot's 2 x max_extrema records) equals three calls of 100 000,
    concatenated."""
    img = make_frame(1920, 1080, 4)
    kp = random_keypoints(1920, 1080, 300000, 23)
    kp["sigma"] = np.exp(np.random.default_rng(3).uniform(np.log(1.0), np.log(20.0), len(kp)))
    ps = api.PopSift(gpu_config(), max_width=1920, max_height=1080, slots=1)
    try:
        parts = [describe(ps, img, kp[i:i + 100000], True) for i in range(0, 300000, 100000)]
        parts = [(p.feat.copy(), p.desc_idx.copy(), p.desc.copy()) for p in parts]
        whole = describe(ps, img, kp, True)
        num = np.concatenate([p[0]["num_ori"] for p in parts])
        assert np.array_equal(whole.feat["num_ori"], num) and num.sum() > 300000
        assert np.array_equal(bits(whole.feat["ori"]), bits(np.concatenate([p[0]["ori"] for p in parts])))
        assert np.array_equal(bits(whole.desc), bits(np.concatenate([p[2] for p in parts])))
    finally:
        ps.uninit()


_SUBPROCESS_RUN = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import test_describe as td
from popsift_b200 import api
from popsift_b200.synth import make_frame
img = make_frame(1280, 720, 9)
kp = td.random_keypoints(1280, 720, 20000, 31)
ps = api.PopSift(td.gpu_config(), max_width=1280, max_height=720, slots=1)
out = {}
for orient in (False, True):
    f = td.describe(ps, img, kp, orient)
    for a, v in td.feature_fields(f).items():
        out["%s%d" % (a, orient)] = v
    out["desc%d" % orient] = f.desc.copy()
f = ps.enqueue(1280, 720, img).get()
out["extract"] = td.canonical(f)
ps.uninit()
np.savez(sys.argv[3], **out)
"""


def _run_in_subprocess(env_extra, path):
    env = dict(os.environ, **env_extra)
    r = subprocess.run([sys.executable, "-c", _SUBPROCESS_RUN, HERE, ROOT, str(path)], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return dict(np.load(str(path)))


def test_tiny_initial_capacity_gives_the_same_results(tmp_path):
    """With POPSIFT_B200_INIT_CAP=100 every buffer grows on the way (records before the launch, ORIENT's descriptors
    through the overflow re-run); the results equal the default capacity's."""
    base = _run_in_subprocess({}, tmp_path / "base.npz")
    small = _run_in_subprocess({"POPSIFT_B200_INIT_CAP": "100"}, tmp_path / "small.npz")
    assert len(base["desc1"]) > 20000
    for k, v in base.items():
        assert small[k].shape == v.shape and small[k].tobytes() == v.tobytes(), k


# ------------------------------------------------------------------------------------------------ shared slot

def canonical(f):
    """an extraction's (octave, x, y, sigma, angle, descriptor) rows, sorted: the order of detected extrema is not fixed"""
    n = f.feat["num_ori"].astype(np.int64)
    i = np.repeat(np.arange(len(n)), n)
    k = np.arange(len(i)) - np.repeat(np.cumsum(n) - n, n)
    rows = np.concatenate([np.stack([f.feat["octave"][i], f.feat["x"][i], f.feat["y"][i], f.feat["sigma"][i], f.feat["ori"][i, k]], 1),
                           f.desc[f.desc_idx[i, k]]], 1).astype(np.float64).reshape(-1, 133)
    return rows[np.lexsort(rows.T[::-1])]


def _snapshot(f, detected):
    if detected:
        return (len(f.feat), canonical(f).tobytes())
    return tuple(v.tobytes() for v in feature_fields(f).values()) + (f.desc.tobytes(), f.desc_idx.tobytes())


def test_detect_and_describe_share_a_slot():
    """Detection and describe calls interleaved on one slot, with enough same-size frames that the detection graph is
    captured and replayed, and describe calls that grow the slot's buffers: every result equals a fresh context's."""
    cfg = gpu_config()
    cfg._c.max_extrema = 2000                        # slot capacity 4000 records: the 6000-keypoint call grows it
    frames = [make_frame(640, 480, s) for s in (1, 2)]
    kps = {"small": random_keypoints(640, 480, 500, 3), "large": random_keypoints(640, 480, 6000, 4)}

    def fresh(op, fi, kname=None, orient=False):
        ps = api.PopSift(cfg, max_width=640, max_height=480, slots=1)
        try:
            f = ps.enqueue(640, 480, frames[fi]).get() if op == "detect" else describe(ps, frames[fi], kps[kname], orient)
            return _snapshot(f, op == "detect")
        finally:
            ps.uninit()

    plan = [("detect", 0), ("detect", 1), ("describe", 0, "small", False), ("detect", 0), ("detect", 1),
            ("describe", 1, "small", True), ("detect", 0), ("describe", 0, "large", True), ("detect", 1), ("detect", 0),
            ("detect", 1), ("describe", 1, "large", False), ("detect", 0)]
    want = {}
    ps = api.PopSift(cfg, max_width=640, max_height=480, slots=1)
    try:
        for step in plan:
            if step not in want:
                want[step] = fresh(*step)
            f = ps.enqueue(640, 480, frames[step[1]]).get() if step[0] == "detect" else describe(ps, frames[step[1]], kps[step[2]], step[3])
            assert _snapshot(f, step[0] == "detect") == want[step], step
    finally:
        ps.uninit()


# ------------------------------------------------------------------------------------------------ other modes

def test_grid_desc_mode_and_float_images_round_trip():
    """desc_mode grid, and float images through ps_describe_f32: the round trip with the given angles is bit-identical
    to the extraction in the same configuration."""
    img = make_frame(640, 480, 6)
    for desc_mode, imode in (("grid", api.PopSift.ByteImages), ("loop", api.PopSift.FloatImages), ("igrid", api.PopSift.FloatImages)):
        cfg = gpu_config("vlfeat", "classic")
        cfg.setDescMode(desc_mode)
        x = img.astype(np.float32) / np.float32(255.0) if imode == api.PopSift.FloatImages else img
        ps = api.PopSift(cfg, imode=imode, max_width=640, max_height=480, slots=1)
        try:
            f, ext = extract(ps, x)
            kp, didx = per_desc_keypoints(f, ext)
            g = describe(ps, x, kp)
            assert f.getDescriptorCount() > 100
            assert np.array_equal(bits(g.desc), bits(f.desc[didx])), (desc_mode, imode)
            kf = per_feature_keypoints(f, ext)
            r = describe(ps, x, kf, True)
            assert np.array_equal(bits(r.desc), bits(f.desc)), (desc_mode, imode)
        finally:
            ps.uninit()


def test_matching_mode_features_dev_from_describe():
    """Under MatchingMode, describe gives a FeaturesDev; api.match_pairs of it against an extracted frame equals matching
    the downloaded descriptor arrays, and its reverse map points into input order."""
    img_a, img_b = make_frame(640, 480, 7), make_frame(640, 480, 8)
    ps = api.PopSift(gpu_config(), mode=api.Config.MatchingMode, max_width=640, max_height=480, slots=1)
    try:
        fb = ps.enqueue(640, 480, img_b).getDev()
        kp = grid_keypoints(640, 480, step=16)
        fa = ps.describe(640, 480, img_a, kp, orientations=True).getDev()
        assert fa.getFeatureCount() == len(kp)
        feat, desc, rev = fa.to_host()
        n = feat["num_ori"].astype(np.int64)
        assert np.array_equal(rev, np.repeat(np.arange(len(kp)), n).astype(np.int32))
        _, desc_b, _ = fb.to_host()
        got = api.match_pairs([fa, fb], [(0, 1), (1, 0)])
        want = api.match_pairs([desc, desc_b], [(0, 1), (1, 0)])
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
    finally:
        ps.uninit()


def test_cpp_describe_round_trip(tmp_path):
    """PopSift::describe (C++ API), describe and enqueue jobs interleaved in one FIFO (tests/cpp/describe_check.cpp)."""
    from popsift_b200 import build as B
    exe = B.DESCRIBE_CHECK
    assert os.path.exists(exe), "build the product first (python -m popsift_b200.build)"
    f = str(tmp_path / "frame.raw")
    make_frame(1280, 720, 12).tofile(f)
    out = subprocess.run([exe, "1280", "720", f], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK "), out.stdout + out.stderr
