"""CPU checks for the describe path (ps_describe_u8 / ps_describe_f32): the keypoint layout, the numpy restatement of the
octave / level rule that tests/test_describe.py uses, and the oracle's orientation stage on caller-given keypoints."""
import numpy as np

import describe_rule as dr
import oracle_lib as ol
import orient_oracle as oo
from popsift_b200 import api
from popsift_b200.synth import make_frame


def test_keypoint_layout_is_24_bytes():
    dt = api.KEYPOINT_DTYPE
    assert dt.itemsize == 24
    assert [dt.fields[k][1] for k in ("x", "y", "sigma", "ori", "octave", "level")] == [0, 4, 8, 12, 16, 20]
    kp = api.keypoints_array([[1.0, 2.0, 3.0, 0.5], [4.0, 5.0, 6.0, -0.5]])
    assert kp.dtype == dt and list(kp["octave"]) == [-1, -1] and list(kp["level"]) == [-1, -1]
    assert np.array_equal(kp["ori"], np.float32([0.5, -0.5]))


# (S, octave, level) for L = 3 and 5 octaves, worked by hand from
#   octave = clamp(floor((S - 0.5) / L), 0, 4),  level = clamp(roundf(S - octave * L), 0, 5)
S_CASES = [
    (0.5, 0, 1),      # half-integer: roundf(0.5) = 1, not banker's 0
    (2.5, 0, 3),      # roundf(2.5) = 3
    (3.5, 1, 1),      # (3.5 - 0.5) / 3 = 1 exactly: octave 1, roundf(0.5) = 1
    (5.5, 1, 3),
    (6.5, 2, 1),
    (3.0, 0, 3),      # a detected lpos = L stays in its octave
    (1.0, 0, 1),
    (-0.5, 0, 0),     # below octave 0: octave clamped to 0, roundf(-0.5) = -1 clamped to 0
    (-10.0, 0, 0),
    (14.4, 4, 2),
    (15.5, 4, 4),     # above the top octave: floor(5) clamped to 4, roundf(3.5) = 4
    (100.0, 4, 5),    # level clamped to L + 2
]


def test_octave_level_rule_hand_cases():
    S = np.array([c[0] for c in S_CASES], np.float32)
    o, lvl = dr.octave_level_from_s(S, 3, 5)
    assert list(o) == [c[1] for c in S_CASES]
    assert list(lvl) == [c[2] for c in S_CASES]


# (sigma, up_fac, octave, level) with sigma0 = 1, L = 3, 5 octaves: log2 of a power of two is exact, so S is exact
SIGMA_CASES = [
    (4.0, 1, 2, 3),        # S = 3 * (2 + 1) = 9
    (4.0, 0, 1, 3),        # S = 6
    (1.0, 1, 0, 3),        # S = 3
    (1.0, 0, 0, 0),        # S = 0: floor(-1/6) = -1 clamped to 0
    (0.125, 1, 0, 0),      # S = -6: below octave 0
    (0.125, 0, 0, 0),
    (1024.0, 1, 4, 5),     # S = 33: above the top octave, level clamped to L + 2
    (1024.0, 0, 4, 5),
    (16.0, 0, 3, 3),       # S = 12: floor(11.5 / 3) = 3, level roundf(12 - 9) = 3
    (2.0, 0, 0, 3),        # S = 3: lpos L of octave 0
]


def test_octave_level_rule_from_sigma_with_up_fac_0_and_1():
    for sigma, up, o_want, l_want in SIGMA_CASES:
        o, lvl, S = dr.octave_level(np.float32([sigma]), 1.0, 3, up, 5)
        assert (int(o[0]), int(lvl[0])) == (o_want, l_want), (sigma, up, float(S[0]))


def test_explicit_octave_keeps_the_derived_level_rule():
    # octave 2 given, level derived: roundf(S - 6)
    o, lvl = dr.octave_level_from_s(np.float32([6.4, 9.5, 1.0]), 3, 5, octave=np.array([2, 2, 2]))
    assert list(o) == [2, 2, 2] and list(lvl) == [0, 4, 0]


def test_rule_gives_back_detected_octave_and_level():
    """On the oracle's extrema (input-image sigma = local sigma * 2^(octave - up_fac)), the rule gives back (octave, lpos)
    for 1 <= lpos <= L, except where S is within float rounding of a half-integer."""
    img = make_frame(640, 480, 3)
    for up in (1, 0):
        cfg = ol.make_config(upscale=float(up))
        o = ol.Oracle(cfg, 640, 480)
        try:
            o.run(img, stages=3)
            ex = o.extrema()
            lpos, octv = ex[:, 3].astype(np.int64), ex[:, 4].astype(np.int64)
            sig = (ex[:, 2] * np.ldexp(np.float32(1), (octv - up).astype(np.int32))).astype(np.float32)
            m = (lpos >= 1) & (lpos <= 3)
            oo, ll, S = dr.octave_level(sig, cfg.sigma, 3, up, o.num_octaves)
            edge = dr.near_rounding_edge(S, octv, 3)
            good = m & ~edge
            assert good.sum() > 200
            assert np.array_equal(oo[good], octv[good]) and np.array_equal(ll[good], lpos[good]), up
        finally:
            o.close()


def test_orc_orient_reproduces_the_oracle_pipeline():
    """orc_orient on the oracle's own extrema gives the pipeline's num_ori and angles bit for bit."""
    img = make_frame(640, 480, 1)
    for mode in ("popsift", "vlfeat"):
        o = ol.Oracle(ol.make_config(mode=mode), 640, 480)
        try:
            o.run(img, stages=7)
            ex = o.extrema()
            feat, _ = o.features()
            assert len(ex) == len(feat) > 200
            num, ori = oo.orient(o, ex[:, 0], ex[:, 1], ex[:, 2], ex[:, 4].astype(np.int32), ex[:, 3].astype(np.int32))
            assert np.array_equal(num, feat["num_ori"])
            want = np.where(np.arange(4)[None, :] < feat["num_ori"][:, None], feat["ori"], 0.0).astype(np.float32)
            assert np.array_equal(ori.view(np.uint32), want.view(np.uint32))
        finally:
            o.close()
