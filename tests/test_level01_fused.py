"""Levels 0 and 1 of octave 0 in one launch (march_level01x2_kernel): on the default path (8-bit input up-scaled exactly
2x) the fused launch must give the same bytes as the two separate launches it replaces (POPSIFT_B200_FUSE_L0=0), in every
plane, feature and descriptor, directly and from the slot's captured graph; every other path must not take it."""
import hashlib
import os
import sys

import numpy as np
import pytest

from popsift_b200 import api
from popsift_b200.synth import make_frame

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (w, h): the benchmark frame; a width whose octave 0 (2w) is not a multiple of the 128-column strip; a frame whose
# octave 0 is one chunk-row high (one segment holds the top and the bottom border); 640x480
SIZES = [(3840, 2160), (1000, 600), (333, 8), (640, 480)]
LEVELS = 3              # the default Config


def _frame(w, h, seed=7):
    if (w, h) == (3840, 2160):
        sys.path.insert(0, ROOT)
        import bench
        return bench.synth_frames(1, 0)[0]
    return make_frame(w, h, seed)


def _cfg(mode=None, direct=False, downsampling=None):
    c = api.Config()
    if mode:
        c.setMode(mode)
    if direct:
        c.setScalingMode(0)
    if downsampling is not None:
        c.setDownsampling(downsampling)
    return c


def _ctx(monkeypatch, fuse, cfg, w, h, **kw):
    monkeypatch.setenv("POPSIFT_B200_FUSE_L0", "1" if fuse else "0")
    return api.PopSift(cfg, max_width=w, max_height=h, slots=1, **kw)


def _digests(ps, levels):
    """sha256 of every Gaussian plane of every octave, in order"""
    return [hashlib.sha256(ps.plane(0, oc, l).tobytes()).hexdigest()
            for oc in range(len(ps.slot_geometry(0))) for l in range(levels + 3)]


def _features(feats):
    """keypoints and descriptors in a canonical order (the order of the output lists is not part of the result)"""
    k, d = feats.keypoints()
    o = np.lexsort(k.T[::-1])
    return k[o].tobytes(), d[o].tobytes()


def _run(monkeypatch, fuse, cfg, w, h, frames, **kw):
    ps = _ctx(monkeypatch, fuse, cfg, w, h, **kw)
    out = []
    for f in frames:
        before = ps.launch_count()
        feats = ps.enqueue(w, h, f).get()
        out.append((_features(feats), _digests(ps, LEVELS), ps.launch_count() - before))
    ps._check(ps._lib.ps_run_pyramid_only(ps._ctx, 0))
    after_pyramid_only = _digests(ps, LEVELS)
    ps.uninit()
    return out, after_pyramid_only


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("mode", [None, "vlfeat"])
def test_fused_planes_and_features_identical(monkeypatch, w, h, mode):
    f = _frame(w, h)
    (fused,), fused_po = _run(monkeypatch, True, _cfg(mode), w, h, [f])
    (sep,), sep_po = _run(monkeypatch, False, _cfg(mode), w, h, [f])
    (ff, fd), (sf, sd) = fused[0], sep[0]
    # octave 0 first (the planes the fused launch writes), then the whole pyramid
    assert fused[1][:LEVELS + 3] == sep[1][:LEVELS + 3]
    assert fused[1] == sep[1]
    assert ff == sf and fd == sd
    assert len(ff) > 0 or (w, h) == (333, 8)
    assert fused_po == sep_po == fused[1]
    # one launch fewer per pyramid on the fused path
    assert sep[2] - fused[2] == 1


def test_fused_graph_replay(monkeypatch):
    """the first image of a geometry runs directly, the second is captured, the third replays the graph"""
    w, h = 1000, 600
    frames = [make_frame(w, h, s) for s in (11, 12, 13)]
    fused, fused_po = _run(monkeypatch, True, _cfg(), w, h, frames)
    sep, sep_po = _run(monkeypatch, False, _cfg(), w, h, frames)
    for a, b in zip(fused, sep):
        assert a[0] == b[0] and a[1] == b[1]
        assert b[2] - a[2] == 1
    assert fused_po == sep_po == fused[2][1]
    assert fused[1][1] != fused[2][1]          # the replayed graph read the third image, not the second


@pytest.mark.parametrize("case", ["float", "no_upscale", "direct"])
def test_unfused_paths_unchanged(monkeypatch, case):
    """float input, octave 0 at the input size and direct scaling keep the two launches: same launch count with the
    switch on and off (their planes and features against the reference are pinned by the parity tests)"""
    w, h = 640, 480
    kw = {}
    f = make_frame(w, h, 5)
    if case == "float":
        kw = {"imode": api.PopSift.FloatImages}
        f = f.astype(np.float32) / 255.0
        mk = lambda: _cfg()
    elif case == "no_upscale":
        mk = lambda: _cfg(downsampling=0)
    else:
        mk = lambda: _cfg(direct=True)
    (on,), on_po = _run(monkeypatch, True, mk(), w, h, [f], **kw)
    (off,), off_po = _run(monkeypatch, False, mk(), w, h, [f], **kw)
    assert on[2] == off[2]
    assert on[0] == off[0] and on[1] == off[1] and on_po == off_po
