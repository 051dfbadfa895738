"""The DoG planes are written only on request: an extraction neither writes nor reads a slot's DoG region (the extrema
stage forms every DoG sample from two Gaussian planes), and ps_debug_plane(PS_PLANE_DOG) fills the octave's planes from
the Gaussian levels the slot holds when it is asked for one."""
import os
import subprocess
import sys

import numpy as np
import pytest

from popsift_b200 import api
from popsift_b200.synth import make_frame

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
W, H = 640, 480


def _cfg(gauss_mode=None):
    c = api.Config()
    if gauss_mode:
        c.setGaussMode(gauss_mode)
    return c


def _sorted(feats):
    k, d = feats.keypoints()
    o = np.lexsort(k.T[::-1])
    return k[o], d[o]


def _dog_planes(ps, slot):
    L = ps._config.levels
    return [[ps.plane(slot, oc, l, dog=True) for l in range(L + 2)] for oc in range(len(ps.slot_geometry(slot)))]


def extraction_ignores_dog_region(gauss_mode=None):
    """frame B alone in a fresh context == frame B in a slot whose DoG region holds frame A's materialised planes, with
    B's pipeline replayed from the captured graph (A runs directly, then under capture)"""
    a, b = make_frame(W, H, 41), make_frame(W, H, 42)
    ps = api.PopSift(_cfg(gauss_mode), max_width=W, max_height=H, slots=1)
    kb, db = _sorted(ps.enqueue(W, H, b).get())
    ps.uninit()
    ps = api.PopSift(_cfg(gauss_mode), max_width=W, max_height=H, slots=1)
    ps.enqueue(W, H, a).get()
    ps.enqueue(W, H, a).get()
    dogs_a = _dog_planes(ps, 0)
    assert any(np.abs(p).max() > 0 for planes in dogs_a for p in planes)
    kb2, db2 = _sorted(ps.enqueue(W, H, b).get())
    ps.uninit()
    assert len(kb) > 20
    assert np.array_equal(kb, kb2) and np.array_equal(db, db2)


@pytest.mark.parametrize("gauss_mode", [None, "fixed9"])
def test_extraction_ignores_dog_region(gauss_mode):
    extraction_ignores_dog_region(gauss_mode)


@pytest.mark.parametrize("env", ["POPSIFT_B200_DENSE_SCAN", "POPSIFT_B200_TILE_KERNELS"])
def test_extraction_ignores_dog_region_other_paths(env):
    """the dense extrema scan and the tile pyramid kernels: the switches are read once per process"""
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_dog_on_demand as t; t.extraction_ignores_dog_region(); print('ok')"
            % (ROOT, HERE))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **{env: "1"}), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-2000:]


def _check_on_demand(ps, slot):
    L = ps._config.levels
    for oc in range(len(ps.slot_geometry(slot))):
        g = [ps.plane(slot, oc, l) for l in range(L + 3)]
        for l in range(L + 2):
            assert np.array_equal(ps.plane(slot, oc, l, dog=True), g[l + 1] - g[l]), (oc, l)


def test_dog_on_demand_after_graph_replay():
    ps = api.PopSift(_cfg(), max_width=W, max_height=H, slots=1)
    for seed in (43, 44, 45):                     # direct, captured, replayed
        ps.enqueue(W, H, make_frame(W, H, seed)).get()
    _check_on_demand(ps, 0)
    ps.uninit()


def test_dog_on_demand_after_pyramid_only():
    ps = api.PopSift(_cfg(), max_width=W, max_height=H, slots=1)
    ps.enqueue(W, H, make_frame(W, H, 46)).get()
    _check_on_demand(ps, 0)                        # materialise the planes of this image ...
    ps._check(ps._lib.ps_run_pyramid_only(ps._ctx, 0))
    _check_on_demand(ps, 0)                        # ... and again after the pyramid alone ran once more
    ps.uninit()


def test_dog_on_demand_after_describe():
    ps = api.PopSift(_cfg(), max_width=W, max_height=H, slots=1)
    kp = np.array([[100.0, 120.0, 2.0, 0.5], [320.0, 240.0, 4.0, 1.0], [500.5, 300.25, 8.0, -2.0]], np.float32)
    f = ps.describe(W, H, make_frame(W, H, 47), kp).get()
    assert f.getFeatureCount() == len(kp)
    _check_on_demand(ps, 0)
    ps.uninit()
