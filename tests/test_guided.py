"""Guided matching on the GPU (ps_match_guided_batch / ps_match_u8_guided_batch): tensor rows against the CUDA-core
guided kernels and against the masked 2-NN oracle on the kernels' own eligibility mask, the unguided matcher as the limit
of a test that admits everything, large and multi-group batches, an end-to-end run on synth.affine_set, argument errors
and the C++ API."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import guided_oracle as go
from popsift_b200 import api
from popsift_b200.synth import affine_set

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTO, EXACT, TENSOR = 0, 1, 2
PS_ERR_ARG = -1
W, H = 1920, 1080
SIZES = [0, 1, 2, 127, 129, 1000, 4097, 7000]


def _dev_set(lib, desc, xy, rng=None):
    """a FeaturesDev with one Feature per descriptor at the given pixel positions, the reverse map a permutation"""
    n = len(desc)
    fd = api.FeaturesDev(lib, n, n)
    perm = np.arange(n, dtype=np.int32) if rng is None else rng.permutation(n).astype(np.int32)
    feat = np.zeros(n, api.FEATURE_DTYPE)
    feat["x"][perm] = xy[:, 0]
    feat["y"][perm] = xy[:, 1]
    feat["num_ori"] = 1
    for arr, ptr in ((feat, fd.getFeatures()), (np.ascontiguousarray(desc, np.float32), fd.getDescriptors()), (perm, fd.getReverseMap())):
        if arr.nbytes:
            assert lib.ps_host_to_dev(ptr, arr.ctypes.data, arr.nbytes) == 0
    return fd


def _unit(rng, n):
    d = np.abs(rng.normal(size=(n, 128))).astype(np.float32)
    return d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12).astype(np.float32)


def _random_sets(seed, u8=False):
    """SIZES descriptors with planted near-duplicates between sets (float unit vectors, or integer-valued 8-bit ones)"""
    rng = np.random.default_rng(seed)
    sets = [_unit(rng, n) for n in SIZES]
    sets[7][100:600] = sets[6][:500] + rng.normal(scale=0.01, size=(500, 128)).astype(np.float32)
    sets[5][:120] = sets[4][:120] + rng.normal(scale=0.01, size=(120, 128)).astype(np.float32)
    sets[6][3000:3900] = sets[5][:900] + rng.normal(scale=0.005, size=(900, 128)).astype(np.float32)
    sets[3][:2] = sets[2] + rng.normal(scale=0.01, size=(2, 128)).astype(np.float32)
    if u8:
        sets = [np.clip(np.round(np.abs(s) * 512), 0, 255).astype(np.float32) for s in sets]
    pts = [rng.uniform([0, 0], [W, H], (n, 2)).astype(np.float32) for n in SIZES]
    return sets, pts, rng


def _models(kind, rng, n):
    return np.stack([(go.random_homography(rng) if kind == go.HOMOGRAPHY else go.random_fundamental(rng)).astype(np.float32)
                     for _ in range(n)])


def _check_oracle(sets, pts, pairs, models, kind, t, rows, rng, per_pair=48):
    """rows == the masked 2-NN oracle on the guided_mask mask (every row of small left sets, `per_pair` sampled otherwise);
    returns the eligible fraction seen"""
    elig = tot = 0
    for p, (l, r) in enumerate(pairs):
        nl, nr = len(sets[l]), len(sets[r])
        if nl == 0:
            assert len(rows[p]) == 0
            continue
        sel = np.arange(nl) if nl <= 2 * per_pair else np.sort(rng.choice(nl, per_pair, replace=False))
        mask = go.mask_exact(kind, t, models[p], pts[l][sel], pts[r])
        want = go.guided_rows(sets[l][sel], sets[r], mask)
        assert np.array_equal(rows[p][sel], want), (l, r, t)
        elig += int(mask.sum()); tot += mask.size
    return elig / max(tot, 1)


# thresholds (pixels) with about 1 %, 10 % and 50 % of the right points eligible on 1920 x 1080 uniform points
THRESHOLDS = {go.HOMOGRAPHY: (80.0, 260.0, 640.0), go.FUNDAMENTAL: (8.0, 75.0, 420.0)}
FRACTIONS = (0.01, 0.10, 0.50)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [go.HOMOGRAPHY, go.FUNDAMENTAL])
def test_guided_rows_tensor_exact_oracle(kind):
    """all 64 ordered pairs of {0, 1, 2, 127, 129, 1000, 4097, 7000} descriptors in one call, a random model per pair, three
    thresholds: AUTO == TENSOR == EXACT, bit for bit, and == the oracle on the kernels' own mask"""
    lib = api.load_library()
    sets, pts, rng = _random_sets(11)
    devs = [_dev_set(lib, s, p, rng) for s, p in zip(sets, pts)]
    pairs = [(i, j) for i in range(len(SIZES)) for j in range(len(SIZES))]
    models = _models(kind, rng, len(pairs))
    name = "homography" if kind == go.HOMOGRAPHY else "fundamental"
    for t, frac in zip(THRESHOLDS[kind], FRACTIONS):
        ex = api.match_pairs_guided(devs, pairs, models, name, t, EXACT)
        for flags in (AUTO, TENSOR):
            got = api.match_pairs_guided(devs, pairs, models, name, t, flags)
            for p in range(len(pairs)):
                assert np.array_equal(got[p], ex[p]), (flags, pairs[p], t)
        seen = _check_oracle(sets, pts, pairs, models, kind, t, ex, rng)
        print("%s t=%g: eligible fraction %.4f" % (name, t, seen))
        assert frac / 3 < seen < min(3 * frac, 0.8), (t, seen)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [go.HOMOGRAPHY, go.FUNDAMENTAL])
def test_guided_u8_rows(kind):
    """8-bit sets: TENSOR == EXACT == the float EXACT guided rows on float32 copies == the oracle"""
    lib = api.load_library()
    sets, pts, rng = _random_sets(12, u8=True)
    devs = [_dev_set(lib, s, p, rng) for s, p in zip(sets, pts)]
    pairs = [(i, j) for i in range(len(SIZES)) for j in range(len(SIZES))]
    models = _models(kind, rng, len(pairs))
    name = "homography" if kind == go.HOMOGRAPHY else "fundamental"
    for t in THRESHOLDS[kind]:
        ex = api.match_pairs_guided(devs, pairs, models, name, t, EXACT, u8=True)
        fl = api.match_pairs_guided(devs, pairs, models, name, t, EXACT)
        for flags in (AUTO, TENSOR):
            got = api.match_pairs_guided(devs, pairs, models, name, t, flags, u8=True)
            for p in range(len(pairs)):
                assert np.array_equal(got[p], ex[p]), (flags, pairs[p], t)
        for p in range(len(pairs)):
            assert np.array_equal(ex[p], fl[p]), (pairs[p], t)
        _check_oracle(sets, pts, pairs, models, kind, t, ex, rng, per_pair=24)


def _plan(sizes, pairs, row_bytes, cap=1 << 30, sms=132):
    from popsift_b200 import build as B
    B.build()
    return subprocess.run([B.MATCH_PLAN_U8_CHECK, "plan", str(sms), str(cap), ",".join(map(str, sizes)),
                           ",".join(str(v) for p in pairs for v in p), str(row_bytes)], capture_output=True, text=True, check=True).stdout


@pytest.mark.gpu
def test_everything_eligible_equals_unguided():
    """H = I with t = 10^6 px admits every right descriptor: guided rows == match_pairs / match_pairs_u8 rows (at these
    sizes the 8-byte larger rows leave the plan unchanged); zero models give (0, 0, 0) everywhere"""
    lib = api.load_library()
    pairs = [(i, j) for i in range(len(SIZES)) for j in range(len(SIZES))]
    assert _plan(SIZES, pairs, 1028) == _plan(SIZES, pairs, 1036)
    assert _plan(SIZES, pairs, 132) == _plan(SIZES, pairs, 140)
    eye = np.tile(np.eye(3, dtype=np.float32), (len(pairs), 1, 1))
    zero = np.zeros_like(eye)
    for u8 in (False, True):
        sets, pts, rng = _random_sets(13, u8)
        devs = [_dev_set(lib, s, p, rng) for s, p in zip(sets, pts)]
        for flags in (AUTO, EXACT):
            want = api.match_pairs_u8(devs, pairs, flags) if u8 else api.match_pairs(devs, pairs, flags)
            got = api.match_pairs_guided(devs, pairs, eye, "homography", 1e6, flags, u8=u8)
            for p in range(len(pairs)):
                assert np.array_equal(got[p], want[p]), (u8, flags, pairs[p])
            for name in ("homography", "fundamental"):
                got = api.match_pairs_guided(devs, pairs, zero, name, 1e6, flags, u8=u8)
                assert all((g == 0).all() for g in got), (u8, flags, name)


def _planted_pair(rng, nl, nr, Hm):
    """left set, right set with the left descriptors planted at known right rows, right points consistent with Hm there"""
    l, r = _unit(rng, nl), _unit(rng, nr)
    at = rng.choice(nr, nl, replace=False)
    r[at] = l + rng.normal(scale=0.01, size=l.shape).astype(np.float32)
    pl = rng.uniform([0, 0], [W, H], (nl, 2))
    pr = rng.uniform([0, 0], [W, H], (nr, 2))
    hl = np.c_[pl, np.ones(nl)] @ Hm.T
    pr[at] = hl[:, :2] / hl[:, 2:3]
    return l, r, pl.astype(np.float32), pr.astype(np.float32), at


@pytest.mark.gpu
def test_large_right_sets_split_in_chunks():
    """64 x 60 000 and 200 x 50 000 (S = 8 chunks per pair): AUTO == TENSOR == EXACT, and the planted matches are found"""
    lib = api.load_library()
    rng = np.random.default_rng(21)
    H1, H2 = go.random_homography(rng), go.random_homography(rng)
    a, b, pa, pb, at1 = _planted_pair(rng, 64, 60000, H1)
    c, d, pc, pd, at2 = _planted_pair(rng, 200, 50000, H2)
    assert _plan([64, 60000, 200, 50000], [(0, 1), (2, 3)], 1036).startswith("groups=1 S=8,")
    devs = [_dev_set(lib, s, p, rng) for s, p in ((a, pa), (b, pb), (c, pc), (d, pd))]
    models = np.stack([H1, H2]).astype(np.float32)
    for u8 in (False, True):
        ex = api.match_pairs_guided(devs, [(0, 1), (2, 3)], models, "homography", 30.0, EXACT, u8=u8)
        if not u8:
            assert (ex[0][:, 0] == at1).all() and (ex[1][:, 0] == at2).all()
        for flags in (AUTO, TENSOR):
            got = api.match_pairs_guided(devs, [(0, 1), (2, 3)], models, "homography", 30.0, flags, u8=u8)
            assert np.array_equal(got[0], ex[0]) and np.array_equal(got[1], ex[1]), (u8, flags)


_GROUP_SCRIPT = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from popsift_b200 import api
import test_guided as tg
z = np.load(sys.argv[2])
lib = api.load_library()
devs = [tg._dev_set(lib, z["s%d" % i], z["p%d" % i]) for i in range(int(z["n"]))]
out = api.match_pairs_guided(devs, [tuple(p) for p in z["pairs"]], z["models"], "fundamental", float(z["t"]), int(z["flags"]),
                             u8=bool(z["u8"]))
np.savez(sys.argv[3], *out)
"""


@pytest.mark.gpu
def test_small_workspace_cap_gives_same_rows(tmp_path):
    """POPSIFT_B200_MATCH_WS small enough for at least three groups (checked with the planner): same rows as one group"""
    lib = api.load_library()
    rng = np.random.default_rng(9)
    sizes = [3000, 2500, 3100, 900, 0, 2000]
    sets = [_unit(rng, n) for n in sizes]
    sets[1][:800] = sets[0][200:1000] + rng.normal(scale=0.01, size=(800, 128)).astype(np.float32)
    pts = [rng.uniform([0, 0], [W, H], (n, 2)).astype(np.float32) for n in sizes]
    pairs = [(i, j) for i in range(len(sets)) for j in range(len(sets)) if (i + j) % 2 == 0 or i == 5]
    models = _models(go.FUNDAMENTAL, rng, len(pairs))
    caps = {False: 8 << 20, True: 600_000}             # float (1 036-byte rows) and 8-bit (140-byte rows) workspaces
    for u8, rb in ((False, 1036), (True, 140)):
        assert int(_plan(sizes, pairs, rb, caps[u8]).split()[0].split("=")[1]) >= 3
    inp, res = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    devs = [_dev_set(lib, s, p) for s, p in zip(sets, pts)]
    for u8 in (False, True):
        ex = api.match_pairs_guided(devs, pairs, models, "fundamental", 75.0, EXACT, u8=u8)
        for flags in (AUTO, TENSOR):
            np.savez(inp, n=len(sets), pairs=np.array(pairs, np.int32), flags=flags, models=models, t=75.0, u8=u8,
                     **{"s%d" % i: s for i, s in enumerate(sets)}, **{"p%d" % i: p for i, p in enumerate(pts)})
            env = dict(os.environ, POPSIFT_B200_MATCH_WS=str(caps[u8]))
            subprocess.run([sys.executable, "-c", _GROUP_SCRIPT, ROOT, inp, res], env=env, check=True, timeout=600)
            z = np.load(res)
            whole = api.match_pairs_guided(devs, pairs, models, "fundamental", 75.0, flags, u8=u8)
            for k in range(len(pairs)):
                assert np.array_equal(z["arr_%d" % k], whole[k]), (u8, flags, pairs[k])
                assert np.array_equal(whole[k], ex[k]), (u8, flags, pairs[k])


def _extract_sets(images, w, h):
    cfg = api.Config()
    cfg.setNormalizationMultiplier(9)
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=w, max_height=h, slots=1)
    return ps, [ps.enqueue(w, h, im).getDev() for im in images]


def _true_err(corr, A):
    pr = corr[:, :2].astype(np.float64) @ A[:, :2].T + A[:, 2]
    return np.linalg.norm(pr - corr[:, 2:].astype(np.float64), axis=1)


# measured on synth.affine_set (t = 2 px, 1024 samples, seed 1), pairs (0, k), k = 1..5, on an H100 80GB HBM3: correct
# correspondences (true error < t), verified unguided inliers -> guided, per pair
#   float: 373 -> 383, 262 -> 269, 488 -> 496, 352 -> 395, 141 -> 319   (1 616 -> 1 862, x1.15); within 2t: 1 876 / 1 876
#   u8:    372 -> 386, 262 -> 270, 488 -> 497, 352 -> 395, 140 -> 318   (1 614 -> 1 866, x1.16); within 2t: 1 882 / 1 882
# asserted below with a margin (the extraction's feature order, and so the RANSAC samples, differ between processes)
GUIDED_MIN_GAIN = 1.08             # guided correct >= this x verified correct, summed over the pairs
GUIDED_MIN_WITHIN_2T = 0.97        # fraction of guided correspondences within 2t of the true map


@pytest.mark.gpu
@pytest.mark.parametrize("u8", [False, True])
def test_affine_set_end_to_end(u8):
    """verify_pairs(guided=True) on synth.affine_set against guided=False: the guided correspondences are what
    match_pairs_guided + match_correspondences give on the verified models, they are mostly correct, and there are at least
    as many correct ones as verified inliers"""
    data = affine_set()
    ps, sets = _extract_sets([im for im, _ in data], 800, 640)
    pairs = [(0, k) for k in range(1, 6)]
    kw = dict(model="homography", threshold=2.0, n_samples=1024, seed=1, u8=u8)
    plain = api.verify_pairs(sets, pairs, **kw)
    guided = api.verify_pairs(sets, pairs, guided=True, **kw)
    models = np.stack([g[0] for g in plain])
    rows = api.match_pairs_guided(sets, pairs, models, "homography", 2.0, u8=u8)
    corr, src = api.match_correspondences(sets, pairs, rows)
    matches = api.match_pairs_u8(sets, pairs) if u8 else api.match_pairs(sets, pairs)
    ucorr, usrc = api.match_correspondences(sets, pairs, matches)
    ok_plain = ok_guided = within = total = 0
    for (_, k), (G, cnt, vrows), (G2, n2, grows), c, s, uc, us in zip(pairs, plain, guided, corr, src, ucorr, usrc):
        assert np.array_equal(G, G2)
        assert n2 == len(c) and np.array_equal(grows, s)
        A = data[k][1]
        e = _true_err(c, A)
        ue = _true_err(uc[np.isin(us, vrows)], A)
        ok_plain += int((ue < 2.0).sum()); ok_guided += int((e < 2.0).sum())
        within += int((e < 4.0).sum()); total += len(e)
        print("u8=%d k=%d: verified %d (correct %d), guided %d (correct %d, within 2t %d)"
              % (u8, k, cnt, (ue < 2.0).sum(), n2, (e < 2.0).sum(), (e < 4.0).sum()))
    print("u8=%d total: verified correct %d, guided correct %d, guided within 2t %d / %d" % (u8, ok_plain, ok_guided, within, total))
    assert ok_guided >= GUIDED_MIN_GAIN * ok_plain, (ok_guided, ok_plain)
    assert within >= GUIDED_MIN_WITHIN_2T * total, (within, total)
    ps.uninit()


@pytest.mark.gpu
def test_argument_errors():
    lib = api.load_library()
    rng = np.random.default_rng(2)
    devs = [_dev_set(lib, _unit(rng, 40), rng.uniform(0, 500, (40, 2)).astype(np.float32)) for _ in range(2)]
    bufs = api._DevBuffers(lib)
    try:
        models = np.tile(np.eye(3, dtype=np.float32).ravel(), 2)
        d_models, d_out = bufs.upload(models), bufs.alloc(80 * 12)
        q = [api._to_u8_dev(lib, s.getDescriptors(), 40, 0) for s in devs]
        bufs.ptrs += q
        host_models = models.copy()

        def call(u8=False, sets=None, pairs=((0, 1), (1, 0)), d_m=d_models, model=0, t=4.0):
            sets = sets if sets is not None else (q if u8 else [s.getDescriptors() for s in devs])
            c_sets = (C.c_void_p * 2)(*sets)
            c_feat = (C.c_void_p * 2)(*[s.getFeatures() for s in devs])
            c_rev = (C.c_void_p * 2)(*[s.getReverseMap() for s in devs])
            c_n = (C.c_int32 * 2)(40, 40)
            c_pairs = (C.c_int32 * (2 * len(pairs)))(*[v for pq in pairs for v in pq])
            fn = lib.ps_match_u8_guided_batch if u8 else lib.ps_match_guided_batch
            return fn(0, 2, c_sets, c_feat, c_rev, c_n, len(pairs), c_pairs, d_m, model, t, d_out, 0)

        for u8 in (False, True):
            assert call(u8) == 0
            assert call(u8, model=2) == PS_ERR_ARG and call(u8, model=-1) == PS_ERR_ARG
            for t in (0.0, -1.0, float("nan"), float("inf")):
                assert call(u8, t=t) == PS_ERR_ARG, t
            assert call(u8, d_m=host_models.ctypes.data) == PS_ERR_ARG
            assert call(u8, pairs=((0, 2),)) == PS_ERR_ARG and call(u8, pairs=((-1, 0),)) == PS_ERR_ARG
            assert call(u8, pairs=()) == 0
        assert call(True, sets=[q[0] + 1, q[1]]) == PS_ERR_ARG                      # misaligned u8 set
        assert call(False, sets=[host_models.ctypes.data, devs[1].getDescriptors()]) == PS_ERR_ARG
    finally:
        bufs.free()
    with pytest.raises(api.PopSiftError):
        api.match_pairs_guided(devs, [(0, 1)], np.zeros((1, 3, 3)), "affine")
    with pytest.raises(api.PopSiftError):
        api.match_pairs_guided(devs, [(0, 1)], np.zeros((2, 3, 3)))


@pytest.mark.gpu
def test_empty_right_sets_need_no_models():
    """when no pair has both rows and a right descriptor, d_models is not needed (NULL here) and never read: every path,
    the CUDA-core EXACT one included, returns rows (0, 0, 0)"""
    lib = api.load_library()
    rng = np.random.default_rng(4)
    devs = [_dev_set(lib, _unit(rng, n), rng.uniform(0, 500, (n, 2)).astype(np.float32)) for n in (37, 0, 130)]
    pairs = [(0, 1), (2, 1), (1, 0), (1, 1)]
    rows = 37 + 130
    bufs = api._DevBuffers(lib)
    try:
        d_out = bufs.alloc(rows * 12)
        q = [api._to_u8_dev(lib, s.getDescriptors(), s.getDescriptorCount(), 0) for s in devs]
        bufs.ptrs += q
        c_feat = (C.c_void_p * 3)(*[s.getFeatures() for s in devs])
        c_rev = (C.c_void_p * 3)(*[s.getReverseMap() for s in devs])
        c_n = (C.c_int32 * 3)(37, 0, 130)
        c_pairs = (C.c_int32 * 8)(*[v for pq in pairs for v in pq])
        for u8 in (False, True):
            c_sets = (C.c_void_p * 3)(*(q if u8 else [s.getDescriptors() for s in devs]))
            fn = lib.ps_match_u8_guided_batch if u8 else lib.ps_match_guided_batch
            for model in (0, 1):
                for flags in (AUTO, EXACT, TENSOR):
                    fill = np.full((rows, 3), 7, np.int32)
                    assert lib.ps_host_to_dev(d_out, fill.ctypes.data, fill.nbytes) == 0
                    assert fn(0, 3, c_sets, c_feat, c_rev, c_n, 4, c_pairs, None, model, 4.0, d_out, flags) == 0, (u8, model, flags)
                    assert (bufs.download(d_out, (rows, 3), np.int32) == 0).all(), (u8, model, flags)
    finally:
        bufs.free()


@pytest.mark.gpu
def test_cpp_match_pairs_guided(tmp_path):
    """popsift::matchPairsGuided / matchPairsGuidedU8 equal the C ABI on three extracted frames (tests/cpp/guided_check.cpp)"""
    from popsift_b200 import build as B
    B.build()
    data = affine_set(640, 480)
    files = []
    for k in (0, 1, 2):
        f = tmp_path / ("f%d.raw" % k)
        data[k][0].tofile(f)
        files.append(str(f))
    out = subprocess.run([B.GUIDED_CHECK, "640", "480"] + files, capture_output=True, text=True, timeout=300)
    print(out.stdout, out.stderr)
    assert out.returncode == 0 and out.stdout.startswith("OK 7"), out.stdout + out.stderr
