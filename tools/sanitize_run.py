"""Small workloads through every kernel family, for compute-sanitizer (memcheck / racecheck):
    compute-sanitizer --tool memcheck python tools/sanitize_run.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from popsift_b200 import api
from popsift_b200.synth import make_frame

def run(w, h, seed, setup=None, frames=2, float_img=False):
    cfg = api.Config()
    if setup:
        setup(cfg)
    img = make_frame(w, h, seed)
    if float_img:
        img = img.astype(np.float32) / np.float32(256.0)
        ps = api.PopSift(cfg, imode=api.PopSift.FloatImages, max_width=w, max_height=h, slots=1)
    else:
        ps = api.PopSift(cfg, max_width=w, max_height=h, slots=1)
    n = None
    for _ in range(frames):
        f = ps.enqueue(w, h, img).get()
        n = (f.getFeatureCount(), f.getDescriptorCount())
    ps.uninit()
    return n

only = sys.argv[1] if len(sys.argv) > 1 else "all"
cases = {
    "default": lambda: run(641, 479, 1, frames=3),
    "small": lambda: run(70, 50, 2),
    "wide": lambda: run(1500, 200, 3),
    "nonint": lambda: run(300, 220, 4, lambda c: c.setDownsampling(-0.5)),
    "ds0": lambda: run(400, 300, 5, lambda c: c.setDownsampling(0)),
    "float": lambda: run(320, 240, 6, float_img=True),
    "filter": lambda: run(640, 480, 7, lambda c: (c.setFilterMaxExtrema(100), c.setFilterGridSize(3), c.setFilterSorting("up"))),
    "direct": lambda: run(320, 240, 8, lambda c: c.setScalingMode(0)),
    "vlfeat-direct": lambda: run(320, 240, 9, lambda c: c.setGaussMode("vlfeat-direct")),
    "relative": lambda: run(320, 240, 10, lambda c: c.setGaussMode("relative")),
    "fixed9": lambda: run(320, 240, 11, lambda c: c.setGaussMode("fixed9")),
    "fixed15": lambda: run(320, 240, 12, lambda c: c.setGaussMode("fixed15")),
    "igrid": lambda: run(320, 240, 13, lambda c: c.setDescMode("igrid")),
    "notile": lambda: run(320, 240, 14, lambda c: c.setDescMode("notile")),
    "opencv": lambda: run(320, 240, 15, lambda c: c.setMode("opencv")),
}
for name, fn in cases.items():
    if only in ("all", name):
        print(name, fn(), flush=True)
if only in ("all", "match"):
    rng = np.random.default_rng(0)
    def unit(n):
        d = rng.random((n, 128), dtype=np.float32)
        return d / np.linalg.norm(d, axis=1, keepdims=True)
    l, r = unit(1100), unit(2300)
    a = api.match_descriptors(l, r, api.FeaturesDev.MATCH_TENSOR)
    b = api.match_descriptors(l, r, api.FeaturesDev.MATCH_EXACT)
    print("match rows differing", int((a != b).any(1).sum()), flush=True)
if only in ("all", "match-batch"):
    # ragged sets, self pairs, an empty left and an empty right set; 1 x 20 left tiles take S > 1, and a 3 MB group cap
    # (set in the environment by the caller: POPSIFT_B200_MATCH_WS=3000000) makes several groups
    rng = np.random.default_rng(1)
    def unit(n):
        d = rng.random((n, 128), dtype=np.float32)
        return d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-12)
    sets = [unit(n) for n in (100, 2500, 129, 0, 1800, 700)]
    pairs = [(0, 1), (1, 0), (2, 2), (3, 1), (1, 3), (4, 5), (5, 4), (0, 4), (2, 1), (1, 1)]
    got = api.match_pairs(sets, pairs, api.FeaturesDev.MATCH_TENSOR)
    bad = sum(int((g != api.match_descriptors(sets[i], sets[j], api.FeaturesDev.MATCH_EXACT)).any(1).sum()) for g, (i, j) in zip(got, pairs))
    print("match-batch rows differing", bad, flush=True)
if only in ("all", "match-u8"):
    # the 8-bit matcher on ragged sets: self pairs, an empty left and an empty right set, a single-descriptor set, one
    # left tile against 20 right tiles (S > 1); with POPSIFT_B200_MATCH_WS=300000 in the environment, several groups
    rng = np.random.default_rng(2)
    sets = [rng.integers(0, 64, size=(n, 128)).astype(np.uint8) for n in (100, 2500, 129, 0, 1800, 700, 1)]
    pairs = [(0, 1), (1, 0), (2, 2), (3, 1), (1, 3), (4, 5), (5, 4), (0, 4), (2, 1), (1, 1), (6, 6), (0, 6)]
    got = api.match_pairs_u8(sets, pairs, api.FeaturesDev.MATCH_TENSOR)
    want = api.match_pairs_u8(sets, pairs, api.FeaturesDev.MATCH_EXACT)
    q = api.descriptors_to_u8(rng.normal(scale=100.0, size=(37, 128)).astype(np.float32))
    print("match-u8 rows differing", sum(int((g != w).any(1).sum()) for g, w in zip(got, want)), "quantised", q.shape, flush=True)
if only in ("all", "describe"):
    # caller-supplied keypoints (ps_describe_u8), both modes: a grid, random positions including the border and
    # out-of-range scales, rejected keypoints, and more keypoints than the slot holds (its buffers grow)
    img = make_frame(641, 479, 16)
    rng = np.random.default_rng(3)
    n = 9000
    kp = np.zeros(n, api.KEYPOINT_DTYPE)
    kp["x"], kp["y"] = rng.uniform(-2, 642, n), rng.uniform(-2, 480, n)
    kp["sigma"] = np.exp(rng.uniform(np.log(0.2), np.log(400.0), n))
    kp["ori"] = rng.uniform(-np.pi, np.pi, n)
    kp["octave"], kp["level"] = -1, -1
    kp["x"][:5] = np.nan
    kp["octave"][5:10], kp["level"][10:15] = 2, 1
    cfg = api.Config()
    cfg._c.max_extrema = 2000
    ps = api.PopSift(cfg, max_width=641, max_height=479, slots=1)
    for orient in (False, True):
        f = ps.describe(641, 479, img, kp, orientations=orient).get()
        print("describe", "orient" if orient else "given", (f.getFeatureCount(), f.getDescriptorCount()), flush=True)
    ps.uninit()
if only in ("all", "verify"):
    # geometric verification: the correspondence gather on real match rows (an empty set, self pairs), then RANSAC with both
    # models on those and on planted batches with empty, tiny and multi-tile pairs, with taps and refits
    frames = [make_frame(320, 240, 17), make_frame(320, 240, 17)[:, ::-1].copy(), np.zeros((240, 320), np.uint8)]
    cfg = api.Config()
    ps = api.PopSift(cfg, mode=api.Config.MatchingMode, max_width=320, max_height=240, slots=1)
    sets = [ps.enqueue(320, 240, im).getDev() for im in frames]
    pairs = [(0, 1), (1, 0), (0, 0), (2, 0), (0, 2)]
    for model in ("homography", "fundamental"):
        out = api.verify_pairs(sets, pairs, model=model, n_samples=100, threshold=3.0)
        print("verify pairs", model, [o[1] for o in out], flush=True)
    rng = np.random.default_rng(4)
    corrs = [rng.uniform(0, 640, size=(n, 4)).astype(np.float32) for n in (0, 3, 7, 8, 50, 2500, 5000)]
    for model in ("homography", "fundamental"):
        res, taps = api.verify_correspondences(corrs, model=model, n_samples=200, threshold=2.0, taps=True)
        print("verify", model, [r[1] for r in res], int((taps[0] >= 0).sum()), flush=True)
    ps.uninit()
if only in ("all", "retrieval"):
    # image retrieval: a codebook and VLAD vectors over sets with an empty one and one of several aggregation chunks, then
    # the similarity + top-m on a dim that ends in a partial k-step, n below one tile and m >= n
    rng = np.random.default_rng(5)
    sets = [rng.random((n, 128)).astype(np.float32) for n in (300, 0, 4500, 7)]
    cb = api.vlad_codebook(sets, k=24, iters=2, seed=1)
    v, a = api.vlad_encode(sets, cb, assign=True)
    print("vlad", v.shape, int(np.bincount(a, minlength=24).min()), flush=True)
    for n, dim, m in ((300, 260, 7), (20, 36, 30), (1, 4, 1)):
        nbr, sc = api.retrieve(rng.normal(size=(n, dim)).astype(np.float32), m)
        print("retrieve", n, dim, m, int(nbr[0, 0]), flush=True)
if only in ("all", "tracks"):
    # feature tracks: the edge entry on a ragged graph (empty sets, self-loops, duplicates, forks) over more than one scan
    # block and radix tile, then the chain entry on real match rows with a self pair, verified and guided
    rng = np.random.default_rng(6)
    n_feat = [0, 3000, 2500, 0, 4000, 1]
    e = rng.integers(0, 9501, size=(6000, 2))
    e[:50, 1] = e[:50, 0]
    edges = np.c_[np.searchsorted(np.cumsum([0] + n_feat), e[:, 0], side="right") - 1, e[:, 0], np.zeros(len(e), int), e[:, 1]]
    off = np.cumsum([0] + n_feat)
    edges[:, 1] -= off[edges[:, 0]]
    edges[:, 2] = np.searchsorted(off, e[:, 1], side="right") - 1
    edges[:, 3] = e[:, 1] - off[edges[:, 2]]
    t = api.build_tracks(n_feat, np.concatenate([edges, edges[:100]]), min_length=3)
    print("tracks edges", len(t.start) - 1, t.n_conflicting, t.n_short, flush=True)
    frames = [make_frame(320, 240, 18), make_frame(320, 240, 18)[:, ::-1].copy(), make_frame(320, 240, 19)]
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=320, max_height=240, slots=1)
    sets = [ps.enqueue(320, 240, im).getDev() for im in frames]
    for guided in (False, True):
        t = api.tracks(sets, [(0, 1), (1, 2), (0, 2), (2, 2)], guided=guided, n_samples=100)
        print("tracks chain", "guided" if guided else "verified", len(t.start) - 1, t.n_conflicting, flush=True)
    ps.uninit()
if only in ("all", "pose"):
    # calibrated two-view geometry: empty, tiny (< 5) and multi-tile pairs with taps and points, then the device chain on
    # real match rows with a self pair
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import pose_oracle as po
    rng = np.random.default_rng(7)
    sc = [po.planted_pose(rng, n, 0.6) for n in (0, 3, 5, 40, 2500)]
    res, taps = api.relative_pose_correspondences([s[0] for s in sc], [s[1] for s in sc], threshold=2.0, n_samples=150,
                                                  points=True, taps=True)
    print("pose", [r.n_inliers for r in res], int((taps[0] >= 0).sum()), flush=True)
    frames = [make_frame(320, 240, 18), make_frame(320, 240, 18)[:, ::-1].copy()]
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=320, max_height=240, slots=1)
    sets = [ps.enqueue(320, 240, im).getDev() for im in frames]
    out = api.relative_poses(sets, [(0, 1), (1, 1)], [(300, 300, 160, 120)] * 2, n_samples=100, points=True)
    print("pose chain", [o[0].n_inliers for o in out], flush=True)
    ps.uninit()
if only in ("all", "triangulate"):
    # multi-view triangulation: tracks of length 1 (too few), 2, across the exhaustive / sampled boundary and of 200 members,
    # an empty set, outliers; then the device chain on real match rows
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import triangulate_oracle as tro
    rng = np.random.default_rng(8)
    sc = tro.planted_scene(rng, 220, [1, 2, 2, 3, 9, 10, 11, 40, 200] * 3, noise=0.5, outliers=0.2)
    off =np.cumsum([0] + [len(f) for f in sc["feats"]])
    sets_of = np.searchsorted(off, sc["members"], side="right") - 1
    tr = api.Tracks(sc["start"], sets_of, sc["members"] - off[sets_of], None, 0, 0, 0)
    feats = []
    for f in sc["feats"]:
        r = np.zeros(len(f), api.FEATURE_DTYPE)
        r["x"], r["y"] = f[:, 0], f[:, 1]
        feats.append(r)
    p = api.triangulate(feats, tr, sc["cams"], sc["poses"], max_error=3.0, n_samples=45, seed=1)
    print("triangulate", p.counts, flush=True)
    frames = [make_frame(320, 240, 18), make_frame(320, 240, 18)[:, ::-1].copy(), make_frame(320, 240, 19)]
    ps = api.PopSift(api.Config(), mode=api.Config.MatchingMode, max_width=320, max_height=240, slots=1)
    sets = [ps.enqueue(320, 240, im).getDev() for im in frames]
    poses = [(np.eye(3), np.array([0.1 * k, 0.0, 0.0])) for k in range(3)]
    t, p = api.triangulated_tracks(sets, [(0, 1), (1, 2), (0, 2)], [(300, 300, 160, 120)] * 3, poses, verify=dict(n_samples=100))
    print("triangulate chain", len(t.start) - 1, p.counts, flush=True)
    ps.uninit()
if only in ("all", "bundle"):
    # bundle adjustment: each loss on a planted scene with a fixed set, a held scale component, a set without features,
    # masked members and non-OK tracks; a non-finite start; structure only
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import bundle_oracle as bo
    rng = np.random.default_rng(9)
    sc = bo.planted(rng, 12, [2, 3, 5, 9, 12] * 20, noise=0.5, outliers=0.1)
    sc["feats"] = list(sc["feats"]) + [np.zeros((0, 2), np.float32)]
    sc["cams"] = np.concatenate([sc["cams"], sc["cams"][:1]])
    sc["poses"] = list(sc["poses"]) + [sc["poses"][0]]
    off = np.cumsum([0] + [len(f) for f in sc["feats"]])
    sets_of = np.searchsorted(off, sc["members"], side="right") - 1
    tr = api.Tracks(sc["start"], sets_of, sc["members"] - off[sets_of], None, 0, 0, 0)
    feats = []
    for f in sc["feats"]:
        r = np.zeros(len(f), api.FEATURE_DTYPE)
        r["x"], r["y"] = f[:, 0], f[:, 1]
        feats.append(r)
    status = sc["status"].copy()
    status[::7] = 3
    mask = sc["mask"].copy()
    mask[::5] = 0
    tp = api.TrackPoints(sc["X0"], np.zeros(100, np.float32), np.zeros(100, np.float32), np.diff(sc["start"]).astype(np.int32), status, mask,
                         None, None)
    fixed = [True] + [False] * 12
    for loss in ("squared", "huber", "cauchy"):
        _, _, rep = api.bundle_adjust(feats, tr, tp, sc["cams"], sc["poses"], fixed, loss=loss, max_iters=5, scale_set=1, scale_axis=2)
        print("bundle", loss, rep, flush=True)
    _, _, rep = api.bundle_adjust(feats, tr, tp, sc["cams"], sc["poses"], [True] * 13, max_iters=3)
    print("bundle structure only", rep, flush=True)
    R, t = sc["poses"][4]
    bad = list(sc["poses"])
    bad[4] = (np.diag([-1.0, 1.0, -1.0]) @ R, np.diag([-1.0, 1.0, -1.0]) @ t)
    _, _, rep = api.bundle_adjust(feats, tr, tp, sc["cams"], bad, fixed)
    print("bundle non-finite start", rep, flush=True)
if only in ("all", "scale"):
    # bundle adjustment, positioning and rotation averaging at the exact work-split boundaries (tests/scale_shapes.py):
    # S = 257 sets, set observation counts of 128 and 129 with empty sets between, T = 257 tracks, M = 4097 members
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import scale_shapes as ss
    for name in ("sets_257", "counts", "tracks_257", "members_4097"):
        sc = ss.SCENES[name]()
        off = np.cumsum([0] + [len(f) for f in sc["feats"]])
        sets_of = np.searchsorted(off, sc["members"], side="right") - 1
        tr = api.Tracks(sc["start"], sets_of, sc["members"] - off[sets_of], None, 0, 0, 0)
        feats = []
        for f in sc["feats"]:
            r = np.zeros(len(f), api.FEATURE_DTYPE)
            r["x"], r["y"] = f[:, 0], f[:, 1]
            feats.append(r)
        T = len(sc["start"]) - 1
        tp = api.TrackPoints(sc["X0"], np.zeros(T, np.float32), np.zeros(T, np.float32), np.diff(sc["start"]).astype(np.int32), sc["status"],
                             sc["mask"], None, None)
        _, _, rep = api.bundle_adjust(feats, tr, tp, sc["cams"], sc["poses"], sc["fixed"].astype(bool), loss="huber", loss_scale=2.0,
                                      max_iters=2, cg_max_iters=50, scale_set=int(np.flatnonzero(sc["fixed"] == 0)[0]), scale_axis=2)
        print("scale bundle", name, rep, flush=True)
        out = api.global_positioning(feats, tr, sc["cams"], sc["R"], np.ones(len(feats), bool), max_iters=2, cg_max_iters=50)
        print("scale positioning", name, out[-1], flush=True)
    Rt, pairs, Rp, nf, _ = ss.GRAPHS["sets_257_hub"]()
    tv = np.zeros(len(pairs), api.TWO_VIEW_DTYPE)
    tv["R"], tv["n_front"], tv["n_inliers"] = np.asarray(Rp, np.float32), nf, nf
    out = api.rotation_averaging(257, pairs, tv, max_iters=2, cg_max_iters=50, min_inliers=0)
    print("scale rotations", out[-1], flush=True)
if only in ("all", "mesh"):
    # integration over more views than one shared-memory chunk with masks, partial blocks on every axis; extraction of
    # the result, of an empty volume, and the count-only call
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import test_mesh as tm
    imgs, cams, poses, depths, masks = tm._random_views(1, 70, w=40, h=30, dist=1.2)
    vol = api.TsdfVolume((-0.6, -0.5, -0.55), 0.02, (61, 50, 55))
    print("mesh integrate", vol.integrate(imgs, cams, poses, depths, masks, trunc=0.05, min_consistent=1), flush=True)
    print("mesh extract", vol.mesh().report, flush=True)
    vol.clear()
    print("mesh empty", vol.mesh().report, flush=True)
    vol.free()
