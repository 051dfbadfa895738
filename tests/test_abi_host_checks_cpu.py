"""The host-side argument checks of the 27 stateless entry points, ps_match .. ps_mesh_texture, observed without a GPU.

Every call passes device = -1. cudaSetDevice(-1) fails on every machine, so a call that gets past its host checks stops
at the device switch with PS_ERR_CUDA, and nothing reaches a GPU. Device-pointer arguments are arbitrary non-zero
integers: nothing reads them before the switch. For each entry point:
- a well-formed call reaches the switch (PS_ERR_CUDA);
- each argument refused before the switch gives PS_ERR_ARG;
- the checks and empty-work returns placed after the switch give PS_ERR_CUDA, which pins where they sit;
- the early returns before the switch give PS_OK with their documented host outputs.
Host outputs (reports, counts, poses, flags, info) start filled with a sentinel and stay untouched by every call that does
not return PS_OK, and ps_last_error(NULL) keeps its text unless the check has a message of its own.
The checks made after the switch (pointer location, alignment, sets, depth CSR, volumes, overlaps) need a device; the
GPU refusal tests cover them.
"""
import ctypes as C

import pytest

from popsift_b200 import api

OK, ARG, CUDA = 0, -1, -2
NAN, INF = float("nan"), float("inf")
DEV = 0x7F0000100000            # stands for device memory; never dereferenced before cudaSetDevice
SENTINEL = 0xA5
PRESET = b"ps_create: bad argument"   # what ps_create(0, NULL, ...) leaves in ps_last_error(NULL)
U8 = C.c_uint8


def _ints(*v, t=C.c_int32):
    return (t * len(v))(*v)


def _ptrs(n):
    return (C.c_void_p * n)(*([DEV] * n))


def _cams(n):
    return (api.PsCamera * n)(*[api.PsCamera(500.0, 510.0, 320.0, 240.0) for _ in range(n)])


def _rigids(n):
    return (api.PsRigid * n)(*[api.PsRigid((C.c_double * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1), (C.c_double * 3)(0.1 * i, 0, 1))
                               for i in range(n)])


def _images(n, w=64, h=48):
    return (api.PsImage * n)(*[api.PsImage(DEV, w, w, h) for _ in range(n)])


def _volume():
    return api.PsVolume((C.c_double * 3)(0, 0, 0), 0.01, 16, 16, 16, 0, DEV, DEV + (1 << 20), DEV + (2 << 20))


# Each builder returns a call's arguments in C order; OUTS names the host outputs that get the sentinel.
BUILD = {
    "ps_match": lambda: dict(device=-1, d_left=DEV, n_left=4, d_right=DEV, n_right=4, d_out=DEV, flags=0),
    "ps_match_batch": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), n_desc=_ints(3, 4), n_pairs=1, pairs=_ints(0, 1),
                                   d_out=DEV, flags=0),
    "ps_descriptors_to_u8": lambda: dict(device=-1, d_in=DEV, n=4, d_out=DEV),
    "ps_match_u8_batch": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), n_desc=_ints(3, 4), n_pairs=1, pairs=_ints(0, 1),
                                      d_out=DEV, flags=0),
    "ps_match_correspondences": lambda: dict(device=-1, n_sets=2, d_feat=_ptrs(2), d_rev=_ptrs(2), n_desc=_ints(3, 4), n_pairs=1,
                                             pairs=_ints(0, 1), d_match=DEV, d_corr=DEV, d_src=DEV, n_corr=_ints(0)),
    "ps_verify_batch": lambda: dict(device=-1, n_pairs=2, d_corr=DEV, corr_start=_ints(0, 8), n_corr=_ints(8, 8),
                                    prm=api.PsVerifyParams(1, 64, 1.0, 1, 7), d_models=DEV, d_n_inliers=DEV, d_inlier_mask=DEV,
                                    taps=None),
    "ps_relative_pose_batch": lambda: dict(device=-1, n_pairs=2, d_corr=DEV, corr_start=_ints(0, 8), n_corr=_ints(8, 8),
                                           cams=_cams(4), prm=api.PsPoseParams(64, 1.0, 1, 0, 7), d_out=DEV, d_inlier_mask=DEV,
                                           d_points=None, taps=None),
    "ps_match_guided_batch": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), d_feat=_ptrs(2), d_rev=_ptrs(2), n_desc=_ints(3, 4),
                                          n_pairs=1, pairs=_ints(0, 1), d_models=DEV, model=0, threshold=2.0, d_out=DEV, flags=0),
    "ps_match_u8_guided_batch": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), d_feat=_ptrs(2), d_rev=_ptrs(2),
                                             n_desc=_ints(3, 4), n_pairs=1, pairs=_ints(0, 1), d_models=DEV, model=1, threshold=2.0,
                                             d_out=DEV, flags=0),
    "ps_vlad_train": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), n_desc=_ints(30, 40), k=8, iters=5, seed=1,
                                  d_centroids=DEV, flags=0),
    "ps_vlad_encode": lambda: dict(device=-1, n_sets=2, d_sets=_ptrs(2), n_desc=_ints(30, 40), k=8, d_centroids=DEV, d_vlad=DEV,
                                   d_assign=None, flags=0),
    "ps_retrieve_pairs": lambda: dict(device=-1, n=10, d_vec=DEV, dim=64, m=4, d_nbr=DEV, d_score=DEV),
    "ps_tracks_from_edges": lambda: dict(device=-1, n_sets=2, n_feat=_ints(5, 6), n_edges=3, d_edges=DEV, min_length=2,
                                         d_track_of=DEV, d_track_start=DEV, d_members=DEV, counts=api.PsTrackCounts()),
    "ps_tracks_from_matches": lambda: dict(device=-1, n_sets=2, n_feat=_ints(5, 6), d_rev=_ptrs(2), n_desc=_ints(3, 4), n_pairs=1,
                                           pairs=_ints(0, 1), d_match=DEV, d_src=DEV, n_corr=_ints(2), d_inlier_mask=None,
                                           min_length=2, d_track_of=DEV, d_track_start=DEV, d_members=DEV,
                                           counts=api.PsTrackCounts()),
    "ps_triangulate_tracks": lambda: dict(device=-1, n_sets=2, n_feat=_ints(5, 6), d_feat=_ptrs(2), cams=_cams(2), poses=_rigids(2),
                                          n_tracks=3, d_track_start=DEV, d_members=DEV, n_members=6,
                                          prm=api.PsTriangulateParams(2.0, 1.0, 2, 32, 5, 0, 1), d_points=DEV, d_obs_mask=DEV,
                                          d_obs_error=None, counts=api.PsTriangulateCounts()),
    "ps_bundle_adjust": lambda: dict(device=-1, n_sets=2, n_feat=_ints(5, 6), d_feat=_ptrs(2), cams=_cams(2), poses_in=_rigids(2),
                                     n_tracks=3, d_track_start=DEV, d_members=DEV, n_members=6, d_points=DEV, d_obs_mask=DEV,
                                     fixed=_ints(1, 0, t=U8), prm=api.PsBundleParams(1, 20, 50, -1, 0, 0, 1.0, 1e-6, 0.1, 1e-4),
                                     poses_out=(api.PsRigid * 2)(), d_obs_error=None, report=api.PsBundleReport()),
    "ps_rotation_averaging": lambda: dict(device=-1, n_sets=3, n_pairs=2, pairs=_ints(0, 1, 1, 2), d_two_view=DEV,
                                          prm=api.PsRotationParams(1, 20, 50, 10, 0.1, 1e-8, 0.1), R_out=(C.c_double * 27)(),
                                          registered=(U8 * 3)(), pair_error=(C.c_float * 2)(), report=api.PsRotationReport()),
    "ps_global_positioning": lambda: dict(device=-1, n_sets=2, n_feat=_ints(5, 6), d_feat=_ptrs(2), cams=_cams(2),
                                          R=(C.c_double * 18)(1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 1, 0, -1, 0, 0, 0, 0, 1),
                                          registered=_ints(1, 1, t=U8), n_tracks=3, d_track_start=DEV, d_members=DEV, n_members=6,
                                          prm=api.PsPositionParams(1, 20, 50, 0, 1.0, 1e-6, 0.1), poses_out=(api.PsRigid * 2)(),
                                          positioned=(U8 * 2)(), d_X=None, report=api.PsPositionReport()),
    "ps_view_graph_filter": lambda: dict(device=-1, n_sets=3, n_pairs=3, pairs=_ints(0, 1, 1, 2, 0, 2), d_two_view=DEV,
                                         prm=api.PsViewGraphParams(10, 1, 1, 0, 0.05, 0.5), keep=(U8 * 3)(),
                                         stats=(api.PsCycleStats * 3)(), d_kept=None, report=api.PsViewGraphReport()),
    "ps_two_view_config_batch": lambda: dict(device=-1, n_pairs=2, d_corr=DEV, corr_start=_ints(0, 8), n_corr=_ints(8, 8),
                                             cams=_cams(4), d_essential=DEV, d_essential_mask=DEV, d_f_inliers=DEV, d_homography=DEV,
                                             d_h_mask=DEV, prm=api.PsTwoViewConfigParams(15, 1.0, 0.5, 0.8, 0.5), d_out=DEV,
                                             d_out_mask=DEV, d_points=None, info=(api.PsTwoViewInfo * 2)()),
    "ps_depth_maps": lambda: dict(device=-1, n_sets=3, images=_images(3), cams=_cams(3), poses=_rigids(3), n_refs=1, refs=_ints(0),
                                  ranges=(C.c_float * 2)(1.0, 10.0), src_start=_ints(0, 2), src_sets=_ints(1, 2),
                                  prm=api.PsDepthParams(64, 3, 4, 1, 0.5, 0.0), d_depth=_ptrs(1), d_cost=_ptrs(1), d_n_src=_ptrs(1),
                                  report=api.PsDepthReport()),
    "ps_depth_filter": lambda: dict(device=-1, n_sets=3, images=_images(3), cams=_cams(3), poses=_rigids(3), n_refs=1, refs=_ints(0),
                                    src_start=_ints(0, 2), src_sets=_ints(1, 2), d_depth=_ptrs(1),
                                    prm=api.PsDepthFilterParams(1.0, 0.01, 1, 0), d_n_consistent=_ptrs(1), d_points=DEV,
                                    report=api.PsDepthFilterReport()),
    "ps_volume_clear": lambda: dict(device=-1, vol=_volume()),
    "ps_tsdf_integrate": lambda: dict(device=-1, n_views=2, images=_images(2), cams=_cams(2), poses=_rigids(2), d_depth=_ptrs(2),
                                      d_n_consistent=None, prm=api.PsTsdfParams(0.05, 0), vol=_volume(), report=api.PsTsdfReport()),
    "ps_tsdf_mesh": lambda: dict(device=-1, vol=_volume(), prm=api.PsMeshParams(1.0, 0), max_vertices=100, max_triangles=200,
                                 d_vertices=DEV, d_triangles=DEV, report=api.PsMeshReport()),
    "ps_mesh_render": lambda: dict(device=-1, n_views=2, sizes=_ints(64, 48, 64, 48), cams=_cams(2), poses=_rigids(2), d_vertices=DEV,
                                   n_vertices=4, d_triangles=DEV, n_triangles=2, prm=api.PsRenderParams(0.01, 0), d_depth=_ptrs(2),
                                   d_tri=_ptrs(2), report=api.PsRenderReport()),
    "ps_mesh_texture": lambda: dict(device=-1, n_views=2, images=_images(2), cams=_cams(2), poses=_rigids(2), d_depth=_ptrs(2),
                                    d_vertices=DEV, n_vertices=4, d_triangles=DEV, n_triangles=2,
                                    prm=api.PsTextureParams(8, 16, 0.01, 0.1, 0.01, 0), d_atlas=DEV, d_view=DEV,
                                    report=api.PsTextureReport()),
}
OUTS = {"ps_match_correspondences": ["n_corr"], "ps_tracks_from_edges": ["counts"], "ps_tracks_from_matches": ["counts"],
        "ps_triangulate_tracks": ["counts"], "ps_bundle_adjust": ["poses_out", "report"],
        "ps_rotation_averaging": ["R_out", "registered", "pair_error", "report"],
        "ps_global_positioning": ["poses_out", "positioned", "report"], "ps_view_graph_filter": ["keep", "stats", "report"],
        "ps_two_view_config_batch": ["info"], "ps_depth_maps": ["report"], "ps_depth_filter": ["report"],
        "ps_tsdf_integrate": ["report"], "ps_tsdf_mesh": ["report"], "ps_mesh_render": ["report"], "ps_mesh_texture": ["report"]}


def at(path, value):
    """a mutation: the argument, struct field or array element at a dotted path ("prm.n_samples", "cams.3.fx") = value"""
    def mutate(a):
        *head, last = path.split(".")
        obj = a
        for k in head:
            obj = obj[int(k)] if k.isdigit() else obj[k] if isinstance(obj, dict) else getattr(obj, k)
        if isinstance(obj, dict):
            obj[last] = value
        elif last.isdigit():
            obj[int(last)] = value
        else:
            setattr(obj, last, value)
    return mutate


def camera_bad(key, i):
    return [("%s %d %s" % (key, i, f), [at("%s.%d.%s" % (key, i, f), v)])
            for f, v in (("fx", NAN), ("fx", 0.0), ("fx", INF), ("fy", -1.0), ("fy", NAN), ("cx", INF), ("cy", NAN))]


def rotation_bad(key, base):
    """a rotation at R[base .. base+9) that is not finite, not orthonormal or a reflection"""
    return [("%s %d nan" % (key, base), [at("%s.%d" % (key, base + 4), NAN)]),
            ("%s %d not orthonormal" % (key, base), [at("%s.%d" % (key, base), 1.001)]),
            ("%s %d reflection" % (key, base), [at("%s.%d" % (key, base + 8), -1.0)])]


def rigid_bad(key, i):
    return [(label, muts) for label, muts in rotation_bad("%s.%d.R" % (key, i), 0)] + \
           [("%s %d t inf" % (key, i), [at("%s.%d.t.2" % (key, i), INF)])]


def image_bad(key, i, min_side):
    return [("%s %d %s" % (key, i, f), [at("%s.%d.%s" % (key, i, f), v)])
            for f, v in (("width", min_side - 1), ("height", min_side - 1), ("width", 65536), ("height", 65536), ("pitch", 63))]


def csr_bad():
    return [("corr_start null", [at("corr_start", None)]), ("n_corr null", [at("n_corr", None)]),
            ("corr_start negative", [at("corr_start.1", -1)]), ("n_corr negative", [at("n_corr.1", -1)])]


def ransac_bad():
    return [("prm %s %r" % (f, v), [at("prm." + f, v)])
            for f, v in (("n_samples", 0), ("n_samples", 65537), ("threshold", NAN), ("threshold", INF), ("threshold", 0.0),
                         ("threshold", -1.0), ("refine", -1), ("refine", 2))]


def solver_bad():
    return [("prm %s %r" % (f, v), [at("prm." + f, v)])
            for f, v in (("loss", -1), ("loss", 3), ("max_iters", -1), ("max_iters", 10001), ("cg_max_iters", 0),
                         ("cg_max_iters", 10001), ("loss_scale", NAN), ("loss_scale", INF), ("loss_scale", 0.0),
                         ("cg_tol", -0.1), ("cg_tol", 1.0), ("cg_tol", NAN))]


def fields(expect, specs):
    return [(expect, "prm %s %r" % (f, v), [at("prm." + f, v)]) for f, v in specs]


def args(expect, specs):
    """one case per (argument path, value)"""
    return [(expect, "%s %r" % (k, v), [at(k, v)]) for k, v in specs]


def refused(cases):
    return [(ARG, label, muts) for label, muts in cases]


MATCH_SETS = args(ARG, [("n_sets", -1), ("n_pairs", -1), ("d_sets", None), ("n_desc", None), ("pairs", None)]) + \
    args(CUDA, [("n_sets", 0), ("n_pairs", 0), ("pairs.1", 2), ("pairs.0", -1), ("n_desc.0", -1), ("d_sets.1", None),
                ("d_out", None)]) + [(CUDA, "no sets, no pairs", [at("n_sets", 0), at("n_pairs", 0)])]
GUIDED = args(ARG, [("n_sets", -1), ("n_pairs", -1), ("d_sets", None), ("d_feat", None), ("d_rev", None), ("n_desc", None),
                    ("pairs", None), ("model", 2), ("model", -1), ("threshold", NAN), ("threshold", 0.0), ("threshold", -1.0),
                    ("threshold", INF)]) + \
    args(CUDA, [("n_pairs", 0), ("pairs.1", 2), ("d_models", None), ("d_out", None), ("n_desc.1", -1)])
BUNDLE_SETS = args(ARG, [("n_sets", -1), ("n_tracks", -1), ("n_members", -1), ("n_feat", None), ("d_feat", None), ("cams", None)])

CASES = {
    "ps_match": args(ARG, [("n_left", -1), ("n_right", -1), ("d_left", None), ("d_out", None), ("d_right", None)]) +
    args(CUDA, [("n_right", 0)]),
    "ps_match_batch": MATCH_SETS,
    "ps_descriptors_to_u8": args(ARG, [("n", -1), ("d_in", None), ("d_out", None)]),
    "ps_match_u8_batch": MATCH_SETS,
    "ps_match_correspondences":
        args(ARG, [("n_sets", -1), ("n_pairs", -1), ("d_feat", None), ("d_rev", None), ("n_desc", None), ("pairs", None),
                   ("n_corr", None)]) +
        args(CUDA, [("n_pairs", 0), ("pairs.1", 2), ("n_desc.0", 0), ("d_match", None), ("d_feat.0", None)]),
    "ps_verify_batch":
        args(ARG, [("n_pairs", -1), ("prm", None), ("prm.model", 2), ("prm.model", -1)]) + refused(ransac_bad() + csr_bad()) +
        args(CUDA, [("prm.n_samples", 1), ("prm.n_samples", 65536), ("prm.refine", 0), ("prm.model", 0), ("d_corr", DEV + 4),
                    ("d_models", None), ("n_corr.0", 0)]) + [(CUDA, "no rows", [at("n_corr.0", 0), at("n_corr.1", 0)])],
    "ps_relative_pose_batch":
        args(ARG, [("n_pairs", -1), ("prm", None), ("cams", None)]) + refused(ransac_bad() + csr_bad()) +
        refused(camera_bad("cams", 0) + camera_bad("cams", 3)) +
        args(CUDA, [("prm.n_samples", 65536), ("d_corr", DEV + 4), ("d_out", None), ("cams.3.cx", -5.0)]),
    "ps_match_guided_batch": GUIDED,
    "ps_match_u8_guided_batch": GUIDED,
    "ps_vlad_train": args(ARG, [("n_sets", -1), ("k", 0), ("k", 1025), ("iters", -1), ("iters", 1001)]) +
    args(CUDA, [("n_sets", 0), ("k", 1024), ("iters", 0), ("iters", 1000), ("n_desc.0", -1), ("d_centroids", None)]),
    "ps_vlad_encode": args(ARG, [("n_sets", -1), ("k", 0), ("k", 1025)]) +
    args(CUDA, [("n_sets", 0), ("n_desc", None), ("d_vlad", None)]),
    "ps_retrieve_pairs": args(ARG, [("n", -1), ("dim", 0), ("dim", -4), ("dim", 66), ("m", 0), ("m", 129)]) +
    [(ARG, "n m >= 2^31", [at("n", 1 << 24), at("m", 128)])] +
    args(CUDA, [("m", 128), ("d_vec", DEV + 4), ("d_nbr", None)]) + [(CUDA, "n m < 2^31", [at("n", (1 << 24) - 1), at("m", 128)])],
    "ps_tracks_from_edges": args(ARG, [("n_edges", -1), ("d_edges", None)]) +
    args(CUDA, [("n_edges", 0), ("min_length", 1), ("counts", None), ("n_feat", None), ("n_feat.0", -1), ("n_sets", -1),
                ("d_track_start", None)]),
    "ps_tracks_from_matches":
        args(ARG, [("n_sets", -1), ("n_pairs", -1), ("d_rev", None), ("n_desc", None), ("pairs", None), ("n_corr", None)]) +
        args(CUDA, [("n_pairs", 0), ("min_length", 1), ("counts", None), ("pairs.1", 2), ("n_corr.0", 4), ("n_corr.0", -1)]),
    "ps_triangulate_tracks":
        args(ARG, [("prm", None), ("counts", None), ("poses", None)]) + BUNDLE_SETS +
        refused(camera_bad("cams", 1) + rigid_bad("poses", 0) + rigid_bad("poses", 1)) +
        fields(ARG, [("max_error", NAN), ("max_error", 0.0), ("max_error", INF), ("min_angle", -1.0), ("min_angle", 90.0),
                     ("min_angle", NAN), ("min_views", 1), ("n_samples", 0), ("n_samples", 65537), ("refine_iters", -1),
                     ("refine_iters", 33)]) +
        fields(CUDA, [("min_angle", 0.0), ("n_samples", 65536), ("refine_iters", 32)]) +
        args(CUDA, [("n_feat.0", -1), ("d_points", None), ("n_members", 0)]),
    "ps_bundle_adjust":
        args(ARG, [("prm", None), ("report", None), ("poses_out", None), ("fixed", None), ("poses_in", None),
                   ("fixed.0", 2), ("fixed.0", 0)]) + BUNDLE_SETS +
        refused(camera_bad("cams", 1) + rigid_bad("poses_in", 1) + solver_bad()) +
        fields(ARG, [("function_tol", NAN), ("function_tol", -1.0), ("initial_lambda", 0.0), ("initial_lambda", 1e33),
                     ("initial_lambda", NAN), ("scale_set", -2), ("scale_set", 2), ("scale_axis", -1), ("scale_axis", 3)]) +
        fields(CUDA, [("loss", 0), ("loss", 2), ("max_iters", 0), ("cg_max_iters", 10000), ("cg_tol", 0.0),
                      ("initial_lambda", 1e32), ("scale_set", 1), ("scale_axis", 2)]) +
        args(CUDA, [("n_feat.0", -1), ("d_points", None), ("fixed.1", 1)]),
    "ps_rotation_averaging":
        args(ARG, [("n_sets", -1), ("n_pairs", -1), ("prm", None), ("R_out", None), ("registered", None), ("report", None),
                   ("pairs", None), ("pairs.3", 3), ("pairs.0", -1)]) + refused(solver_bad()) +
        fields(ARG, [("min_inliers", -1), ("step_tol", NAN), ("step_tol", -1.0), ("step_tol", INF)]) +
        args(CUDA, [("n_pairs", 0), ("pair_error", None), ("d_two_view", None), ("prm.loss", 2)]) +
        [(CUDA, "no sets, no pairs", [at("n_sets", 0), at("n_pairs", 0)])],
    "ps_global_positioning":
        args(ARG, [("prm", None), ("report", None), ("n_sets", -1), ("n_tracks", -1), ("n_members", -1), ("n_feat", None),
                   ("d_feat", None), ("cams", None), ("R", None), ("registered", None), ("poses_out", None),
                   ("positioned", None), ("registered.1", 2)]) +
        refused(camera_bad("cams", 1) + rotation_bad("R", 0) + rotation_bad("R", 9) + solver_bad()) +
        fields(ARG, [("function_tol", NAN), ("function_tol", -1.0)]) +
        args(CUDA, [("registered.1", 0), ("n_feat.0", -1), ("d_track_start", None), ("n_members", 0)]),
    "ps_view_graph_filter":
        args(ARG, [("n_sets", -1), ("n_pairs", -1), ("prm", None), ("keep", None), ("report", None), ("pairs", None),
                   ("pairs.5", 3), ("pairs.2", -1)]) +
        fields(ARG, [("min_inliers", -1), ("min_consistent", -1), ("keep_untested", -1), ("keep_untested", 2),
                     ("max_cycle_error", NAN), ("max_cycle_error", -1.0), ("max_cycle_error", INF), ("min_fraction", -0.1),
                     ("min_fraction", 1.1), ("min_fraction", NAN)]) +
        fields(CUDA, [("keep_untested", 0), ("max_cycle_error", 0.0), ("min_fraction", 1.0)]) +
        args(CUDA, [("n_pairs", 0), ("stats", None), ("d_two_view", None)]) +
        [(CUDA, "no sets, no pairs", [at("n_sets", 0), at("n_pairs", 0)])],
    "ps_two_view_config_batch":
        args(ARG, [("n_pairs", -1), ("prm", None), ("info", None), ("cams", None)]) + refused(csr_bad() + camera_bad("cams", 3)) +
        fields(ARG, [("min_inliers", -1), ("threshold", NAN), ("threshold", 0.0), ("threshold", INF)] +
               [(f, v) for f in ("min_ef_ratio", "max_h_ratio", "min_rotation_ratio") for v in (-0.1, 1.1, NAN)]) +
        fields(CUDA, [("min_ef_ratio", 0.0), ("max_h_ratio", 1.0)]) +
        args(CUDA, [("d_corr", DEV + 4), ("d_essential", None), ("d_points", DEV)]),
    "ps_depth_maps":
        args(ARG, [("n_sets", -1), ("n_refs", -1), ("prm", None), ("report", None), ("ranges", None), ("ranges.0", NAN),
                   ("ranges.1", INF), ("ranges.0", 0.0), ("ranges.0", 10.0)]) +
        fields(ARG, [("n_depths", 1), ("n_depths", 1025), ("radius", 0), ("radius", 8), ("top_k", 0), ("top_k", 33),
                     ("min_sources", 0), ("min_sources", 33), ("max_cost", 0.0), ("max_cost", 2.1), ("max_cost", NAN),
                     ("min_var", NAN), ("min_var", -1.0), ("min_var", INF)]) +
        fields(CUDA, [("n_depths", 1024), ("radius", 7), ("top_k", 32), ("max_cost", 2.0)]) +
        args(CUDA, [("refs.0", 3), ("src_sets.0", 0), ("images.1.width", 6), ("cams.2.fx", 0.0), ("poses.1.t.0", NAN),
                    ("images", None), ("d_depth", None), ("n_sets", 0)]),
    "ps_depth_filter":
        args(ARG, [("n_sets", -1), ("n_refs", -1), ("prm", None), ("report", None)]) +
        fields(ARG, [("max_reproj_error", NAN), ("max_reproj_error", 0.0), ("max_reproj_error", INF), ("max_depth_diff", INF),
                     ("max_depth_diff", 0.0), ("max_depth_diff", NAN), ("min_consistent", 0), ("min_consistent", 256)]) +
        fields(CUDA, [("min_consistent", 255)]) +
        args(CUDA, [("refs.0", 3), ("images.0.width", 0), ("cams.1.fy", NAN), ("d_points", None), ("src_start", None)]),
    "ps_volume_clear": args(ARG, [("vol", None)]) + args(CUDA, [("vol.nx", 1), ("vol.voxel", 0.0), ("vol.tsdf", None)]),
    "ps_tsdf_integrate":
        args(ARG, [("n_views", -1), ("prm", None), ("vol", None), ("report", None), ("images", None), ("cams", None),
                   ("poses", None), ("d_depth", None), ("prm.trunc", NAN), ("prm.trunc", 0.0), ("prm.trunc", INF),
                   ("prm.min_consistent", -1), ("prm.min_consistent", 256), ("prm.min_consistent", 1)]) +
        refused(image_bad("images", 1, 1) + camera_bad("cams", 1) + rigid_bad("poses", 1)) +
        args(CUDA, [("n_views", 0), ("vol.nx", 1), ("images.1.width", 1), ("d_n_consistent", _ptrs(2))]) +
        [(CUDA, "prm.min_consistent 255 with masks", [at("prm.min_consistent", 255), at("d_n_consistent", _ptrs(2))])] +
        [(CUDA, "no views, no arrays", [at("n_views", 0), at("images", None), at("cams", None), at("poses", None),
                                        at("d_depth", None)])],
    "ps_tsdf_mesh": args(ARG, [("vol", None), ("prm", None), ("report", None), ("max_vertices", -1), ("max_triangles", -1),
                               ("prm.min_weight", NAN), ("prm.min_weight", 0.0), ("prm.min_weight", INF)]) +
    args(CUDA, [("vol.nz", 2049), ("max_vertices", 0), ("d_triangles", None)]),
    "ps_mesh_render":
        args(ARG, [("prm", None), ("report", None), ("n_views", -1), ("n_vertices", -1), ("n_triangles", -1),
                   ("n_triangles", 1 << 31), ("d_vertices", None), ("d_triangles", None), ("prm.z_near", NAN),
                   ("prm.z_near", 0.0), ("prm.z_near", INF), ("sizes", None), ("cams", None), ("poses", None), ("d_depth", None),
                   ("d_tri", None), ("sizes.2", 0), ("sizes.2", 65536), ("sizes.3", 0), ("sizes.3", 65536)]) +
        refused(camera_bad("cams", 1) + rigid_bad("poses", 1)) +
        args(CUDA, [("n_views", 0), ("n_triangles", 0), ("n_triangles", (1 << 31) - 1), ("sizes.3", 65535), ("n_vertices", 0)]) +
        [(CUDA, "no triangles, no mesh", [at("n_triangles", 0), at("d_vertices", None), at("d_triangles", None)])],
    "ps_mesh_texture":
        args(ARG, [("prm", None), ("report", None), ("n_views", -1), ("n_vertices", -1), ("n_triangles", -1),
                   ("n_triangles", 1 << 31), ("d_vertices", None), ("d_triangles", None), ("images", None), ("cams", None),
                   ("poses", None), ("d_depth", None), ("d_atlas", None), ("d_view", None)]) +
        fields(ARG, [("z_near", NAN), ("z_near", 0.0), ("depth_tol", NAN), ("depth_tol", -1.0), ("depth_tol", INF),
                     ("min_cos", -0.1), ("min_cos", 1.0), ("min_cos", NAN), ("cell", 2), ("cell", 65), ("cells_per_row", 0),
                     ("cells_per_row", 8192)]) +
        [(ARG, "atlas taller than 65535", [at("n_triangles", 8191 * 16 + 1)])] +
        refused(image_bad("images", 1, 2) + camera_bad("cams", 1) + rigid_bad("poses", 1)) +
        fields(CUDA, [("cell", 3), ("cell", 64), ("min_cos", 0.0), ("cells_per_row", 8191)]) +
        args(CUDA, [("n_triangles", 0), ("n_views", 0), ("n_triangles", 8191 * 16), ("images.1.width", 2)]) +
        [(CUDA, "no triangles, no outputs", [at("n_triangles", 0), at("d_atlas", None), at("d_view", None)])],
}


@pytest.fixture(scope="module")
def lib():
    return api.load_library()


def _call(lib, entry, a, sentinel=True):
    """fill the host outputs with the sentinel, preset ps_last_error(NULL), call; returns the code"""
    fn = getattr(lib, entry)
    assert len(fn.argtypes) == len(a), entry
    for k in OUTS.get(entry, []) if sentinel else []:
        if a[k] is not None:
            C.memset(C.addressof(a[k]), SENTINEL, C.sizeof(a[k]))
    assert lib.ps_create(0, None, 0, 0, 0) is None and lib.ps_last_error(None) == PRESET
    cargs = [C.addressof(v) if t is C.c_void_p and isinstance(v, (C.Structure, C.Array)) else v
             for v, t in zip(a.values(), fn.argtypes)]
    return fn(*cargs)


def _untouched(entry, a):
    for k in OUTS.get(entry, []):
        if a[k] is not None:
            assert C.string_at(C.addressof(a[k]), C.sizeof(a[k])) == bytes([SENTINEL]) * C.sizeof(a[k]), (entry, k)


def test_every_entry_point_is_covered(lib):
    assert len(BUILD) == 27 and set(BUILD) == set(CASES)
    for entry in BUILD:
        assert hasattr(lib, entry) and len(getattr(lib, entry).argtypes) == len(BUILD[entry]())


@pytest.mark.parametrize("entry", sorted(BUILD))
def test_well_formed_call_reaches_the_device(lib, entry):
    a = BUILD[entry]()
    assert _call(lib, entry, a) == CUDA
    _untouched(entry, a)
    assert lib.ps_last_error(None) == PRESET


@pytest.mark.parametrize("entry,expect,muts", [pytest.param(e, x, m, id="%s-%s" % (e, label))
                                               for e in sorted(CASES) for x, label, m in CASES[e]])
def test_argument_checks(lib, entry, expect, muts):
    """PS_ERR_ARG: refused before the device is set; PS_ERR_CUDA: accepted, or checked only after it"""
    a = BUILD[entry]()
    for m in muts:
        m(a)
    assert _call(lib, entry, a) == expect
    _untouched(entry, a)
    assert lib.ps_last_error(None) == PRESET


@pytest.mark.parametrize("pairs", [(0, 1, 1, 2, 0, 1), (0, 1, 1, 2, 1, 0), (2, 1, 0, 2, 1, 2)])
def test_view_graph_duplicate_pair(lib, pairs):
    a = BUILD["ps_view_graph_filter"]()
    a["pairs"] = _ints(*pairs)
    assert _call(lib, "ps_view_graph_filter", a) == ARG
    _untouched("ps_view_graph_filter", a)
    assert lib.ps_last_error(None) == b"ps_view_graph_filter: two pairs join the same two sets"


def _zero(s):
    return C.string_at(C.addressof(s), C.sizeof(s)) == bytes(C.sizeof(s))


@pytest.mark.parametrize("entry,muts", [
    ("ps_match", [at("n_left", 0)]),
    ("ps_match", [at("n_left", 0), at("d_left", None), at("d_out", None), at("n_right", 0), at("d_right", None)]),
    ("ps_descriptors_to_u8", [at("n", 0), at("d_in", None), at("d_out", None)]),
    ("ps_verify_batch", [at("n_pairs", 0), at("corr_start", None), at("n_corr", None)]),
    ("ps_relative_pose_batch", [at("n_pairs", 0), at("corr_start", None), at("n_corr", None), at("cams", None)]),
    ("ps_retrieve_pairs", [at("n", 0), at("d_vec", None)]),
    ("ps_two_view_config_batch", [at("n_pairs", 0), at("corr_start", None), at("cams", None)]),
])
def test_empty_calls_before_the_device(lib, entry, muts):
    """empty work returns PS_OK before the device is set and writes nothing"""
    a = BUILD[entry]()
    for m in muts:
        m(a)
    assert _call(lib, entry, a) == OK
    _untouched(entry, a)
    assert lib.ps_last_error(None) == PRESET


@pytest.mark.parametrize("entry,muts,out", [
    ("ps_triangulate_tracks", [at("n_tracks", 0)], "counts"),
    ("ps_depth_maps", [at("n_refs", 0), at("refs", None), at("ranges", None)], "report"),
    ("ps_depth_filter", [at("n_refs", 0), at("refs", None)], "report"),
])
def test_empty_calls_zero_their_counts(lib, entry, muts, out):
    a = BUILD[entry]()
    for m in muts:
        m(a)
    assert _call(lib, entry, a) == OK
    assert _zero(a[out])


def test_bundle_adjust_without_tracks(lib):
    """PS_BA_NO_OBSERVATIONS, and poses_out = poses_in, also when they are the same array"""
    a = BUILD["ps_bundle_adjust"]()
    a["n_tracks"] = 0
    assert _call(lib, "ps_bundle_adjust", a) == OK
    rep = a["report"]
    assert rep.termination == 3 and all(getattr(rep, f) == 0 for f, _ in api.PsBundleReport._fields_ if f != "termination")
    assert bytes(a["poses_out"]) == bytes(a["poses_in"])
    a = BUILD["ps_bundle_adjust"]()
    a["n_tracks"] = 0
    before = bytes(a["poses_in"])
    a["poses_out"] = a["poses_in"]
    assert _call(lib, "ps_bundle_adjust", a, sentinel=False) == OK
    assert bytes(a["poses_in"]) == before and a["report"].termination == 3


def test_global_positioning_without_tracks(lib):
    """PS_GP_NO_OBSERVATIONS, the given rotations with t = 0, nothing positioned"""
    a = BUILD["ps_global_positioning"]()
    a["n_tracks"] = 0
    assert _call(lib, "ps_global_positioning", a) == OK
    rep = a["report"]
    assert rep.termination == 2 and all(getattr(rep, f) == 0 for f, _ in api.PsPositionReport._fields_ if f != "termination")
    for i in range(2):
        assert list(a["poses_out"][i].R) == list(a["R"][9 * i:9 * i + 9]) and list(a["poses_out"][i].t) == [0.0, 0.0, 0.0]
    assert list(a["positioned"]) == [0, 0]
