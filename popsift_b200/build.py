"""Builds the product's native code IN-TREE with nvcc for sm_90a (H100; no JIT cache).

    python -m popsift_b200.build            # libpopsift_b200.so + popsift-demo

Outputs (git-ignored):
    popsift_b200/lib/libpopsift_b200.so     C-ABI (include/popsift_b200.h) + C++ API (include/popsift/*.h)
    popsift_b200/bin/popsift-demo           CLI mirroring the reference's popsift-demo
"""
from __future__ import annotations

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "popsift_b200")
CSRC = os.path.join(PKG, "csrc")
LIB_DIR = os.path.join(PKG, "lib")
BIN_DIR = os.path.join(PKG, "bin")
OBJ_DIR = os.path.join(PKG, "build")
LIB = os.path.join(LIB_DIR, "libpopsift_b200.so")
DEMO = os.path.join(BIN_DIR, "popsift-demo")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC",
              "--fmad=false",   # no implicit contraction anywhere; every fma in the kernels is explicit
              "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]

LIB_SOURCES = ["ps_tables.cpp", "ps_ctx.cu", "ps_batch.cu", "k_pyramid.cu", "k_pyramid_march.cu", "tma_util.cu", "k_match.cu", "k_match_u8.cu", "k_extrema.cu", "k_filter.cu", "k_orient.cu", "k_desc.cu", "k_desc_modes.cu", "k_describe.cu", "k_verify.cu", "k_pose.cu", "k_retrieval.cu", "k_tracks.cu", "k_triangulate.cu", "k_bundle.cu", "k_global.cu", "k_viewgraph.cu", "k_twoview.cu", "k_depth.cu", "k_mesh.cu", "k_render.cu", "workspace.cu",
               "host/sift_conf.cpp", "host/features.cpp", "host/popsift.cpp", "host/device_prop.cpp", "host/log_dump.cpp"]
DEMO_SOURCES = ["app/popsift_demo.cpp", "app/pgmread.cpp"]
MATCH_SOURCES = ["app/popsift_match.cpp"]            # + app/pgmread.cpp
MATCH = os.path.join(BIN_DIR, "popsift-match")
API_CHECK = os.path.join(BIN_DIR, "api_check")
API_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "api_check.cpp")
API_BENCH = os.path.join(BIN_DIR, "api_bench")
API_BENCH_SRC = os.path.join(ROOT, "tests", "cpp", "api_bench.cpp")
PART_CHECK = os.path.join(BIN_DIR, "partition_check")
PART_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "partition_check.cpp")
PGM_CHECK = os.path.join(BIN_DIR, "pgmread_check")
MATCH_PLAN_CHECK = os.path.join(BIN_DIR, "match_plan_check")
MATCH_PLAN_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "match_plan_check.cpp")
MATCH_PLAN_U8_CHECK = os.path.join(BIN_DIR, "match_plan_u8_check")
MATCH_PLAN_U8_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "match_plan_u8_check.cpp")
MATCH_PAIRS_CHECK = os.path.join(BIN_DIR, "match_pairs_check")
MATCH_PAIRS_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "match_pairs_check.cpp")
MATCH_U8_CHECK = os.path.join(BIN_DIR, "match_u8_check")
MATCH_U8_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "match_u8_check.cpp")
PGM_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "pgmread_check.cpp")
DESCRIBE_CHECK = os.path.join(BIN_DIR, "describe_check")
DESCRIBE_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "describe_check.cpp")
VERIFY_SAMPLE_CHECK = os.path.join(BIN_DIR, "verify_sample_check")
VERIFY_SAMPLE_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "verify_sample_check.cpp")
VERIFY_CHECK = os.path.join(BIN_DIR, "verify_check")
VERIFY_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "verify_check.cpp")
GUIDED_MASK = os.path.join(BIN_DIR, "guided_mask")
GUIDED_MASK_SRC = os.path.join(ROOT, "tests", "cpp", "guided_mask.cpp")
GUIDED_CHECK = os.path.join(BIN_DIR, "guided_check")
GUIDED_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "guided_check.cpp")
RETRIEVAL_HOST = os.path.join(BIN_DIR, "retrieval_host")
RETRIEVAL_HOST_SRC = os.path.join(ROOT, "tests", "cpp", "retrieval_host.cpp")
RETRIEVAL_CHECK = os.path.join(BIN_DIR, "retrieval_check")
RETRIEVAL_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "retrieval_check.cpp")
TRACKS_CHECK = os.path.join(BIN_DIR, "tracks_check")
TRACKS_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "tracks_check.cpp")
POSE_SOLVER_CHECK = os.path.join(BIN_DIR, "pose_solver_check")
POSE_SOLVER_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "pose_solver_check.cpp")
POSE_CHECK = os.path.join(BIN_DIR, "pose_check")
POSE_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "pose_check.cpp")
TRIANGULATE_MATH_CHECK = os.path.join(BIN_DIR, "triangulate_math_check")
TRIANGULATE_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "triangulate_math_check.cpp")
TRIANGULATE_CHECK = os.path.join(BIN_DIR, "triangulate_check")
TRIANGULATE_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "triangulate_check.cpp")
BUNDLE_MATH_CHECK = os.path.join(BIN_DIR, "bundle_math_check")
BUNDLE_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "bundle_math_check.cpp")
BUNDLE_CHECK = os.path.join(BIN_DIR, "bundle_check")
BUNDLE_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "bundle_check.cpp")
GLOBAL_MATH_CHECK = os.path.join(BIN_DIR, "global_math_check")
GLOBAL_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "global_math_check.cpp")
GLOBAL_CHECK = os.path.join(BIN_DIR, "global_check")
GLOBAL_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "global_check.cpp")
VIEWGRAPH_MATH_CHECK = os.path.join(BIN_DIR, "viewgraph_math_check")
VIEWGRAPH_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "viewgraph_math_check.cpp")
VIEWGRAPH_CHECK = os.path.join(BIN_DIR, "viewgraph_check")
VIEWGRAPH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "viewgraph_check.cpp")
TWOVIEW_MATH_CHECK = os.path.join(BIN_DIR, "twoview_math_check")
TWOVIEW_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "twoview_math_check.cpp")
TWOVIEW_CHECK = os.path.join(BIN_DIR, "twoview_check")
TWOVIEW_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "twoview_check.cpp")
DEPTH_MATH_CHECK = os.path.join(BIN_DIR, "depth_math_check")
DEPTH_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "depth_math_check.cpp")
DEPTH_CHECK = os.path.join(BIN_DIR, "depth_check")
DEPTH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "depth_check.cpp")
MESH_MATH_CHECK = os.path.join(BIN_DIR, "mesh_math_check")
MESH_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "mesh_math_check.cpp")
MESH_CHECK = os.path.join(BIN_DIR, "mesh_check")
MESH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "mesh_check.cpp")
RENDER_MATH_CHECK = os.path.join(BIN_DIR, "render_math_check")
RENDER_MATH_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "render_math_check.cpp")
RENDER_CHECK = os.path.join(BIN_DIR, "render_check")
RENDER_CHECK_SRC = os.path.join(ROOT, "tests", "cpp", "render_check.cpp")


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _headers():
    out = []
    for base in (os.path.join(ROOT, "include"), CSRC):
        for dp, _, fs in os.walk(base):
            out += [os.path.join(dp, f) for f in fs if f.endswith((".h", ".hpp", ".cuh"))]
    return out


def build(verbose: bool = False, force: bool = False) -> str:
    for d in (LIB_DIR, BIN_DIR, OBJ_DIR):
        os.makedirs(d, exist_ok=True)
    # products of other compiler flags (another architecture) are rebuilt, whatever their timestamps
    stamp = os.path.join(OBJ_DIR, "flags")
    flags = " ".join(ARCH + NVCC_FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    hdrs = _headers()
    objs = []
    procs = []
    for src in LIB_SOURCES + DEMO_SOURCES + MATCH_SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(OBJ_DIR, src.replace("/", "_") + ".o")
        objs.append((src, obj))
        if force or _newer(obj, [sp] + hdrs):
            cmd = ["nvcc"] + ARCH + NVCC_FLAGS + ["-x", "cu", "-c", sp, "-o", obj]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(out.decode(errors="replace"))
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s" % src)
    lib_objs = [o for s, o in objs if s in LIB_SOURCES]
    demo_objs = [o for s, o in objs if s in DEMO_SOURCES]
    if force or _newer(LIB, lib_objs):
        subprocess.check_call(["nvcc"] + ARCH + ["-shared", "-o", LIB] + lib_objs + ["-lpthread"])
    if demo_objs and (force or _newer(DEMO, demo_objs + [LIB])):
        subprocess.check_call(["nvcc"] + ARCH + ["-o", DEMO] + demo_objs +
                              ["-L" + LIB_DIR, "-lpopsift_b200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../lib", "-lpthread"])
    match_objs = [o for s, o in objs if s in MATCH_SOURCES or s == "app/pgmread.cpp"]
    if len(match_objs) == 2 and (force or _newer(MATCH, match_objs + [LIB])):
        subprocess.check_call(["nvcc"] + ARCH + ["-o", MATCH] + match_objs +
                              ["-L" + LIB_DIR, "-lpopsift_b200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../lib", "-lpthread"])
    if os.path.exists(API_CHECK_SRC) and (force or _newer(API_CHECK, [API_CHECK_SRC, LIB] + hdrs)):
        # a plain host compiler is enough for a caller of the C++ API: no CUDA in the translation unit
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), API_CHECK_SRC, "-o", API_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    if os.path.exists(API_BENCH_SRC) and (force or _newer(API_BENCH, [API_BENCH_SRC, LIB] + hdrs)):
        # end-to-end timing through the C++ API from pageable frames (bench.py's e2e leg)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), API_BENCH_SRC, "-o", API_BENCH,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    part_hdr = os.path.join(CSRC, "k_partition.h")
    if os.path.exists(PART_CHECK_SRC) and (force or _newer(PART_CHECK, [PART_CHECK_SRC, part_hdr])):
        # host-only sweep of the marching kernels' work partition (no CUDA, no library)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + CSRC, PART_CHECK_SRC, "-o", PART_CHECK])
    plan_hdr = os.path.join(CSRC, "k_match_plan.h")
    if os.path.exists(MATCH_PLAN_CHECK_SRC) and (force or _newer(MATCH_PLAN_CHECK, [MATCH_PLAN_CHECK_SRC, plan_hdr])):
        # host-only sweep of the batched matcher's planner (no CUDA, no library)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + CSRC, MATCH_PLAN_CHECK_SRC, "-o", MATCH_PLAN_CHECK])
    if os.path.exists(MATCH_PLAN_U8_CHECK_SRC) and (force or _newer(MATCH_PLAN_U8_CHECK, [MATCH_PLAN_U8_CHECK_SRC, plan_hdr])):
        # the same planner at the 8-bit matcher's 132-byte rows (host only)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + CSRC, MATCH_PLAN_U8_CHECK_SRC, "-o", MATCH_PLAN_U8_CHECK])
    if os.path.exists(MATCH_PAIRS_CHECK_SRC) and (force or _newer(MATCH_PAIRS_CHECK, [MATCH_PAIRS_CHECK_SRC, LIB] + hdrs)):
        # popsift::matchPairs against FeaturesDev::matchIndices through the C++ API
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), MATCH_PAIRS_CHECK_SRC, "-o", MATCH_PAIRS_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    if os.path.exists(MATCH_U8_CHECK_SRC) and (force or _newer(MATCH_U8_CHECK, [MATCH_U8_CHECK_SRC, LIB] + hdrs)):
        # popsift::matchPairsU8 against the float matcher on the quantised descriptors, through the C++ and C APIs
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), MATCH_U8_CHECK_SRC, "-o", MATCH_U8_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    if os.path.exists(DESCRIBE_CHECK_SRC) and (force or _newer(DESCRIBE_CHECK, [DESCRIBE_CHECK_SRC, LIB] + hdrs)):
        # PopSift::describe round trip with describe and enqueue jobs in one FIFO, through the C++ API
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), DESCRIBE_CHECK_SRC, "-o", DESCRIBE_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    sample_hdr = os.path.join(CSRC, "k_verify_sample.h")
    if os.path.exists(VERIFY_SAMPLE_CHECK_SRC) and (force or _newer(VERIFY_SAMPLE_CHECK, [VERIFY_SAMPLE_CHECK_SRC, sample_hdr])):
        # host-only: the RANSAC sample hash, the same __host__ __device__ function the kernel uses (no CUDA, no library)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + CSRC, VERIFY_SAMPLE_CHECK_SRC, "-o", VERIFY_SAMPLE_CHECK])
    if os.path.exists(VERIFY_CHECK_SRC) and (force or _newer(VERIFY_CHECK, [VERIFY_CHECK_SRC, LIB] + hdrs)):
        # popsift::verifyPairs against the C ABI (ps_match_correspondences + ps_verify_batch), through the C++ API
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), VERIFY_CHECK_SRC, "-o", VERIFY_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    guided_hdr = os.path.join(CSRC, "k_guided.h")
    if os.path.exists(GUIDED_MASK_SRC) and (force or _newer(GUIDED_MASK, [GUIDED_MASK_SRC, guided_hdr])):
        # host-only: guided matching's eligibility mask, the same __host__ __device__ function the kernels use (no CUDA, no
        # library); no contraction, so that every rounding is the one the function spells out
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, GUIDED_MASK_SRC, "-o", GUIDED_MASK])
    if os.path.exists(GUIDED_CHECK_SRC) and (force or _newer(GUIDED_CHECK, [GUIDED_CHECK_SRC, LIB] + hdrs)):
        # popsift::matchPairsGuided(U8) against the C ABI (ps_match_guided_batch / ps_match_u8_guided_batch)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), GUIDED_CHECK_SRC, "-o", GUIDED_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    retr_hdrs = [os.path.join(CSRC, "k_retrieval.h"), sample_hdr]
    if os.path.exists(RETRIEVAL_HOST_SRC) and (force or _newer(RETRIEVAL_HOST, [RETRIEVAL_HOST_SRC] + retr_hdrs)):
        # host-only: retrieval's initial draw and score chain, the same __host__ __device__ functions the kernels use (no
        # CUDA, no library); no contraction, so that every rounding is the one the functions spell out
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, RETRIEVAL_HOST_SRC, "-o", RETRIEVAL_HOST])
    if os.path.exists(RETRIEVAL_CHECK_SRC) and (force or _newer(RETRIEVAL_CHECK, [RETRIEVAL_CHECK_SRC, LIB] + hdrs)):
        # popsift::vladCodebook / vladEncode / retrievePairs against the C ABI (popsift_b200_retrieval.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), RETRIEVAL_CHECK_SRC, "-o", RETRIEVAL_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    if os.path.exists(TRACKS_CHECK_SRC) and (force or _newer(TRACKS_CHECK, [TRACKS_CHECK_SRC, LIB] + hdrs)):
        # popsift::buildTracks (both overloads) against the C ABI (popsift_b200_tracks.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), TRACKS_CHECK_SRC, "-o", TRACKS_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    pose_hdrs = [os.path.join(CSRC, "k_pose_solve.h"), sample_hdr]
    if os.path.exists(POSE_SOLVER_CHECK_SRC) and (force or _newer(POSE_SOLVER_CHECK, [POSE_SOLVER_CHECK_SRC] + pose_hdrs)):
        # host-only: the five-point solver, the pose decomposition, the triangulation and the m = 5 sample hash, the same
        # __host__ __device__ functions the kernels use (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, POSE_SOLVER_CHECK_SRC, "-o", POSE_SOLVER_CHECK])
    if os.path.exists(POSE_CHECK_SRC) and (force or _newer(POSE_CHECK, [POSE_CHECK_SRC, LIB] + hdrs)):
        # popsift::relativePoses against the C ABI (popsift_b200_pose.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), POSE_CHECK_SRC, "-o", POSE_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    tri_hdrs = [os.path.join(CSRC, "k_triangulate.h")] + pose_hdrs
    if os.path.exists(TRIANGULATE_MATH_CHECK_SRC) and (force or _newer(TRIANGULATE_MATH_CHECK, [TRIANGULATE_MATH_CHECK_SRC] + tri_hdrs)):
        # host-only: the rays, hypotheses, residuals and Gauss-Newton steps of triangulation, the same __host__ __device__
        # functions the kernels use (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, TRIANGULATE_MATH_CHECK_SRC, "-o",
                               TRIANGULATE_MATH_CHECK])
    if os.path.exists(TRIANGULATE_CHECK_SRC) and (force or _newer(TRIANGULATE_CHECK, [TRIANGULATE_CHECK_SRC, LIB] + hdrs)):
        # popsift::triangulateTracks against the C ABI (popsift_b200_triangulate.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), TRIANGULATE_CHECK_SRC, "-o",
                               TRIANGULATE_CHECK, "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    ba_hdrs = [os.path.join(CSRC, "k_bundle.h")] + tri_hdrs
    if os.path.exists(BUNDLE_MATH_CHECK_SRC) and (force or _newer(BUNDLE_MATH_CHECK, [BUNDLE_MATH_CHECK_SRC] + ba_hdrs)):
        # host-only: the Jacobians, loss, Rodrigues update and small solves of bundle adjustment, the same __host__
        # __device__ functions the kernels use (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, BUNDLE_MATH_CHECK_SRC, "-o",
                               BUNDLE_MATH_CHECK])
    if os.path.exists(BUNDLE_CHECK_SRC) and (force or _newer(BUNDLE_CHECK, [BUNDLE_CHECK_SRC, LIB] + hdrs)):
        # popsift::bundleAdjust against the C ABI (popsift_b200_bundle.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), BUNDLE_CHECK_SRC, "-o",
                               BUNDLE_CHECK, "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    gl_hdrs = [os.path.join(CSRC, "k_global.h")] + ba_hdrs
    if os.path.exists(GLOBAL_MATH_CHECK_SRC) and (force or _newer(GLOBAL_MATH_CHECK, [GLOBAL_MATH_CHECK_SRC] + gl_hdrs)):
        # host-only: the rotation logarithm, pair residual, rotation update and observation rule of the global-pose
        # kernels, the same __host__ __device__ functions (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, GLOBAL_MATH_CHECK_SRC, "-o",
                               GLOBAL_MATH_CHECK])
    if os.path.exists(GLOBAL_CHECK_SRC) and (force or _newer(GLOBAL_CHECK, [GLOBAL_CHECK_SRC, LIB] + hdrs)):
        # popsift::rotationAveraging / globalPositioning against the C ABI (popsift_b200_global.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), GLOBAL_CHECK_SRC, "-o",
                               GLOBAL_CHECK, "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    vg_hdrs = [os.path.join(CSRC, "k_viewgraph.h")] + gl_hdrs
    if os.path.exists(VIEWGRAPH_MATH_CHECK_SRC) and (force or _newer(VIEWGRAPH_MATH_CHECK, [VIEWGRAPH_MATH_CHECK_SRC] + vg_hdrs)):
        # host-only: the cycle error of the view-graph filter, the same __host__ __device__ function the kernel uses (no
        # CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, VIEWGRAPH_MATH_CHECK_SRC, "-o",
                               VIEWGRAPH_MATH_CHECK])
    if os.path.exists(VIEWGRAPH_CHECK_SRC) and (force or _newer(VIEWGRAPH_CHECK, [VIEWGRAPH_CHECK_SRC, LIB] + hdrs)):
        # popsift::filterViewGraph against the C ABI (popsift_b200_viewgraph.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), VIEWGRAPH_CHECK_SRC, "-o",
                               VIEWGRAPH_CHECK, "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    tv_hdrs = [os.path.join(CSRC, "k_twoview.h")] + pose_hdrs
    if os.path.exists(TWOVIEW_MATH_CHECK_SRC) and (force or _newer(TWOVIEW_MATH_CHECK, [TWOVIEW_MATH_CHECK_SRC] + tv_hdrs)):
        # host-only: Kabsch, the homography's normalisation, sign and decomposition, the pruning and the triangulation angle
        # of the two-view configuration, the same __host__ __device__ functions the kernel uses (no CUDA, no library); no
        # contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, TWOVIEW_MATH_CHECK_SRC, "-o",
                               TWOVIEW_MATH_CHECK])
    if os.path.exists(TWOVIEW_CHECK_SRC) and (force or _newer(TWOVIEW_CHECK, [TWOVIEW_CHECK_SRC, LIB] + hdrs)):
        # popsift::twoViewGeometries against the C ABI (popsift_b200_twoview.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), TWOVIEW_CHECK_SRC, "-o",
                               TWOVIEW_CHECK, "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    depth_hdrs = [os.path.join(CSRC, "k_depth.h"), sample_hdr]
    if os.path.exists(DEPTH_MATH_CHECK_SRC) and (force or _newer(DEPTH_MATH_CHECK, [DEPTH_MATH_CHECK_SRC] + depth_hdrs)):
        # host-only: the depth kernels' warp, NCC, aggregation, parabola and consistency test, the same __host__ __device__
        # functions the kernels use (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, DEPTH_MATH_CHECK_SRC, "-o",
                               DEPTH_MATH_CHECK])
    if os.path.exists(DEPTH_CHECK_SRC) and (force or _newer(DEPTH_CHECK, [DEPTH_CHECK_SRC, LIB] + hdrs)):
        # popsift::depthMaps / filterDepthMaps against the C ABI (popsift_b200_depth.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), DEPTH_CHECK_SRC, "-o", DEPTH_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    mesh_hdrs = [os.path.join(CSRC, "k_mesh.h"), sample_hdr]
    if os.path.exists(MESH_MATH_CHECK_SRC) and (force or _newer(MESH_MATH_CHECK, [MESH_MATH_CHECK_SRC] + mesh_hdrs)):
        # host-only: the integration's projection, signed distance and running averages, the Kuhn table and the edge
        # vertex, the same functions and tables the kernels use (no CUDA, no library); no contraction, as in the kernels
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, MESH_MATH_CHECK_SRC, "-o",
                               MESH_MATH_CHECK])
    if os.path.exists(MESH_CHECK_SRC) and (force or _newer(MESH_CHECK, [MESH_CHECK_SRC, LIB] + hdrs)):
        # popsift::clearVolume / integrateDepthMaps / extractMesh against the C ABI (popsift_b200_mesh.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), MESH_CHECK_SRC, "-o", MESH_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    render_hdrs = [os.path.join(CSRC, "k_render.h"), sample_hdr]
    if os.path.exists(RENDER_MATH_CHECK_SRC) and (force or _newer(RENDER_MATH_CHECK, [RENDER_MATH_CHECK_SRC] + render_hdrs)):
        # host-only: the rasteriser's projection, edge functions, depth and key, and the texturing's facing test, probe,
        # texel barycentrics and bilinear sample, the same functions the kernels use (no CUDA, no library); no contraction
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I" + CSRC, RENDER_MATH_CHECK_SRC, "-o",
                               RENDER_MATH_CHECK])
    if os.path.exists(RENDER_CHECK_SRC) and (force or _newer(RENDER_CHECK, [RENDER_CHECK_SRC, LIB] + hdrs)):
        # popsift::renderMesh / textureMesh against the C ABI (popsift_b200_render.h)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), RENDER_CHECK_SRC, "-o", RENDER_CHECK,
                               "-L" + LIB_DIR, "-lpopsift_b200", "-Wl,-rpath," + "$ORIGIN/../lib", "-lpthread"])
    pgm_src = os.path.join(CSRC, "app", "pgmread.cpp")
    if os.path.exists(PGM_CHECK_SRC) and (force or _newer(PGM_CHECK, [PGM_CHECK_SRC, pgm_src, os.path.join(CSRC, "app", "pgmread.h")])):
        # host-only check of popsift-demo's image reader
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(CSRC, "app"), PGM_CHECK_SRC, pgm_src, "-o", PGM_CHECK])
    with open(stamp, "w") as f:
        f.write(flags)
    return LIB


if __name__ == "__main__":
    build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(LIB)
