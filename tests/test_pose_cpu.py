"""ps_relative_pose_batch without a GPU: the host-compiled solver, decomposition and sample hash (pose_solver_check, the
same __host__ __device__ code as the kernels) against tests/pose_oracle.py and the planted truth, the oracle against its
truth and OpenCV, and the ABI layout."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import pose_oracle as po          # noqa: E402
import verify_oracle as vo        # noqa: E402
from popsift_b200 import api      # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "popsift_b200", "bin", "pose_solver_check")


def _run(mode, payload, tmp_path):
    if not os.path.exists(CHECK):
        pytest.skip("pose_solver_check is not built (python -m popsift_b200.build)")
    i, o = tmp_path / (mode + ".in"), tmp_path / (mode + ".out")
    i.write_bytes(payload)
    subprocess.check_call([CHECK, mode, str(i), str(o)])
    return o.read_bytes()


def _clean_samples(rng, n):
    out, truth, scenes = [], [], []
    for _ in range(n):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, 5, 1.0, 0.0)
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(5)])).T
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(5)])).T
        out.append(np.hstack([xl[:, :2], xr[:, :2]]))
        truth.append(po.essential(R, t))
    return np.array(out), truth


def _solve(samples, tmp_path):
    N = len(samples)
    raw = _run("solve", np.array([N], np.int64).tobytes() + np.asarray(samples, np.float64).tobytes(), tmp_path)
    cnt = np.frombuffer(raw[:4 * N], np.int32)
    sol = np.frombuffer(raw[4 * N:], np.float64).reshape(N, 10, 3, 3)
    return cnt, sol


def test_solver_contains_truth(tmp_path):
    # 10^4 noise-free planted samples.  Measured on this data: 97.9 % within 1e-9 of the true E (Frobenius, both scaled),
    # 99.5 % within 1e-6, 99.94 % within 1e-3.  The solution count is never short; the misses are roots of an
    # ill-conditioned degree-10 polynomial whose (x, y, z) the Gauss-Newton polish cannot bring to full precision
    samples, truth = _clean_samples(np.random.default_rng(11), 10000)
    cnt, sol = _solve(samples, tmp_path)
    assert cnt.min() >= 0 and cnt.max() <= 10 and (cnt % 2 == 0).all()      # real roots of a real degree-10 polynomial
    d = np.array([min([np.linalg.norm(S - vo.scale_output(vo.FUNDAMENTAL, T)) for S in sol[i, :cnt[i]]] or [9.0])
                  for i, T in enumerate(truth)])
    assert (d <= 1e-9).mean() >= 0.97
    assert (d <= 1e-6).mean() >= 0.99
    assert (d <= 1e-3).mean() >= 0.999


def test_solver_matches_oracle_on_stable_samples(tmp_path):
    samples, _ = _clean_samples(np.random.default_rng(12), 600)
    cnt, sol = _solve(samples, tmp_path)
    n_stable = agree = 0
    for i in range(len(samples)):
        S, stable = po.five_point(samples[i], info=True)
        if not stable:
            continue
        n_stable += 1
        agree += po.same_set(list(sol[i, :cnt[i]]), S, 1e-7)
    # measured: 583 of 600 stable samples give the oracle's set within 1e-7; every disagreement has the same count and
    # differs in precision only (1e-7 .. 1e-1 on a few ill-conditioned roots)
    assert n_stable >= 300
    assert agree >= 0.95 * n_stable


def test_oracle_recovers_planted_pose():
    rng = np.random.default_rng(13)
    for _ in range(50):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, 5, 1.0, 0.0)
        rows, _ = po.calibrate(clean, cams[0], cams[1], 1.0)
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(5)])).T
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(5)])).T
        S = po.five_point(np.hstack([xl[:, :2], xr[:, :2]]))
        assert po.contains(S, po.essential(R, t), 1e-8)
    for _ in range(20):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, 200, 1.0, 0.0)
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(200)])).T
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(200)])).T
        k, Rc, tc, counts = po.choose(po.essential(R, t), np.hstack([xl[:, :2], xr[:, :2]]))
        assert po.rot_angle(Rc, R) < 1e-6 and po.dir_angle(tc, t) < 1e-6 and counts[k] == 200


def test_decomposition_picks_truth_in_every_position(tmp_path):
    rng = np.random.default_rng(14)
    N, M = 400, 60
    payload = [np.array([N, M], np.int64).tobytes()]
    truth = []
    for i in range(N):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, M, 1.0, 0.0, forward=bool(i % 2))
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(M)])).T
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(M)])).T
        E = vo.scale_output(vo.FUNDAMENTAL, po.essential(R, t))
        payload.append(np.concatenate([E.ravel(), np.hstack([xl[:, :2], xr[:, :2]]).ravel()]).astype(np.float64).tobytes())
        truth.append((R, t))
    raw = _run("pose", b"".join(payload), tmp_path)
    head = np.frombuffer(raw[:20 * N], np.int32).reshape(N, 5)
    rt = np.frombuffer(raw[20 * N:], np.float64).reshape(N, 12)
    for i, (R, t) in enumerate(truth):
        assert po.rot_angle(rt[i, :9].reshape(3, 3), R) < 1e-6
        assert po.dir_angle(rt[i, 9:], t) < 1e-6
        assert head[i, 1 + head[i, 0]] == M
    assert set(head[:, 0].tolist()) == {0, 1, 2, 3}


def test_sample_hash_m5(tmp_path):
    rng = np.random.default_rng(15)
    N = 100000
    seed = 0x1234_5678_9ABC_DEF0
    p = rng.integers(0, 1 << 20, N).astype(np.int32)
    s = rng.integers(0, 65536, N).astype(np.int32)
    n = rng.integers(1, 50000, N).astype(np.int32)
    n[:1000] = rng.integers(1, 8, 1000)
    rec = np.stack([p, s, n], 1).astype(np.int32)
    raw = _run("sample", np.array([seed], np.uint64).tobytes() + np.array([N], np.int64).tobytes() + rec.tobytes(), tmp_path)
    res = np.frombuffer(raw, np.uint32).reshape(N, 6)
    valid, idx = vo.samples(seed, p, s, n, 5)
    assert (res[:, 0].astype(bool) == valid).all()
    assert (res[valid, 1:] == idx[valid]).all()


def _cv2():
    try:
        import cv2 as m
        return m
    except ImportError:
        pytest.skip("cv2 is not available")


def test_oracle_against_opencv_five_point():
    cv = _cv2()
    rng = np.random.default_rng(16)
    checked = agree = 0
    for _ in range(100):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, 5, 1.0, 0.0)
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(5)])).T[:, :2]
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(5)])).T[:, :2]
        S, stable = po.five_point(np.hstack([xl, xr]), info=True)
        # OpenCV's E maps points1 to points2: x2^T E x1 = 0, as here
        Ecv, _ = cv.findEssentialMat(xl, xr, np.eye(3), method=cv.LMEDS)
        if Ecv is None or not stable:
            continue
        cvs = [vo.scale_output(vo.FUNDAMENTAL, Ecv[3 * k:3 * k + 3]) for k in range(len(Ecv) // 3)]
        checked += 1
        agree += po.same_set(S, cvs, 1e-6)
    # OpenCV 4.13 drops or perturbs a solution on some stable samples; the oracle keeps the truth on all of them
    # (test_oracle_recovers_planted_pose)
    assert checked >= 50 and agree >= 0.8 * checked


def test_oracle_against_opencv_recover_pose():
    cv = _cv2()
    rng = np.random.default_rng(17)
    for _ in range(30):
        corr, cams, R, t, inl, err, clean = po.planted_pose(rng, 100, 1.0, 0.0)
        xl = (np.linalg.inv(po.K(cams[0])) @ np.vstack([clean[:, :2].T, np.ones(100)])).T[:, :2]
        xr = (np.linalg.inv(po.K(cams[1])) @ np.vstack([clean[:, 2:].T, np.ones(100)])).T[:, :2]
        E = po.essential(R, t)
        k, Rc, tc, _ = po.choose(E, np.hstack([xl, xr]))
        _, Rcv, tcv, _ = cv.recoverPose(E, xl, xr, np.eye(3))
        assert po.rot_angle(Rc, Rcv) < 1e-6 and po.dir_angle(tc, tcv.ravel()) < 1e-6


def test_abi_layout():
    assert C.sizeof(api.PsCamera) == 16
    assert C.sizeof(api.PsPoseParams) == 24 and api.PsPoseParams.seed.offset == 16
    assert api.TWO_VIEW_DTYPE.itemsize == 128


def test_pose_exports():
    hdr = open(os.path.join(ROOT, "include", "popsift_b200_pose.h")).read()
    declared = re.findall(r"^int (ps_\w+)\(", hdr, re.M)
    assert declared == api.POSE_EXPORTS
    others = set(api.EXPORTS) | set(api.GUIDED_EXPORTS) | set(api.RETRIEVAL_EXPORTS) | set(api.TRACKS_EXPORTS)
    assert not set(api.POSE_EXPORTS) & others
    lib = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
    if not os.path.exists(lib):
        pytest.skip("library not built")
    L = C.CDLL(lib)
    for name in api.POSE_EXPORTS:
        assert hasattr(L, name)
