"""CPU restatement of guided matching (include/popsift_b200_guided.h).

- `sq_err64`: the eligibility test's error in float64 (squared transfer error for a homography, squared Sampson distance
  for a fundamental matrix); eligible means err < t^2.
- `mask_exact`: the float32 mask of the kernels' own __host__ __device__ function (k_guided.h), through the host program
  tests/cpp/guided_mask (built by popsift_b200.build).
- `guided_rows`: the masked 2-NN -- match_oracle.sq_dist_matrix in the reference's order, ineligible entries +inf, then
  match_oracle.best_two.  That is the row definition of the header, including (0, 0, 0) when nothing is eligible and
  (j, 0, 1) when only j is."""
from __future__ import annotations

import os
import subprocess
import tempfile

import numpy as np

import match_oracle as mo

HOMOGRAPHY, FUNDAMENTAL = 0, 1


def sq_err64(model: int, M, pl, pr) -> np.ndarray:
    """(n_l, n_r) float64 errors of every (left point, right point) under the 3x3 model M (left -> right, pixels)"""
    M = np.asarray(M, np.float64).reshape(3, 3)
    pl = np.asarray(pl, np.float64).reshape(-1, 2)
    pr = np.asarray(pr, np.float64).reshape(-1, 2)
    hl = np.c_[pl, np.ones(len(pl))]
    hr = np.c_[pr, np.ones(len(pr))]
    a = hl @ M.T                                   # (n_l, 3): H x_l or F x_l
    with np.errstate(divide="ignore", invalid="ignore"):
        if model == HOMOGRAPHY:
            u, v, w = a[:, 0:1], a[:, 1:2], a[:, 2:3]
            X, Y = pr[None, :, 0], pr[None, :, 1]
            return ((u - X * w) ** 2 + (v - Y * w) ** 2) / (w * w)
        b = hr @ M                                 # (n_r, 3): F^T x_r
        e = a @ hr.T                               # (n_l, n_r): x_r . F x_l
        den = (a[:, 0:1] ** 2 + a[:, 1:2] ** 2) + (b[None, :, 0] ** 2 + b[None, :, 1] ** 2)
        return e * e / den


def eligible64(model: int, t: float, M, pl, pr) -> np.ndarray:
    return sq_err64(model, M, pl, pr) < float(t) ** 2


def mask_exact(model: int, t: float, M, pl, pr, exe: str | None = None) -> np.ndarray:
    """the kernels' float32 test, bit for bit (tests/cpp/guided_mask): (n_l, n_r) bool"""
    if exe is None:
        from popsift_b200 import build as B
        exe = B.GUIDED_MASK
    pl = np.ascontiguousarray(pl, np.float32).reshape(-1, 2)
    pr = np.ascontiguousarray(pr, np.float32).reshape(-1, 2)
    with tempfile.TemporaryDirectory() as d:
        inp, out = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(inp, "wb") as f:
            f.write(np.int32(model).tobytes() + np.float32(t).tobytes() + np.asarray(M, np.float32).reshape(9).tobytes())
            f.write(np.int32(len(pl)).tobytes() + pl.tobytes() + np.int32(len(pr)).tobytes() + pr.tobytes())
        r = subprocess.run([exe, inp, out], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        return np.fromfile(out, np.uint8).reshape(len(pl), len(pr)).astype(bool)


def guided_rows(left: np.ndarray, right: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """(n_left, 3) int32 rows of the masked 2-NN (float32 descriptors, the reference's distance order)"""
    nl, nr = len(left), len(right)
    if nl == 0:
        return np.zeros((0, 3), np.int32)
    if nr == 0:
        return np.zeros((nl, 3), np.int32)
    d = mo.sq_dist_matrix(np.asarray(left, np.float32), np.asarray(right, np.float32))
    d[~mask] = np.inf
    return mo.best_two(d)


def random_homography(rng, w=1920, h=1080, jitter=0.15) -> np.ndarray:
    """a homography that moves the image corners by up to jitter * size, scaled to H22 = 1"""
    src = np.array([[0, 0], [w, 0], [w, h], [0, h]], np.float64)
    dst = src + rng.uniform(-jitter, jitter, (4, 2)) * [w, h]
    A = []
    for (x, y), (u, v) in zip(src, dst):
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y, -u])
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y, -v])
    H = np.linalg.svd(np.asarray(A))[2][-1].reshape(3, 3)
    return H / H[2, 2]


def random_fundamental(rng, w=1920, h=1080) -> np.ndarray:
    """F = K^-T [t]x R K^-1 of a random relative pose, Frobenius norm 1"""
    f = rng.uniform(0.8, 1.5) * w
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    ang = rng.normal(0, 0.1, 3)
    Rx = np.array([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]])
    Ry = np.array([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]])
    Rz = np.array([[np.cos(ang[2]), -np.sin(ang[2]), 0], [np.sin(ang[2]), np.cos(ang[2]), 0], [0, 0, 1]])
    t = rng.normal(0, 1, 3)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Ki = np.linalg.inv(K)
    F = Ki.T @ tx @ (Rz @ Ry @ Rx) @ Ki
    return F / np.linalg.norm(F)
