"""Image retrieval restated in numpy (include/popsift_b200_retrieval.h): the initial draw of ps_vlad_train, nearest-centroid
assignment in the matcher's float32 order, one k-means step and the VLAD encoding in float64, and the top-m rule of
ps_retrieve_pairs."""
import numpy as np

import match_oracle as mo

M64 = (1 << 64) - 1


def mix(z: int) -> int:
    """splitmix64's finaliser (k_verify_sample.h verify_mix)"""
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(seed: int, N: int, k: int) -> list:
    """the k distinct pool indices of the initial codebook, in draw order"""
    key = mix(seed & M64)
    out, seen, c = [], set(), 0
    while len(out) < k:
        v = ((mix((key + c) & M64) >> 32) * N) >> 32
        c += 1
        if v in seen:
            continue
        seen.add(v)
        out.append(v)
    return out


def assign(x: np.ndarray, centroids: np.ndarray) -> np.ndarray:
    """nearest centroid per descriptor: the matcher's float32 distances, strict < in index order (lower index on ties)"""
    if len(x) == 0:
        return np.zeros(0, np.int32)
    return mo.best_two(mo.sq_dist_matrix(np.asarray(x, np.float32), np.asarray(centroids, np.float32)))[:, 0].astype(np.int32)


def kmeans_step(x: np.ndarray, centroids: np.ndarray, a: np.ndarray) -> np.ndarray:
    """centroid = float64 mean of its members rounded to float32; no members: unchanged"""
    out = np.array(centroids, np.float32, copy=True)
    x64 = np.asarray(x, np.float64)
    for c in range(len(out)):
        sel = a == c
        if sel.any():
            out[c] = (x64[sel].sum(axis=0) / sel.sum()).astype(np.float32)
    return out


def vlad(x: np.ndarray, centroids: np.ndarray, a: np.ndarray) -> np.ndarray:
    """one set's VLAD vector in float64: residual sums, intra-normalisation, signed square root, L2"""
    k = len(centroids)
    v = np.zeros((k, 128), np.float64)
    x64, c64 = np.asarray(x, np.float64), np.asarray(centroids, np.float64)
    for c in range(k):
        sel = a == c
        if sel.any():
            v[c] = (x64[sel] - c64[c]).sum(axis=0)
    n = np.linalg.norm(v, axis=1, keepdims=True)
    v = np.divide(v, n, out=np.zeros_like(v), where=n > 0)
    v = np.sign(v) * np.sqrt(np.abs(v))
    g = np.linalg.norm(v)
    return (v / g if g > 0 else v).reshape(-1)


def topm(S: np.ndarray, m: int):
    """per row i the m best j != i of the score rows S (rows 0 .. len(S)-1 of the n x n matrix, n = S.shape[1]):
    descending, equal scores to the lower j (+0 == -0), NaN below every number; empty slots j = -1, score -inf.
    Returns (nbr (len(S), m) int32, score (len(S), m) float32)."""
    rows, n = S.shape
    nbr = np.full((rows, m), -1, np.int32)
    sc = np.full((rows, m), -np.inf, np.float32)
    for i in range(rows):
        js = [j for j in range(n) if j != i]
        nums = [j for j in js if not np.isnan(S[i, j])]
        nans = [j for j in js if np.isnan(S[i, j])]
        order = sorted(nums, key=lambda j: (-float(S[i, j]), j)) + nans
        for q, j in enumerate(order[:m]):
            nbr[i, q], sc[i, q] = j, S[i, j]
    return nbr, sc


def select_pairs(nbr) -> list:
    """sorted unordered pairs (i < j) of the union of every row's neighbours, -1 dropped"""
    out = set()
    for i, row in enumerate(np.asarray(nbr)):
        for j in row:
            if j >= 0 and j != i:
                out.add((min(i, int(j)), max(i, int(j))))
    return sorted(out)
