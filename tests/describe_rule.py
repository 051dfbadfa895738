"""numpy restatement of the octave / level rule of ps_describe_* for keypoints with octave = level = -1
(include/popsift_b200.h), in float32 like the kernel:

    S      = L * (log2f(sigma) + up_fac - log2f(sigma0))
    octave = clamp(floor((S - 0.5) / L), 0, n_octaves - 1)
    level  = clamp(roundf(S - octave * L), 0, L + 2)          (roundf: halves away from zero)

and of the rest of the keypoint validation, so that the tests can predict which keypoints are rejected."""
import numpy as np

F = np.float32


def scale_index(sigma, sigma0, levels, up_fac):
    """S in float32, evaluated in the kernel's order"""
    sigma = np.asarray(sigma, F)
    with np.errstate(divide="ignore", invalid="ignore"):
        return F(levels) * ((np.log2(sigma) + F(up_fac)) - np.log2(F(sigma0)))


def octave_level_from_s(S, levels, n_octaves, octave=None):
    """(octave, level) from S; `octave` (optional, -1 = derive) takes an explicit octave instead"""
    S = np.asarray(S, F)
    L = F(levels)
    o = np.floor(((S - F(0.5)) / L).astype(np.float64))
    o = np.clip(np.nan_to_num(o, nan=0.0, posinf=n_octaves, neginf=0.0), 0, n_octaves - 1).astype(np.int64)
    if octave is not None:
        octave = np.asarray(octave, np.int64)
        o = np.where(octave >= 0, octave, o)
    t = (S - (o * levels).astype(F)).astype(np.float64)
    r = np.sign(t) * np.floor(np.abs(t) + 0.5)          # roundf, exact in float64
    lvl = np.clip(np.nan_to_num(r, nan=0.0), 0, levels + 2).astype(np.int64)
    return o, lvl


def octave_level(sigma, sigma0, levels, up_fac, n_octaves, octave=None):
    S = scale_index(sigma, sigma0, levels, up_fac)
    o, lvl = octave_level_from_s(S, levels, n_octaves, octave)
    return o, lvl, S


def near_rounding_edge(S, o, levels, eps=1e-4):
    """keypoints whose derived level or octave sits within eps of a rounding boundary: log2f on the device and numpy's
    log2 may differ in the last bit there"""
    S = np.asarray(S, np.float64)
    t = S - o * levels
    return (np.abs(t - np.round(t - 0.5) - 0.5) < eps) | (np.abs((S - 0.5) / levels - np.round((S - 0.5) / levels)) < eps)


def place(kp, sigma0, levels, up_fac, dims, orient):
    """what the kernel does with a KEYPOINT_DTYPE array: (valid, octave, level, local x, y, sigma, S); dims = [(W_o, H_o)]"""
    n_oct = len(dims)
    x, y, s, a = (kp[k].astype(F) for k in ("x", "y", "sigma", "ori"))
    eo, el = kp["octave"].astype(np.int64), kp["level"].astype(np.int64)
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(s) & (s > 0)
    if not orient:
        ok &= np.isfinite(a)
    ok &= (eo == -1) | ((eo >= 0) & (eo < n_oct))
    ok &= (el == -1) | ((el >= 0) & (el <= levels + 2))
    S = scale_index(np.where(ok, s, F(1)), sigma0, levels, up_fac)
    o, lvl = octave_level_from_s(S, levels, n_oct, np.where(ok, eo, -1))
    lvl = np.where(el >= 0, el, lvl)
    sc = np.ldexp(F(1), (up_fac - o).astype(np.int32)).astype(F)
    with np.errstate(invalid="ignore", over="ignore"):
        xl, yl, sl = x * sc, y * sc, s * sc
    W = np.array([d[0] for d in dims])[o]
    H = np.array([d[1] for d in dims])[o]
    with np.errstate(invalid="ignore"):
        ok &= (xl >= 0) & (xl <= (W - 1).astype(F)) & (yl >= 0) & (yl <= (H - 1).astype(F))
    return ok, o, lvl, xl, yl, sl, S
