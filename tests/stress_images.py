"""Deterministic adversarial test images for the extraction path (numpy only).

popsift_b200.synth.make_frame draws smooth, band-limited texture whose steps stay below ~36 grey levels.  The images
here reach what it never does: full-contrast 0 / 255 gradients (the descriptor's fixed-point bins), very dense extrema
(stage-3 queue overflow, capacity growth), structure in the outermost rows and columns (border clamps of orientation and
descriptor, OpenCV's 5-pixel margin), saturated plateaus, DoG values near the threshold, and the top of the float-image
range.  Every image is built with integer arithmetic only, so the same name gives the same bytes everywhere
(tests/test_host_cpu.py pins their sha256).

    image(name)            uint8 (h, w); names ending in _f32 give float32 in [0, 1]
    image(name, w, h)      the same content at another size (not pinned)
"""
from __future__ import annotations

import numpy as np

from popsift_b200.synth import make_frame

W, H = 640, 480

# name -> (default width, default height)
SIZES = {
    "checker_p2": (W, H), "checker_p3": (W, H), "checker_p8": (W, H), "checker_rot30_p6": (W, H),
    "block_noise_4": (W, H), "binary_noise": (320, 240), "saturated": (W, H), "dark": (W, H),
    "border_impulses": (W, H), "step_edges": (W, H), "const_0": (160, 120), "const_255": (160, 120),
    "binary_noise_f32": (320, 240), "checker_p8_f32": (W, H),
    # one 6 x 6 blob per 3 x 3 square at octave 0: ~920 000 3x3x3 DoG extrema, more than the candidate extrema kernel's
    # stage-3 queues hold (1024 per block)
    "checker_p3_4k": (3840, 2160),
}
NAMES = tuple(SIZES)


def _grid(w, h):
    return np.mgrid[0:h, 0:w].astype(np.int64)


def _checker(w, h, p):
    y, x = _grid(w, h)
    return (255 * (((x // p) + (y // p)) & 1)).astype(np.uint8)


def _checker_rot30(w, h, p):
    """checkerboard of period p in coordinates rotated by atan(500 / 866) = 30.0007 degrees (exact integers)"""
    y, x = _grid(w, h)
    u = 866 * x + 500 * y
    v = -500 * x + 866 * y
    return (255 * (((u // (1000 * p)) + (v // (1000 * p))) & 1)).astype(np.uint8)


def _binary_noise(w, h, seed, block=1):
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 2, size=((h + block - 1) // block, (w + block - 1) // block), dtype=np.uint8) * np.uint8(255)
    return np.ascontiguousarray(np.repeat(np.repeat(b, block, 0), block, 1)[:h, :w])


def _border_impulses(w, h):
    """grey 128 with 0 / 255 impulses and 1-pixel lines in rows / columns 0, 1, 2, n-3, n-2, n-1, at the four corners
    and in the interior.  A single pixel's DoG response falls monotonically with scale (no scale-space extremum), so
    the impulses along the borders are squares of side 1, 2, 3, 4 and 6 starting in those rows / columns: the larger
    ones are detected with their keypoint a few pixels from the edge, their orientation window and descriptor support
    reaching over it."""
    img = np.full((h, w), 128, np.uint8)
    sides = (1, 2, 3, 4, 6)
    for k, d in enumerate((0, 1, 2)):
        for j, x in enumerate(range(24 + 7 * k, w - 30, 37)):
            s = sides[(j + k) % len(sides)]
            v = 255 if (j + k) & 1 else 0
            img[d:d + s, x:x + s] = v                                  # top: rows d .. d + s - 1
            img[h - d - s:h - d, x + 11:x + 11 + s] = 255 - v          # bottom: rows h-d-s .. h-d-1
        for j, y in enumerate(range(20 + 5 * k, h - 30, 31)):
            s = sides[(j + 2 * k) % len(sides)]
            v = 0 if (j + k) & 1 else 255
            img[y:y + s, d:d + s] = v                                  # left
            img[y + 9:y + 9 + s, w - d - s:w - d] = 255 - v            # right
    for (y, x) in ((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (1, 1), (1, w - 2), (h - 2, 1), (h - 2, w - 2)):
        img[y, x] = 255
    for (y, x) in ((2, 2), (2, w - 3), (h - 3, 2), (h - 3, w - 3)):
        img[y, x] = 0
    # 1-pixel lines: along the outermost and second rows / columns, and one of each in the interior
    img[0, w // 4:w // 4 + 40] = 255
    img[1, w // 2:w // 2 + 40] = 0
    img[h - 1, w // 3:w // 3 + 40] = 0
    img[h - 2, 2 * w // 3:2 * w // 3 + 40] = 255
    img[h // 4:h // 4 + 30, 0] = 0
    img[h // 2:h // 2 + 30, 1] = 255
    img[h // 3:h // 3 + 30, w - 1] = 255
    img[2 * h // 3:2 * h // 3 + 30, w - 2] = 0
    img[h // 2, w // 4:w // 4 + 50] = 255
    img[h // 4:h // 4 + 50, w // 2] = 0
    for (y, x, v) in ((h // 3, w // 3, 255), (h // 3, 2 * w // 3, 0), (2 * h // 3, w // 2, 255), (5, 5, 0), (h - 6, w - 6, 255)):
        img[y, x] = v
    return img


def _step_edges(w, h):
    """a vertical step at x = w/3 and a diagonal step x - y = w/2, each from 0 to 255"""
    y, x = _grid(w, h)
    return (255 * ((x >= w // 3) ^ (x - y >= w // 2))).astype(np.uint8)


def image(name: str, w: int = 0, h: int = 0) -> np.ndarray:
    dw, dh = SIZES[name]
    w, h = w or dw, h or dh
    if name.endswith("_f32"):
        return (image(name[:-4], w, h) == 255).astype(np.float32)           # exactly 0.0 and 1.0
    if name.startswith("checker_rot30_p"):
        return _checker_rot30(w, h, int(name[len("checker_rot30_p"):]))
    if name == "checker_p3_4k":
        return _checker(w, h, 3)
    if name.startswith("checker_p"):
        return _checker(w, h, int(name[len("checker_p"):]))
    if name == "block_noise_4":
        return _binary_noise(w, h, 404, block=4)
    if name == "binary_noise":
        return _binary_noise(w, h, 401)
    if name == "saturated":
        f = make_frame(w, h, 61).astype(np.int32)
        return np.clip((f - 128) * 6 + 128, 0, 255).astype(np.uint8)
    if name == "dark":
        f = make_frame(w, h, 62).astype(np.int32)
        return np.clip((f - 64) // 32, 0, 3).astype(np.uint8)                # values 0 .. 3
    if name == "border_impulses":
        return _border_impulses(w, h)
    if name == "step_edges":
        return _step_edges(w, h)
    if name == "const_0":
        return np.zeros((h, w), np.uint8)
    if name == "const_255":
        return np.full((h, w), 255, np.uint8)
    raise KeyError(name)
