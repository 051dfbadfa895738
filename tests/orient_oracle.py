"""ctypes binding of tests/orient_oracle.c -- TEST INFRASTRUCTURE: the CPU oracle's orientation stage alone, on
caller-given keypoints, for an oracle_lib.Oracle that has run at least its pyramid stage.

The library is compiled on first use with the oracle's flags (oracle/Makefile) into a per-user temporary directory,
keyed by the hash of its sources, so that a read-only checkout works too."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "orient_oracle.c")
DEPS = [SRC, os.path.join(HERE, "..", "oracle", "sift_oracle.c"), os.path.join(HERE, "..", "oracle", "sift_oracle.h")]
CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-frounding-math", "-fno-fast-math", "-fopenmp", "-shared"]

_lib = None


def _cc():
    return "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for p in DEPS:
            with open(p, "rb") as f:
                h.update(f.read())
        out_dir = os.path.join(tempfile.gettempdir(), "popsift_b200_orient_oracle_%d" % os.getuid())
        os.makedirs(out_dir, exist_ok=True)
        path = os.path.join(out_dir, "liborient_oracle_%s.so" % h.hexdigest()[:16])
        if not os.path.exists(path):
            tmp = path + ".%d.tmp" % os.getpid()
            subprocess.check_call([_cc()] + CFLAGS + ["-o", tmp, SRC, "-lm"])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_orient.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def orient(oracle, x, y, sigma, octave, lpos):
    """(num_ori [n], angles [n, 4], unused 0) of the given keypoints (octave-local x, y, sigma; octave and lpos) on the
    pyramid of `oracle` (an oracle_lib.Oracle after run()): the oracle's orientation stage alone"""
    kp = np.ascontiguousarray(np.stack([x, y, sigma], 1), dtype=np.float32)
    ol_ = np.ascontiguousarray(np.stack([octave, lpos], 1), dtype=np.int32)
    num = np.zeros(len(kp), dtype=np.int32)
    ori = np.zeros((len(kp), 4), dtype=np.float32)
    if len(kp):
        assert lib().orc_orient(oracle.ctx, len(kp), kp.ctypes.data, ol_.ctypes.data, num.ctypes.data, ori.ctypes.data) == 0
    return num, ori
