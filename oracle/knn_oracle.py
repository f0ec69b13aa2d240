"""Python binding of oracle/knn_oracle.c, the brute-force CPU restatement of the reference's distCUDA2 (TEST INFRASTRUCTURE ONLY).
The shared library is compiled with gcc into oracle/_build/ by build() (called from __graft_entry__.build(), or on first use)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "knn_oracle.c")
LIB = os.path.join(_HERE, "_build", "libknn_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    """Compile libknn_oracle.so with the flags oracle/Makefile uses for lgo.c (no contraction, no fast math)."""
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        tmp = LIB + f".tmp{os.getpid()}"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", tmp,
                               SRC, "-lm"])
        os.replace(tmp, LIB)
    return LIB


def knn_mean_dist3(points) -> np.ndarray:
    """distCUDA2 of submodules/simple-knn, brute force: float32 [P,3] -> float32 [P].  O(P^2): meant for P up to ~20 000."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.lgo_knn_mean_dist3.restype = None
        _lib.lgo_knn_mean_dist3.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    pts = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    out = np.empty(pts.shape[0], np.float32)
    _lib.lgo_knn_mean_dist3(pts.shape[0], pts.ctypes.data, out.ctypes.data)
    return out
