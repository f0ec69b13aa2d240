"""In-tree build of liblgrast.so (nvcc, sm_90a).  No JIT cache: the .so lives next to the sources, so a tree built once (on a
machine without a GPU, too) runs anywhere it is copied."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "_lib")
LIB_PATH = os.path.join(LIB_DIR, "liblgrast.so")
SOURCES = ["lgrast.cu"]
# every header under csrc/ (a header missing from this list once let an edited kernel run as its previous binary) + the C-ABI header
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [os.path.join("..", "..", "include", "lgrast.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
]


HASH_PATH = LIB_PATH + ".srchash"


def _source_hash() -> str:
    """content hash of every source/header and the compiler flags (mtimes do not survive a copy of the tree)"""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for d in sorted(os.path.join(CSRC, s) for s in SOURCES + HEADERS):
        if os.path.exists(d):
            with open(d, "rb") as f:
                h.update(os.path.basename(d).encode() + b"\0" + f.read())
    return h.hexdigest()


def _stale() -> bool:
    """True when liblgrast.so is missing or was not built from the sources as they are now."""
    if not os.path.exists(LIB_PATH) or not os.path.exists(HASH_PATH):
        return True
    with open(HASH_PATH) as f:
        return f.read().strip() != _source_hash()


def have_nvcc() -> bool:
    return bool(shutil.which("nvcc")) or os.path.exists("/usr/local/cuda/bin/nvcc")


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/lgrast.cu into _lib/liblgrast.so if missing or stale.  Returns the path."""
    if not force and not _stale():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build liblgrast.so (and there is no CPU fallback)")
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = LIB_PATH + f".tmp{os.getpid()}"
    cmd = [nvcc] + NVCC_FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", tmp]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    digest = _source_hash()
    subprocess.check_call(cmd)
    os.replace(tmp, LIB_PATH)
    with open(HASH_PATH + ".tmp", "w") as f:
        f.write(digest + "\n")
    os.replace(HASH_PATH + ".tmp", HASH_PATH)
    return LIB_PATH
