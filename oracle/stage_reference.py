#!/usr/bin/env python
"""Stage the UNMODIFIED reference under oracle/_ref/stock (never committed), next to the reference kernels that oracle/Makefile builds, so
that test-only builds of the reference live in one place.  Needs the reference checkout ($REFERENCE, default /root/reference); without it
this does nothing.

    python oracle/stage_reference.py [--force]

Produces, all under oracle/_ref/stock/:

  diff_gaussian_rasterization/   the reference's own torch extension (RAST/setup.py: rasterize_points.cu + ext.cpp + cuda_rasterizer/*,
                                 pybind module `_C`), installed with
                                     TORCH_CUDA_ARCH_LIST=9.0a NVCC_APPEND_FLAGS="-include cstdint" \
                                     pip install --no-index --no-build-isolation --no-deps --target oracle/_ref/stock <copy of RAST>
                                 (from a temporary copy: the build writes into its source tree and the reference checkout may be read-only;
                                  `-include cstdint` because rasterizer_impl.h forgets that header under gcc 13)
  LightGaussian/                 the reference's Python tree, copied verbatim: the training / pruning / rendering scripts and the
                                 packages they import (scene, utils, arguments, gaussian_renderer, vectree, lpipsPyTorch)
  shims/                         copies of this repository's three offline stand-ins (icecream, plyfile, simple_knn) for the STOCK
                                 stack, which must not see dropin/ (that would swap in our renderer)

Two stacks are then runnable (tests/test_gpu_scripts.py, bench.py --impl reference):
  ours   PYTHONPATH = <repo>/dropin : <repo> : oracle/_ref/stock/LightGaussian
  stock  PYTHONPATH = oracle/_ref/stock : oracle/_ref/stock/shims : oracle/_ref/stock/LightGaussian
"""
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REFERENCE", "/root/reference")
RAST = os.path.join(REF, "submodules", "compress-diff-gaussian-rasterization")
OUT = os.path.join(ROOT, "oracle", "_ref", "stock")

PY_DIRS = ["scene", "utils", "arguments", "gaussian_renderer", "vectree", "lpipsPyTorch"]
PY_FILES = ["prune_finetune.py", "distill_train.py", "prune.py", "render.py", "render_video.py", "train_densify_prune.py", "metrics.py"]


def stage_extension(force=False):
    so_dir = os.path.join(OUT, "diff_gaussian_rasterization")
    if not force and os.path.isdir(so_dir) and any(f.startswith("_C") and f.endswith(".so") for f in os.listdir(so_dir)):
        return "present"
    with tempfile.TemporaryDirectory() as work:
        tmp = os.path.join(work, "RAST")
        shutil.copytree(RAST, tmp)
        env = dict(os.environ, TORCH_CUDA_ARCH_LIST="9.0a", NVCC_APPEND_FLAGS="-include cstdint", MAX_JOBS="6", FORCE_CUDA="1")
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--upgrade", "--target", OUT, tmp]
        subprocess.check_call(cmd, env=env)
    return "built"


def stage_python_tree():
    dst = os.path.join(OUT, "LightGaussian")
    shutil.rmtree(dst, ignore_errors=True)
    os.makedirs(dst)
    ignore = shutil.ignore_patterns("__pycache__", "*.pyc", "*.so", "*.pth", "*.png", "*.jpg")
    for d in PY_DIRS:
        shutil.copytree(os.path.join(REF, d), os.path.join(dst, d), ignore=ignore)
    for f in PY_FILES:
        shutil.copy2(os.path.join(REF, f), os.path.join(dst, f))
    return dst


def stage_shims():
    dst = os.path.join(OUT, "shims")
    shutil.rmtree(dst, ignore_errors=True)
    os.makedirs(dst)
    drop = os.path.join(ROOT, "dropin")
    shutil.copy2(os.path.join(drop, "icecream.py"), dst)
    shutil.copy2(os.path.join(drop, "plyfile.py"), dst)
    shutil.copytree(os.path.join(drop, "simple_knn"), os.path.join(dst, "simple_knn"), ignore=shutil.ignore_patterns("__pycache__"))
    return dst


def main(force=False):
    if not os.path.isdir(RAST):
        print(f"stage_reference: no reference checkout at {REF}: nothing staged")
        return 0
    os.makedirs(OUT, exist_ok=True)
    print("extension:", stage_extension(force))
    print("python tree:", stage_python_tree())
    print("shims:", stage_shims())
    return 0


if __name__ == "__main__":
    sys.exit(main(force="--force" in sys.argv))
