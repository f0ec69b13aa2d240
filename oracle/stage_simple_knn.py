#!/usr/bin/env python
"""Stage the reference's UNMODIFIED simple-knn extension (submodules/simple-knn: spatial.cu + simple_knn.cu + ext.cpp, pybind module
`simple_knn._C`, distCUDA2) into the stock stack, oracle/_ref/stock/simple_knn (never committed), so that the stock stack runs the
reference's own distCUDA2.  Run after oracle/stage_reference.py; needs the reference checkout ($REFERENCE, default /root/reference),
without it this does nothing.

    python oracle/stage_simple_knn.py [--force]

  * installed like the rasterizer extension, from a temporary copy (the build writes into its source tree):
        TORCH_CUDA_ARCH_LIST=9.0a NVCC_APPEND_FLAGS="-include cfloat" \\
        pip install --no-index --no-build-isolation --no-deps --target oracle/_ref/stock <copy of submodules/simple-knn>
    `-include cfloat` because simple_knn.cu uses FLT_MAX without <cfloat>, which nvcc 12.9 rejects at lines 90 and 154;
  * the installed directory holds only the extension module, so it is made a regular package (an empty __init__.py): a namespace
    directory would lose to any regular `simple_knn` package later on the stock stack's path;
  * the copy of this repository's drop-in that oracle/stage_reference.py places in oracle/_ref/stock/shims/simple_knn is removed:
    the stock stack must not reach our distCUDA2;
  * a failed build raises, so build() stops instead of leaving a stock stack without the reference's distCUDA2.
"""
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REFERENCE", "/root/reference")
SKNN = os.path.join(REF, "submodules", "simple-knn")
OUT = os.path.join(ROOT, "oracle", "_ref", "stock")
PKG = os.path.join(OUT, "simple_knn")


def built() -> bool:
    return os.path.isdir(PKG) and any(f.startswith("_C") and f.endswith(".so") for f in os.listdir(PKG))


def main(force=False):
    if not os.path.isdir(SKNN):
        print(f"stage_simple_knn: no reference checkout at {REF}: nothing staged")
        return 0
    status = "present"
    if force or not built():
        os.makedirs(OUT, exist_ok=True)
        with tempfile.TemporaryDirectory() as work:
            tmp = os.path.join(work, "simple-knn")
            shutil.copytree(SKNN, tmp)
            env = dict(os.environ, TORCH_CUDA_ARCH_LIST="9.0a", NVCC_APPEND_FLAGS="-include cfloat", MAX_JOBS="6", FORCE_CUDA="1")
            cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--upgrade", "--target", OUT, tmp]
            subprocess.check_call(cmd, env=env)
        if not built():
            raise RuntimeError(f"stage_simple_knn: building {SKNN} left no simple_knn/_C*.so under {OUT}")
        status = "built"
    init = os.path.join(PKG, "__init__.py")
    if not os.path.exists(init):
        open(init, "w").close()
    shutil.rmtree(os.path.join(OUT, "shims", "simple_knn"), ignore_errors=True)
    print("simple-knn:", status, PKG)
    return 0


if __name__ == "__main__":
    sys.exit(main(force="--force" in sys.argv))
