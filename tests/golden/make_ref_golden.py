"""Generates tests/golden/ref_<config>.npz: outputs of the REFERENCE'S OWN CUDA kernels
(oracle/_ref/libref_rasterizer.so, compiled unmodified from /root/reference by oracle/Makefile) on the seeded
inputs of tests/util.py:CONFIGS.  Needs a GPU:

    python tests/golden/make_ref_golden.py <out dir>    # then copy the .npz into tests/golden/

The inputs are NOT stored (they are regenerated from the seed); a checksum guards against generator drift.
"""
import hashlib
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.util import CONFIGS, make_config, run_ref  # noqa: E402


def checksum(act, dpix):
    c = 0
    for k in sorted(act):
        c = zlib.crc32(np.ascontiguousarray(act[k]).tobytes(), c)
    return zlib.crc32(dpix.tobytes(), c)


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for name in CONFIGS:
        act, view, dpix = make_config(name)
        fwd = run_ref(view, act, dL_dpix=dpix)
        cnt = run_ref(view, act, count=True)
        d = dict(input_crc=np.uint32(checksum(act, dpix)), num_rendered=np.int64(fwd["num_rendered"]), color=fwd["color"],
                 radii=fwd["radii"], final_T=fwd["final_T"], n_contrib=fwd["n_contrib"], point_list=fwd["point_list"],
                 ranges=fwd["ranges"], ref_racy_count=cnt["gaussians_count"], ref_racy_score=cnt["important_score"],
                 count_color_sha256=np.frombuffer(hashlib.sha256(np.ascontiguousarray(cnt["color"]).tobytes()).digest(), np.uint8))
        for k, v in fwd["geom"].items():
            d["geom_" + k] = v
        for k, v in fwd["grads"].items():
            d["grad_" + k] = v
        path = os.path.join(out_dir, f"ref_{name}.npz")
        np.savez_compressed(path, **d)
        print(name, "R", fwd["num_rendered"], "visible", int((fwd["radii"] > 0).sum()), os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "golden_out"))
