"""Deterministic mode (CPU check of the built library): the kernels it launches contain no floating-point ATOM / RED instructions.
Integer atomics (the reached-instance bitmap, ballot counters) are fine.  The default blend backward and VecTree accumulation kernels
still contain theirs, which shows the check can fail."""
import os
import re
import shutil
import subprocess

import pytest

from lightgaussian_b200 import build

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
FLOAT_ATOMIC = re.compile(r"\b(?:ATOM|RED)[GS]?\.[A-Z0-9_.]*\bF(?:16|32|64)\b|\b(?:ATOM|RED)[GS]?\.[A-Z0-9_.]*\.F(?:16|32|64)")

DETERMINISTIC = ("blend_backward_ring_kernelILb1E", "det_gather_kernel", "det_iota_kernel", "det_point_list_kernel",
                 "vq_det_keys_kernel", "vq_det_segsum_kernel", "blend_forward_ring_kernelILb0ELb1ELb1E")
DEFAULT_WITH_FLOAT_ATOMICS = ("blend_backward_ring_kernelILb0E", "vq_accumulate_kernel")


@pytest.fixture(scope="module")
def sass():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    lib = build.build_library()
    out = subprocess.run([CUOBJDUMP, "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = chunk.split("\n", 1)
        funcs[name.strip()] = body
    return funcs


def _find(funcs, key):
    hits = [n for n in funcs if key in n]
    assert hits, f"no kernel matching {key} in the library"
    return hits


def _float_atomics(body):
    return [m.group(0) for m in FLOAT_ATOMIC.finditer(body)]


@pytest.mark.parametrize("key", DETERMINISTIC)
def test_deterministic_kernels_have_no_float_atomics(sass, key):
    for name in _find(sass, key):
        assert not _float_atomics(sass[name]), f"{name}: {sorted(set(_float_atomics(sass[name])))}"


@pytest.mark.parametrize("key", DEFAULT_WITH_FLOAT_ATOMICS)
def test_default_kernels_still_have_theirs(sass, key):
    assert any(_float_atomics(sass[name]) for name in _find(sass, key))
