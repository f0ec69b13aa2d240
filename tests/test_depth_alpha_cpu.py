"""Depth and alpha planes without a GPU: the new kernel instantiations in the built library (vector reductions, no spills, registers
no higher than the default kernels'), and the keyword checks of render() that refuse a request before anything is read."""
import re
import subprocess
from types import SimpleNamespace

import pytest
import torch

from lightgaussian_b200 import build
from lightgaussian_b200.model import pipeline_params
from lightgaussian_b200.renderer import render
from tests.test_deterministic_sass import CUOBJDUMP, _find, sass  # noqa: F401  (module fixture: the library's SASS by kernel name)

REDG = re.compile(r"\bREDG\.E\.ADD\.(F32x4|F32x2|F32)\.")


def _usage():
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", build.build_library()], check=True, capture_output=True, text=True).stdout
    return {n: (int(r), int(s), int(loc)) for n, r, s, loc in
            re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}


def _one(usage, key):
    names = [n for n in usage if key in n]
    assert len(names) == 1, (key, sorted(usage))
    return usage[names[0]]


# (depth variant, the default kernel it extends)
PAIRS = [("blend_forward_ring_kernelILb0ELb1ELb0ELb0ELb1E", "blend_forward_ring_kernelILb0ELb1ELb0ELb0ELb0E"),
         ("blend_backward_ring_kernelILb0ELb1E", "blend_backward_ring_kernelILb0ELb0E"),
         ("preprocess_backward_raw_depth_kernel", "preprocess_backward_raw_kernel"),
         ("preprocess_backward_compact_depth_kernel", "preprocess_backward_compact_kernel"),
         ("kback_zero_flag_depth_kernelILb1E", "kback_zero_flag_kernelILb1E"),
         ("kback_zero_flag_depth_kernelILb0E", "kback_zero_flag_kernelILb0E")]


@pytest.mark.parametrize("depth,default", PAIRS)
def test_depth_kernels_do_not_spill(depth, default):
    usage = _usage()
    reg, stack, local = _one(usage, depth)
    dreg, dstack, _ = _one(usage, default)
    assert local == 0, (depth, local)
    assert stack <= dstack and reg <= dreg, (depth, (reg, stack), default, (dreg, dstack))


def test_depth_blend_backward_adds_word_9_with_word_8(sass):  # noqa: F811
    """the flush adds words 0-3 and 4-7 with two 16-byte reductions and words 8-9 with one 8-byte reduction: no scalar reduction"""
    body = sass[_find(sass, "blend_backward_ring_kernelILb0ELb1E")[0]]
    ops = REDG.findall(body)
    assert ops.count("F32") == 0, ops
    assert ops.count("F32x4") >= 2 and ops.count("F32x2") * 2 == ops.count("F32x4"), ops


def test_depth_forward_has_no_atomics(sass):  # noqa: F811
    body = sass[_find(sass, "blend_forward_ring_kernelILb0ELb1ELb0ELb0ELb1E")[0]]
    assert not REDG.search(body) and "ATOMG" not in body


def _cpu_model():
    P = 4
    z = lambda *s: torch.zeros(*s)  # noqa: E731
    return SimpleNamespace(_xyz=z(P, 3), _features_dc=z(P, 1, 3), _features_rest=z(P, 15, 3), _scaling=z(P, 3), _rotation=z(P, 4),
                           _opacity=z(P, 1), active_sh_degree=3, max_sh_degree=3)


def test_render_refuses_before_reading_the_camera():
    cam = object()    # any read of the camera would fail with AttributeError
    with pytest.raises(RuntimeError, match="expected None, 'z' or 'inverse'"):
        render(cam, _cpu_model(), pipeline_params(), None, depth="disparity")
    with pytest.raises(RuntimeError, match="override_color"):
        render(cam, _cpu_model(), pipeline_params(), None, override_color=torch.zeros(4, 3), alpha=True)
    with pytest.raises(RuntimeError, match="convert_SHs_python"):
        render(cam, _cpu_model(), pipeline_params(convert_SHs_python=True), None, depth="z")
    with pytest.raises(RuntimeError, match="raw float32 CUDA leaves"):   # CPU leaves: not the fused path
        render(cam, _cpu_model(), pipeline_params(), None, depth="inverse")
