"""Absolute-gradient densification statistic without a GPU: the new kernel's resources and reductions in the built library, the
LGR_DENSIFY_GRAD switches, and the float64 arbiter of absgrad (tests/native/absgrad_host.c) against its definition, the sum over
pixels of |dL/dmean2D| of the C oracle's own blend_backward with dL/dpix kept at one pixel."""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from lightgaussian_b200 import build
from lightgaussian_b200.model import pipeline_params
from lightgaussian_b200.renderer import render
from oracle.lgo import Oracle
from tests.test_depth_alpha_cpu import REDG, _one, _usage
from tests.test_deterministic_sass import CUOBJDUMP, _find, sass  # noqa: F401  (module fixture: the library's SASS by kernel name)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ABS_SRC = os.path.join(ROOT, "tests", "native", "absgrad_host.c")
_abs_lib = []


def _absgrad_lib():
    """tests/native/absgrad_host.c, compiled next to the other host helpers (or in a temporary directory when the tree is read-only)"""
    if not _abs_lib:
        out = os.path.join(ROOT, "tests", "native", "_build")
        try:
            os.makedirs(out, exist_ok=True)
            if not os.access(out, os.W_OK):
                raise OSError(out)
        except OSError:
            out = tempfile.mkdtemp(prefix="absgrad_host_")
        lib = os.path.join(out, "libabsgrad_host.so")
        if not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(ABS_SRC):
            tmp = f"{lib}.tmp{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", ABS_SRC, "-o", tmp, "-lm"])
            os.replace(tmp, lib)
        f = C.CDLL(lib).absgrad_blend_backward
        f.restype = None
        f.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 10
        _abs_lib.append(f)
    return _abs_lib[0]


def absgrad_float64(W, H, P, ranges, point_list, means2D, conic_opacity, colors, bg, final_T, n_contrib, dL_dpix):
    """[P,2] float64: per Gaussian, the sums over the pixels that blend it of |that pixel's dL/dmean2D term|, on the given state"""
    d = lambda a: np.ascontiguousarray(np.asarray(a, np.float64))  # noqa: E731
    u = lambda a: np.ascontiguousarray(np.asarray(a, np.uint32))  # noqa: E731
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    pl = u(point_list) if np.size(point_list) else np.zeros(1, np.uint32)
    arrs = [u(ranges), pl, d(means2D), d(conic_opacity), d(colors), d(bg), d(final_T), u(n_contrib), d(dL_dpix)]
    out = np.zeros((P, 2), np.float64)
    _absgrad_lib()(P, W, H, *[p(a) for a in arrs], p(out))
    return out
ABS = "blend_backward_absgrad_kernel"
DEFAULT = "blend_backward_ring_kernelILb0ELb0E"

# Hopper: 64 K registers, 228 KB of shared memory and 1 KB reserved per block; the default blend backward fits 4 blocks of 288
SM_REGS, SM_SMEM, BLOCK_RESERVED, THREADS = 65536, 228 * 1024, 1024, 288


def _dyn_smem_abs():
    """blend_back_smem_bytes(zero_rows = true, det = false, abs = true) from the layouts in csrc/lgr_blend.cuh"""
    r128 = lambda n: (n + 127) // 128 * 128  # noqa: E731
    ring = 4 * 32 * 12 * 4 + 8 * 4 + 8 * 4 + 4 * 4 + 4 + 4            # BlendRing: records, full/empty barriers, counts, live, tile_max
    warp = 2 * 16 * 33 * 4 + 3 * 16 * 4 + 32 * 16 + 16 * 16          # BlendBackWarp (w, g, mid/mgx/mgy, d) + BlendBackWarpAbs::mco
    return r128(ring) + r128(8 * warp) + 5760                          # + the zero page (KB_ZERO_BYTES)


def _static_smem(name):
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", build.build_library()], check=True, capture_output=True, text=True).stdout
    m = [int(s) for n, s in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:\d+ SHARED:(\d+)", out) if name in n]
    assert len(m) == 1, name
    return m[0]


def test_absgrad_kernel_fits_four_blocks_per_sm_without_spills():
    usage = _usage()
    reg, stack, local = _one(usage, ABS)
    dreg, dstack, _ = _one(usage, DEFAULT)
    assert local == 0, local
    assert reg <= dreg and stack <= dstack, ((reg, stack), (dreg, dstack))
    assert 4 * THREADS * reg <= SM_REGS, reg
    per_block = _static_smem(ABS) + _dyn_smem_abs() + BLOCK_RESERVED
    assert 4 * per_block <= SM_SMEM, per_block


def test_default_kernel_name_is_still_unique():
    _one(_usage(), DEFAULT)


def test_absgrad_flush_uses_vector_reductions(sass):  # noqa: F811
    """words 0-3 and 4-7 with 16-byte reductions, absgrad with one 8-byte reduction per flush site, and no more scalar reductions
    than the default kernel's (word 8)"""
    ops = REDG.findall(sass[_find(sass, ABS)[0]])
    dops = REDG.findall(sass[_find(sass, DEFAULT)[0]])
    sites = dops.count("F32x4") // 2
    assert sites >= 1 and ops.count("F32x4") == 2 * sites and ops.count("F32x2") == sites, (ops, dops)
    assert ops.count("F32") <= dops.count("F32"), (ops, dops)


def _import_dropin(env):
    code = "import gaussian_renderer"
    e = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]), **env)
    return subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, cwd=ROOT)


def test_dropin_refuses_bad_settings_at_import():
    r = _import_dropin({"LGR_DENSIFY_GRAD": "absolute"})
    assert r.returncode != 0 and "LGR_DENSIFY_GRAD='absolute'" in r.stderr, r.stderr[-2000:]
    r = _import_dropin({"LGR_DENSIFY_GRAD": "abs", "LGR_FUSED_OPTIM": "0"})
    assert r.returncode != 0 and "LGR_FUSED_OPTIM=0" in r.stderr, r.stderr[-2000:]
    for v in ("abs", "grad"):
        r = _import_dropin({"LGR_DENSIFY_GRAD": v})
        assert r.returncode == 0, r.stderr[-2000:]


def _cpu_model():
    P = 4
    z = lambda *s: torch.zeros(*s)  # noqa: E731
    return SimpleNamespace(_xyz=z(P, 3), _features_dc=z(P, 1, 3), _features_rest=z(P, 15, 3), _scaling=z(P, 3), _rotation=z(P, 4),
                           _opacity=z(P, 1), active_sh_degree=3, max_sh_degree=3)


def test_render_refuses_before_reading_the_camera(monkeypatch):
    cam = object()    # any read of the camera would fail with AttributeError
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    with pytest.raises(RuntimeError, match="LGR_DENSIFY_GRAD=abs needs the fused path"):
        render(cam, _cpu_model(), pipeline_params(), None)
    with pytest.raises(RuntimeError, match="render\\(depth=..., alpha=...\\)"):
        render(cam, _cpu_model(), pipeline_params(), None, alpha=True)
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "l1")
    with pytest.raises(RuntimeError, match="LGR_DENSIFY_GRAD='l1'"):
        render(cam, _cpu_model(), pipeline_params(), None)


def test_add_densification_stats_raises_without_absgrad(monkeypatch):
    from lightgaussian_b200 import densify
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "abs")
    g = SimpleNamespace(xyz_gradient_accum=torch.zeros(4, 1), denom=torch.zeros(4, 1))
    vp = torch.zeros(4, 3, requires_grad=True)
    with pytest.raises(RuntimeError, match="no .absgrad"):
        densify.add_densification_stats(g, vp, torch.ones(4, dtype=torch.bool))
    monkeypatch.setenv("LGR_DENSIFY_GRAD", "sum")
    with pytest.raises(RuntimeError, match="LGR_DENSIFY_GRAD='sum'"):
        densify.add_densification_stats(g, vp, torch.ones(4, dtype=torch.bool))


# ------------------------------------------------------------------------------------------------
# the float64 arbiter against its definition
# ------------------------------------------------------------------------------------------------
def _needles(raw, k):
    raw = dict(raw)
    s = raw["scaling"].copy()
    s[:k, 0] += 3.0
    s[:k, 1:] -= 2.5
    raw["scaling"] = s
    return raw


@pytest.mark.parametrize("P,W,H,needles", [(1, 8, 6, 0), (40, 17, 5, 0), (300, 24, 16, 60), (120, 33, 18, 120)])
def test_float64_absgrad_is_the_sum_of_one_pixel_backwards(P, W, H, needles):
    from lightgaussian_b200.synth import make_cameras, make_scene
    from tests.util import activate, view_from_camera
    o = Oracle(double=True)
    scene = make_scene(P, sh_degree=3, seed=40 + P, scale_mult=4.0)
    raw = _needles(scene["raw"], needles)
    act = activate(raw, 3)
    view = view_from_camera(make_cameras(3, W, H)[1], (0.1, 0.2, 0.3), 3, 1.0)
    geom = o.preprocess(view, act["means3D"], act["opacities"], act["shs"], None, act["scales"], act["rotations"])
    point_list, ranges = o.bin(view, geom["means2D"], geom["depths"], geom["radii"], geom["tiles_touched"])
    fwd = o.blend_forward(view, ranges, point_list, geom["means2D"], geom["rgb"], geom["conic_opacity"])
    assert np.any(fwd["n_contrib"] > 0)
    dpix = np.random.default_rng(P).standard_normal((3, H, W))
    args = (view, P, ranges, point_list, geom["means2D"], geom["conic_opacity"], geom["rgb"], fwd["final_T"], fwd["n_contrib"])
    ag = absgrad_float64(W, H, P, ranges, point_list, geom["means2D"], geom["conic_opacity"], geom["rgb"], view.bg, fwd["final_T"],
                         fwd["n_contrib"], dpix)
    total = np.zeros((P, 2))
    for py in range(H):
        for px in range(W):
            one = np.zeros_like(dpix)
            one[:, py, px] = dpix[:, py, px]
            total += np.abs(o.blend_backward(*args, one)["dL_dmean2D"])
    assert np.any(total > 0)
    np.testing.assert_allclose(ag, total, rtol=1e-12, atol=0)
