"""Densification of GaussianModel (scene/gaussian_model.py:602-788) on the native kernels of csrc/lgr_densify.cuh, bit-identical to
the reference's torch code on the same state and random-number generator:

  add_densification_stats   xyz_gradient_accum[f] += ||grad[f, :2]||, denom[f] += 1 in one launch, with no host synchronisation.
  densify_and_prune         clone + split + prune in one plan (one host synchronisation for the three counts) and one pass that
                            writes the 6 parameters, 12 Adam moments and 3 auxiliary buffers; the reference rebuilds all 18 optimizer
                            tensors four times with torch.cat / boolean indexing.  The split children's samples are drawn through
                            torch's generator as the reference draws them: 2S x 3 normals, including those of children pruned later.

The one operation not in these kernels is the split's batched 3x3 . 3x1 product, which runs as torch.bmm on the reference's own
operands: no fixed operation order reproduces cuBLAS's result on every sample.

Inputs the kernels do not take (CPU or non-float32 tensors, a missing gradient, unexpected optimizer groups) go to the class's own method.  `install(GaussianModel)` makes the class use these two functions (optim.install calls it)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import capi, trace
from .optim import _GROUP_ATTR

_ROLE = {"xyz": capi.DENSIFY_XYZ, "scaling": capi.DENSIFY_SCALING}
_ROW_SHAPE = {"xyz": (3,), "scaling": (3,), "rotation": (4,), "opacity": (1,)}


def _original(gaussians, name):
    m = getattr(type(gaussians), name)
    return getattr(m, "__wrapped__", m)


def _f32(x) -> float:
    """a Python scalar as torch compares it with a float32 tensor: rounded to float32"""
    return float(np.float32(x))


def _f32_cuda(t, device, shape) -> bool:
    return (isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dtype == torch.float32
            and tuple(t.shape) == tuple(shape))


def _dense_f32(t, device, shape) -> bool:
    return _f32_cuda(t, device, shape) and t.is_contiguous()


def add_densification_stats(gaussians, viewspace_point_tensor, update_filter):
    """GaussianModel.add_densification_stats (:784-788)"""
    grad = getattr(viewspace_point_tensor, "grad", None)
    accum, denom = getattr(gaussians, "xyz_gradient_accum", None), getattr(gaussians, "denom", None)
    P = accum.shape[0] if isinstance(accum, torch.Tensor) else -1
    device = grad.device if isinstance(grad, torch.Tensor) else None
    if not (isinstance(grad, torch.Tensor) and grad.is_cuda and grad.dtype == torch.float32 and grad.dim() == 2 and grad.shape[0] == P
            and grad.shape[1] >= 2 and grad.stride(1) == 1 and grad.stride(0) >= 2
            and isinstance(update_filter, torch.Tensor) and update_filter.dtype == torch.bool and update_filter.device == device
            and update_filter.is_contiguous() and tuple(update_filter.shape) == (P,)
            and _dense_f32(accum, device, (P, 1)) and _dense_f32(denom, device, (P, 1))):
        return _original(gaussians, "add_densification_stats")(gaussians, viewspace_point_tensor, update_filter)
    trace.bump("densify_stats_native")
    lib = capi.load()
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats(P, grad.data_ptr(), grad.stride(0), update_filter.data_ptr(), accum.data_ptr(), denom.data_ptr(),
                                         capi.current_stream_ptr(device)), "lgr_densify_stats")


def _groups(gaussians):
    """[(group, name, param, state or None)] when every tensor densify_and_prune rewrites is one the kernels take, else None"""
    opt = getattr(gaussians, "optimizer", None)
    xyz = getattr(gaussians, "_xyz", None)
    if opt is None or not isinstance(xyz, torch.Tensor) or xyz.dim() != 2:
        return None
    P, device = xyz.shape[0], xyz.device
    out = []
    for group in opt.param_groups:
        name = group.get("name")
        if name not in _GROUP_ATTR or len(group["params"]) != 1:
            return None
        p = group["params"][0]
        if p is not getattr(gaussians, _GROUP_ATTR[name]):
            return None
        if not _f32_cuda(p, device, (P,) + tuple(_ROW_SHAPE.get(name, p.shape[1:]))):
            return None
        st = opt.state.get(p, None)
        if st is not None and not all(_f32_cuda(st.get(k), device, p.shape) for k in ("exp_avg", "exp_avg_sq")):
            return None
        out.append((group, name, p, st))
    if sorted(n for _, n, _, _ in out) != sorted(_GROUP_ATTR):
        return None
    if not (_dense_f32(getattr(gaussians, "xyz_gradient_accum", None), device, (P, 1)) and _dense_f32(gaussians.denom, device, (P, 1))
            and _dense_f32(getattr(gaussians, "max_radii2D", None), device, (P,))):
        return None
    return out


def densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size):
    """GaussianModel.densify_and_prune (:745-761): densify_and_clone, densify_and_split, then the opacity / size prune"""
    groups = _groups(gaussians)
    if groups is None:
        return _original(gaussians, "densify_and_prune")(gaussians, max_grad, min_opacity, extent, max_screen_size)
    trace.bump("densify_native")
    lib = capi.load()
    opt = gaussians.optimizer
    # any layout is read (torch.cat writes the reference's results row-major whatever its inputs' layout)
    leaf = {name: p.detach().contiguous() for _, name, p, _ in groups}
    P, device = leaf["xyz"].shape[0], leaf["xyz"].device
    # densification_postfix has just zeroed max_radii2D when the reference evaluates big_points_vs = max_radii2D > max_screen_size
    prune_all = bool(max_screen_size) and 0.0 > float(max_screen_size)
    with torch.cuda.device(device):
        stream = capi.current_stream_ptr(device)
        ws = torch.empty((int(lib.lgr_densify_workspace_bytes(P)),), dtype=torch.uint8, device=device)
        counts = (C.c_int32 * 4)()
        capi.check(lib.lgr_densify_plan(P, gaussians.xyz_gradient_accum.data_ptr(), gaussians.denom.data_ptr(), leaf["scaling"].data_ptr(),
                                        leaf["opacity"].data_ptr(), _f32(max_grad), _f32(gaussians.percent_dense * extent), _f32(min_opacity),
                                        _f32(0.1 * extent), int(prune_all), int(bool(max_screen_size)), ws.data_ptr(), ws.numel(), counts,
                                        stream), "lgr_densify_plan")
        kept, clones, children, splits = (int(c) for c in counts)
        # torch.normal(mean=zeros, std) is normal_(0, 1), then mul_(std), add_(mean): the kernel applies n * std + 0.  Drawn even for
        # children pruned later, and when S = 0, as the reference draws them.
        normals = torch.empty((2 * splits, 3), dtype=torch.float32, device=device).normal_(0, 1)
        offsets = None
        if splits:
            rots = torch.empty((2 * splits, 3, 3), dtype=torch.float32, device=device)
            samples = torch.empty((2 * splits, 3, 1), dtype=torch.float32, device=device)
            capi.check(lib.lgr_densify_split_inputs(P, ws.data_ptr(), counts, leaf["scaling"].data_ptr(), leaf["rotation"].data_ptr(),
                                                    normals.data_ptr(), rots.data_ptr(), samples.data_ptr(), stream), "lgr_densify_split_inputs")
            # no fixed order of this 3x3 . 3x1 product reproduces cuBLAS's on every sample: the same torch.bmm on the same operands does
            offsets = torch.bmm(rots, samples)
        rows = kept + clones + 2 * children
        jobs = []          # (src or None, dst, role)
        for _, name, p, st in groups:
            dst = torch.empty((rows,) + tuple(p.shape[1:]), dtype=torch.float32, device=device)
            jobs.append((leaf[name], dst, _ROLE.get(name, capi.DENSIFY_COPY)))
            if st is not None:
                jobs += [(st[k].contiguous(), torch.empty_like(dst), capi.DENSIFY_MOMENT) for k in ("exp_avg", "exp_avg_sq")]
        aux = {"xyz_gradient_accum": (rows, 1), "denom": (rows, 1), "max_radii2D": (rows,)}
        for shape in aux.values():
            jobs.append((None, torch.empty(shape, dtype=torch.float32, device=device), capi.DENSIFY_ZERO))
        arr = (capi.LgrDensifyTensor * len(jobs))()
        for a, (src, dst, role) in zip(arr, jobs):
            a.src = src.data_ptr() if src is not None and src.numel() else None
            a.dst = dst.data_ptr() if dst.numel() else None
            a.role, a.row_words = role, int(np.prod(dst.shape[1:], dtype=np.int64))     # 0 for _features_rest at SH degree 0: skipped
        if rows:
            capi.check(lib.lgr_densify_rows(P, ws.data_ptr(), counts, leaf["xyz"].data_ptr(), offsets.data_ptr() if splits else None,
                                            len(jobs), arr, stream), "lgr_densify_rows")
    outs = iter(dst for _, dst, _ in jobs)
    for group, name, old, st in groups:
        new = torch.nn.Parameter(next(outs).requires_grad_(True))
        if st is not None:
            st["exp_avg"], st["exp_avg_sq"] = next(outs), next(outs)
            del opt.state[old]
            opt.state[new] = st
        group["params"][0] = new
        setattr(gaussians, _GROUP_ATTR[name], new)
    for n in aux:
        setattr(gaussians, n, next(outs))
    torch.cuda.empty_cache()


def install(GaussianModel):
    """Replace the class's add_densification_stats / densify_and_prune by the functions above; the originals stay reachable as
    `__wrapped__` and take the inputs the kernels do not.  Idempotent."""
    if getattr(GaussianModel, "_lgr_native_densify", False):
        return GaussianModel
    for name, fn in (("add_densification_stats", add_densification_stats), ("densify_and_prune", densify_and_prune)):
        original = getattr(GaussianModel, name)

        def method(self, *args, _fn=fn, **kwargs):
            return _fn(self, *args, **kwargs)

        method.__wrapped__ = original
        method.__name__ = name
        setattr(GaussianModel, name, method)
    GaussianModel._lgr_native_densify = True
    return GaussianModel
