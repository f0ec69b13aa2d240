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

from . import capi, rasterizer, trace
from .optim import _GROUP_ATTR
from .renderer import densify_grad_mode

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
    """GaussianModel.add_densification_stats (:784-788).  With the view-parallel densification exchange on
    (parallel.enable_gradient_exchange(world > 1, densification=True)) it adds every rank's view of the step, in rank order, on every
    rank: from the slots of the step's sparse exchange when its backward published them, else through one all-gather.
    With LGR_DENSIFY_GRAD=abs (read at each call) it adds ||absgrad[f]|| instead, from the `absgrad` [P,2] that render()'s backward
    set on the tensor; it raises where that statistic is missing or cannot be added natively (no fall-back to the class's method)."""
    if densify_grad_mode() == "abs":
        _add_absgrad_stats(gaussians, viewspace_point_tensor, update_filter)
        return
    grad = getattr(viewspace_point_tensor, "grad", None)
    accum, denom = getattr(gaussians, "xyz_gradient_accum", None), getattr(gaussians, "denom", None)
    P = accum.shape[0] if isinstance(accum, torch.Tensor) else -1
    device = grad.device if isinstance(grad, torch.Tensor) else None
    exchanged = rasterizer.densification_exchange()
    if not (isinstance(grad, torch.Tensor) and grad.is_cuda and grad.dtype == torch.float32 and grad.dim() == 2 and grad.shape[0] == P
            and grad.shape[1] >= 2 and grad.stride(1) == 1 and grad.stride(0) >= 2
            and isinstance(update_filter, torch.Tensor) and update_filter.dtype == torch.bool and update_filter.device == device
            and update_filter.is_contiguous() and tuple(update_filter.shape) == (P,)
            and _dense_f32(accum, device, (P, 1)) and _dense_f32(denom, device, (P, 1))):
        if exchanged:   # the class's own method would add this rank's view only: the replicas would take different decisions
            raise RuntimeError("view-parallel densification needs a float32 CUDA view-space gradient [P,>=2], a contiguous bool filter [P] "
                               "and float32 [P,1] xyz_gradient_accum / denom on the same device")
        return _original(gaussians, "add_densification_stats")(gaussians, viewspace_point_tensor, update_filter)
    if exchanged:
        ex = rasterizer._exchange
        rec, ex["stats_record"] = ex["stats_record"], None
        if rec is not None and rec["P"] == P and rec["device"] == device:
            xs = rec["xs"]
            stats_exchanged(xs, rec["k"], xs.rank, rec["serial"], ex["world"], grad, update_filter, accum, denom)
        else:
            stats_allgather(grad, update_filter, accum, denom, ex["world"], ex["group"])
        return
    trace.bump("densify_stats_native")
    lib = capi.load()
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats(P, grad.data_ptr(), grad.stride(0), update_filter.data_ptr(), accum.data_ptr(), denom.data_ptr(),
                                         capi.current_stream_ptr(device)), "lgr_densify_stats")


def _add_absgrad_stats(gaussians, viewspace_point_tensor, update_filter):
    """xyz_gradient_accum[f] += ||absgrad[f]||, denom[f] += 1 through lgr_densify_stats (row stride 2)"""
    absgrad = getattr(viewspace_point_tensor, "absgrad", None)
    if absgrad is None:
        raise RuntimeError("LGR_DENSIFY_GRAD=abs: the view-space tensor has no .absgrad; render it with LGR_DENSIFY_GRAD=abs set and "
                           "gradients enabled, and call backward first")
    if rasterizer.densification_exchange():
        raise RuntimeError("LGR_DENSIFY_GRAD=abs: the view-parallel densification exchange has no absgrad")
    accum, denom = getattr(gaussians, "xyz_gradient_accum", None), getattr(gaussians, "denom", None)
    P = accum.shape[0] if isinstance(accum, torch.Tensor) else -1
    device = absgrad.device
    if not (_dense_f32(absgrad, device, (P, 2)) and isinstance(update_filter, torch.Tensor) and update_filter.dtype == torch.bool
            and update_filter.device == device and update_filter.is_contiguous() and tuple(update_filter.shape) == (P,)
            and _dense_f32(accum, device, (P, 1)) and _dense_f32(denom, device, (P, 1))):
        raise RuntimeError("LGR_DENSIFY_GRAD=abs needs a float32 CUDA absgrad [P,2], a contiguous bool filter [P] and float32 [P,1] "
                           "xyz_gradient_accum / denom on the same device")
    trace.bump("densify_stats_native")
    trace.bump("densify_stats_absgrad")
    lib = capi.load()
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats(P, absgrad.data_ptr(), 2, update_filter.data_ptr(), accum.data_ptr(), denom.data_ptr(),
                                         capi.current_stream_ptr(device)), "lgr_densify_stats")


_error_words = {}   # "cuda:<index>" -> int32 [1] device word of lgr_densify_stats_exchanged's checks


def _device_key(device) -> str:
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return str(device)


def error_word(device):
    """the device word the exchanged statistics calls on `device` report mismatches into (see stats_exchanged)"""
    key = _device_key(device)
    if key not in _error_words:
        _error_words[key] = torch.zeros((1,), dtype=torch.int32, device=device)
    return _error_words[key]


def stats_exchanged(xs, k, rank, serial, world, grad, update_filter, accum, denom):
    """add_densification_stats of a view-parallel step whose backward published its statistics in buffer k of the sparse exchange `xs`
    (rasterizer._SparseExchange, or one simulated rank of it): every rank's view, in rank order, added to accum / denom.  `rank` is the
    caller's rank, `serial` the step serial the packs were stamped with.  The kernel checks the caller's own slot against `grad` and
    `update_filter` and every slot's serial; a mismatch sets error_word(device), which makes the next densify_and_prune raise.
    No host synchronisation, no collective."""
    trace.bump("densify_stats_exchanged")
    lib = capi.load()
    P, device = accum.shape[0], accum.device
    err = error_word(device)
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats_exchanged(P, int(world), int(rank), xs.ptr_tables[k], int(serial) & 0xFFFFFFFF, grad.data_ptr(),
                                                   grad.stride(0), update_filter.data_ptr(), accum.data_ptr(), denom.data_ptr(),
                                                   err.data_ptr(), capi.current_stream_ptr(device)), "lgr_densify_stats_exchanged")


def stats_encode(grad, update_filter):
    """this rank's view as one float32 per Gaussian: |grad[i, :2]| where update_filter is set, -1.0 elsewhere"""
    lib = capi.load()
    P, device = update_filter.shape[0], update_filter.device
    out = torch.empty((P,), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats_encode(P, grad.data_ptr(), grad.stride(0), update_filter.data_ptr(), out.data_ptr(),
                                                capi.current_stream_ptr(device)), "lgr_densify_stats_encode")
    return out


def stats_add_views(views, accum, denom):
    """adds the encoded views [world, P] to accum / denom in row order, with add_densification_stats' arithmetic"""
    lib = capi.load()
    world, P = views.shape
    device = accum.device
    views = views.contiguous()
    with torch.cuda.device(device):
        capi.check(lib.lgr_densify_stats_add_views(P, world, views.data_ptr(), accum.data_ptr(), denom.data_ptr(),
                                                   capi.current_stream_ptr(device)), "lgr_densify_stats_add_views")


def stats_allgather(grad, update_filter, accum, denom, world, group):
    """add_densification_stats of a view-parallel step without published statistics (dense exchange, a backward outside the fused
    node): encode, one all-gather into [world, P] over the exchange group, add the views in rank order"""
    import torch.distributed as dist
    trace.bump("densify_stats_allgather")
    mine = stats_encode(grad, update_filter)
    views = torch.empty((int(world), mine.shape[0]), dtype=torch.float32, device=mine.device)
    dist.all_gather_into_tensor(views, mine, group=group)
    stats_add_views(views, accum, denom)


def _exchange_error_to_host(device):
    """queues the copy of the exchanged statistics' error word into pinned memory and clears the word; None when the exchanged
    statistics never ran on `device`.  The caller reads the returned tensor after its next stream synchronisation."""
    word = _error_words.get(_device_key(device))
    if word is None:
        return None
    host = torch.empty((1,), dtype=torch.int32, pin_memory=True)
    host.copy_(word, non_blocking=True)
    word.zero_()
    return host


def _raise_on_exchange_error(host):
    if host is None or int(host[0]) == 0:
        return
    e = int(host[0])
    why = [w for bit, w in ((capi.SPARSE_STATS_ERR_HEADER, "a statistics call that did not match its step's exchange (a pack without "
                                                             "statistics, another step's buffer, or another P)"),
                            (capi.SPARSE_STATS_ERR_FILTER, "an update filter other than this view's radii > 0"),
                            (capi.SPARSE_STATS_ERR_GRAD, "a view-space gradient other than this view's dL/dmeans2D")) if e & bit]
    raise RuntimeError("view-parallel densification statistics are inconsistent across ranks: " + "; ".join(why) +
                       ". densify_and_prune refuses to run, so that the replicas cannot diverge")


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
        xyz = getattr(gaussians, "_xyz", None)
        if isinstance(xyz, torch.Tensor) and xyz.is_cuda:
            with torch.cuda.device(xyz.device):
                host = _exchange_error_to_host(xyz.device)
                if host is not None:
                    torch.cuda.current_stream(xyz.device).synchronize()
            _raise_on_exchange_error(host)
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
        # the checks of the view-parallel statistics calls since the last event: read back with the plan's one synchronisation
        err_host = _exchange_error_to_host(device)
        capi.check(lib.lgr_densify_plan(P, gaussians.xyz_gradient_accum.data_ptr(), gaussians.denom.data_ptr(), leaf["scaling"].data_ptr(),
                                        leaf["opacity"].data_ptr(), _f32(max_grad), _f32(gaussians.percent_dense * extent), _f32(min_opacity),
                                        _f32(0.1 * extent), int(prune_all), int(bool(max_screen_size)), ws.data_ptr(), ws.numel(), counts,
                                        stream), "lgr_densify_plan")
        if err_host is not None and P == 0:
            torch.cuda.current_stream(device).synchronize()   # the plan returns before synchronising when there are no rows
        _raise_on_exchange_error(err_host)
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
