"""Optimizer side of the training loops (SURVEY.md section 8f, row N3).

`FusedAdamW` is `torch.optim.AdamW` (same constructor, param_groups, state layout `step / exp_avg / exp_avg_sq`, state_dict) whose
`step()` issues ONE kernel for all parameter groups (`lgr_adamw_step`) instead of torch's ~9 foreach launches per group; the
per-element arithmetic reproduces torch's default CUDA path (torch/optim/adam.py `_multi_tensor_adam`) bit for bit.  The reference
builds its optimizer as `torch.optim.AdamW(l, lr=0.0, eps=1e-15)` over six groups of one tensor each
(scene/gaussian_model.py:184-217) and only ever touches `state[p]["exp_avg"]`, `state[p]["exp_avg_sq"]`, `param_groups[i]["lr"]`,
`["params"][0]`, `["name"]` and `state_dict()` afterwards (:219-225, :544-660) -- all of which this class keeps.

`SelectiveAdamW` (opt-in, `LGR_SELECTIVE_ADAM=1`) is the same optimizer restricted to the Gaussians whose gradient row is not all
zero (`lgr_adamw_step_selective`); the rows a step did not reach keep their parameters and moments untouched.

`compact_rows` / `prune_points` are the fused form of `GaussianModel._prune_optimizer` + `prune_points` (:564-600): one stream
compaction of the mask, then ONE gather launch for the parameters and both Adam moments of every group.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import capi, trace


class FusedAdamW(torch.optim.AdamW):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, **kw):
        for flag in ("maximize", "capturable", "differentiable", "fused"):
            if kw.get(flag):
                raise NotImplementedError(f"FusedAdamW: {flag}=True is not implemented (the reference does not use it)")
        if amsgrad:
            raise NotImplementedError("FusedAdamW: amsgrad=True is not implemented (the reference does not use it)")
        kw.pop("foreach", None)
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, **kw)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = capi.load()
        trace.bump("adamw_steps")
        for (device, beta1, beta2, eps, wd), items in self._prepare().items():
            for i0 in range(0, len(items), 8):
                chunk = items[i0:i0 + 8]
                arr = (capi.LgrAdamwTensor * len(chunk))()
                for a, (p, g, m, v, lr, step, row_elems, row_stride) in zip(arr, chunk):
                    a.param, a.grad, a.exp_avg, a.exp_avg_sq = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
                    a.numel, a.lr, a.step = p.numel(), lr, step
                    a.row_elems, a.param_row_stride = row_elems, row_stride
                with torch.cuda.device(device):
                    st = lib.lgr_adamw_step(len(chunk), arr, beta1, beta2, eps, wd, capi.current_stream_ptr(device))
                capi.check(st, "lgr_adamw_step")
        return loss

    def _prepare(self):
        """Checks every parameter with a gradient, creates its state on first use and increments its step, as torch's AdamW does.
        Returns {(device, beta1, beta2, eps, weight_decay): [(p, g, m, v, lr, step, row_elems, row_stride)]} with every gradient in a
        layout the kernels take."""
        by_cfg = {}
        for group in self.param_groups:
            if isinstance(group["lr"], torch.Tensor):
                raise NotImplementedError("FusedAdamW: tensor learning rates are not implemented")
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("AdamW does not support sparse gradients")
                if not (p.is_cuda and p.dtype == torch.float32):
                    raise RuntimeError("FusedAdamW needs float32 CUDA parameters: there is no CPU path")
                # a parameter is updated IN PLACE whatever its layout: dense ones by the vectorised path, row-strided views such as
                # the distillation student's _features_rest[:, :8, :] (scene/gaussian_model.py:129-136; registered as is by
                # distill_train.py:79) through (row_elems, row_stride); the keys of optimizer.state stay the caller's tensors
                row_elems = row_stride = 0
                permuted = not p.is_contiguous() and _permuted_dense(p)
                if not p.is_contiguous() and not permuted:
                    trace.bump("adamw_strided_params")
                    row_elems, row_stride = _row_strided(p)
                    if row_elems == 0:
                        raise RuntimeError(f"FusedAdamW: parameter of shape {tuple(p.shape)} and strides {p.stride()} is neither dense "
                                           "nor a row-strided view of a dense tensor")
                state = self.state[p]
                if len(state) == 0:                                   # torch/optim/adam.py _init_group
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)      # dense for a non-dense view
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                m, v = state["exp_avg"], state["exp_avg_sq"]
                if permuted:
                    # a dense parameter in a permuted layout, such as the _xyz GaussianModel.create_from_pcd builds from a transposed numpy
                    # array: the update is element-wise, so every tensor is walked in the parameter's own memory order
                    g = p.grad if p.grad.stride() == p.stride() else torch.empty_like(p).copy_(p.grad)
                    if m.stride() != p.stride() or v.stride() != p.stride():
                        raise RuntimeError("FusedAdamW: optimizer state must have its parameter's layout")
                else:
                    g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                    if not (m.is_contiguous() and v.is_contiguous()):
                        raise RuntimeError("FusedAdamW: optimizer state must be contiguous")
                key = (p.device, float(beta1), float(beta2), float(group["eps"]), float(group["weight_decay"]))
                by_cfg.setdefault(key, []).append((p, g, m, v, float(group["lr"]), float(state["step"]), row_elems, row_stride))
        return by_cfg


class SelectiveAdamW(FusedAdamW):
    """FusedAdamW that updates only the Gaussians a step reached: the selective (sparse) Adam of Taming-3DGS and gsplat's
    SelectiveAdam, with the mask taken from the gradients themselves.  Opt-in: results differ from torch's AdamW by design.

    Every parameter with a gradient must have the same number of rows P (one per Gaussian).  Row i is active when any element of
    row i of any of those gradients is not equal to zero (+0 and -0 are zero; a NaN makes the row active).  Every element of an active
    row is updated bit-identically to FusedAdamW / torch.optim.AdamW with its group's hyper-parameters and step count; the parameter,
    exp_avg and exp_avg_sq of an inactive row are left untouched (no momentum step, no weight decay).  state["step"] is incremented
    for every parameter with a gradient, whichever rows were active, so a row that wakes up uses the global step for bias correction.
    Same constructor, state layout and state_dict as torch.optim.AdamW: checkpoints move freely between the three.  The groups must
    share betas, eps and weight_decay (the reference's six groups differ only in lr)."""

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        # everything that can refuse the step does so before any state changes
        live = [(g, p) for g in self.param_groups for p in g["params"] if p.grad is not None]
        rows = {p.shape[0] if p.dim() else 1 for _, p in live}
        if len(rows) > 1:
            raise RuntimeError(f"SelectiveAdamW: parameters with a gradient must share their number of rows, got {sorted(rows)}")
        if len({(float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"])) for g, _ in live}) > 1:
            raise NotImplementedError("SelectiveAdamW: all groups must share betas, eps and weight_decay")
        if len({p.device for _, p in live}) > 1 or len(live) > 8:
            raise NotImplementedError("SelectiveAdamW: at most 8 parameters with a gradient, on one device (one row mask spans them all)")
        for _, p in live:
            if p.numel():
                _row_view(p)     # _prepare gives the gradient and the moments this layout or a contiguous one
        lib = capi.load()
        trace.bump("adamw_selective_steps")
        for (device, beta1, beta2, eps, wd), items in self._prepare().items():
            P = rows.pop()
            arr = (capi.LgrAdamwRowTensor * len(items))()
            for a, (p, g, m, v, lr, step, _, _) in zip(arr, items):
                a.param, a.grad, a.exp_avg, a.exp_avg_sq = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
                a.width, a.lr, a.step = (p.numel() // P) if P else 0, lr, step
                if a.width:
                    a.param_row_stride, a.param_col_stride = _row_view(p)
                    a.grad_row_stride, a.grad_col_stride = _row_view(g, p)
                    a.exp_avg_row_stride, a.exp_avg_col_stride = _row_view(m, p)
                    a.exp_avg_sq_row_stride, a.exp_avg_sq_col_stride = _row_view(v, p)
            with torch.cuda.device(device):
                st = lib.lgr_adamw_step_selective(len(items), arr, P, beta1, beta2, eps, wd, capi.current_stream_ptr(device))
            capi.check(st, "lgr_adamw_step_selective")
        return loss


def _row_view(t, like=None):
    """(row stride, column stride) of `t` seen as [P, width]: column c is the c-th element of a row in the memory order of the
    parameter `like` (default: `t` itself), so that p, g, m and v pair up element by element.  Raises when the non-row dimensions
    do not flatten to one column stride."""
    order = sorted((d for d in range(1, t.dim()) if t.size(d) != 1), key=(like if like is not None else t).stride)
    cs = t.stride(order[0]) if order else 1
    expect = cs
    for d in order:
        if t.stride(d) != expect:
            raise RuntimeError(f"SelectiveAdamW: a tensor of shape {tuple(t.shape)} and strides {t.stride()} is not a [rows, width] view")
        expect *= t.size(d)
    return (t.stride(0) if t.dim() else 1), cs

def _permuted_dense(p):
    """True when `p` fills its memory exactly once in some order of its dimensions (a transposed or permuted dense tensor)"""
    expect = 1
    for d in sorted(range(p.dim()), key=p.stride):
        if p.size(d) != 1 and p.stride(d) != expect:
            return False
        expect *= p.size(d)
    return True


def _row_strided(p):
    """(elements per row, row stride) when `p` is a view whose rows are dense and start `stride` elements apart, else (0, 0)."""
    if p.dim() < 2 or p.numel() == 0:
        return 0, 0
    inner = 1
    for d in range(p.dim() - 1, 0, -1):          # dims 1.. must be dense among themselves
        if p.size(d) != 1 and p.stride(d) != inner:
            return 0, 0
        inner *= p.size(d)
    if p.stride(0) < inner:
        return 0, 0
    return inner, p.stride(0)


def compact_rows(tensors, keep):
    """[t[keep] for t in tensors] for row-major float32/int32 CUDA tensors sharing dim 0, in one gather launch.
    `keep` is a bool/uint8 CUDA mask over the rows."""
    lib = capi.load()
    if keep.dtype == torch.bool:
        keep = keep.view(torch.uint8)
    if not (keep.is_cuda and keep.dtype == torch.uint8 and keep.dim() == 1 and keep.is_contiguous()):
        raise RuntimeError("compact_rows: the mask must be a contiguous 1-D bool/uint8 CUDA tensor")
    P, device = keep.shape[0], keep.device
    for t in tensors:
        if not (t.is_cuda and t.device == device and t.shape[0] == P and t.element_size() == 4 and t.is_contiguous()):
            raise RuntimeError("compact_rows: tensors must be contiguous 4-byte CUDA tensors with the mask's number of rows")
    ws = torch.empty(int(lib.lgr_compact_workspace_bytes(P)), dtype=torch.uint8, device=device)
    src_row = torch.empty(max(P, 1), dtype=torch.int32, device=device)
    n_out = C.c_int32(0)
    stream = capi.current_stream_ptr(device)
    with torch.cuda.device(device):
        st = lib.lgr_compact_plan(P, keep.data_ptr(), src_row.data_ptr(), ws.data_ptr(), ws.numel(), C.byref(n_out), stream)
        capi.check(st, "lgr_compact_plan")
        rows = int(n_out.value)
        outs = [torch.empty((rows,) + tuple(t.shape[1:]), dtype=t.dtype, device=device) for t in tensors]
        for i0 in range(0, len(tensors), 24):
            chunk = list(zip(tensors[i0:i0 + 24], outs[i0:i0 + 24]))
            arr = (capi.LgrCompactTensor * len(chunk))()
            for a, (t, o) in zip(arr, chunk):
                a.src, a.dst = t.data_ptr() if t.numel() else None, o.data_ptr() if o.numel() else None
                a.row_words = (t.numel() // P) if (P and o.numel()) else 0
            st = lib.lgr_compact_rows(rows, src_row.data_ptr(), len(chunk), arr, stream)
            capi.check(st, "lgr_compact_rows")
    return outs


_GROUP_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
               "rotation": "_rotation"}


def prune_points(gaussians, mask):
    """GaussianModel.prune_points(mask) (scene/gaussian_model.py:587-600) with the optimizer surgery of _prune_optimizer (:564-585)
    done by ONE compaction: same resulting parameters, Adam moments, optimizer.state keys and auxiliary buffers.
    Install with `GaussianModel.prune_points = lightgaussian_b200.optim.prune_points`."""
    keep = ~mask
    opt = gaussians.optimizer
    entries = []            # (group, stored_state or None)
    tensors = []
    for group in opt.param_groups:
        p = group["params"][0]
        st = opt.state.get(p, None)
        entries.append((group, st))
        tensors.append(p.detach())
        if st is not None:
            tensors += [st["exp_avg"], st["exp_avg_sq"]]
    aux_names = [n for n in ("xyz_gradient_accum", "denom", "max_radii2D") if isinstance(getattr(gaussians, n, None), torch.Tensor)
                 and getattr(gaussians, n).shape[:1] == mask.shape]
    tensors += [getattr(gaussians, n) for n in aux_names]
    outs = iter(compact_rows([t.contiguous() for t in tensors], keep))
    for group, st in entries:
        old = group["params"][0]
        new = torch.nn.Parameter(next(outs).requires_grad_(True))
        if st is not None:
            st["exp_avg"], st["exp_avg_sq"] = next(outs), next(outs)
            del opt.state[old]
            opt.state[new] = st
        group["params"][0] = new
        setattr(gaussians, _GROUP_ATTR[group["name"]], new)
    for n in aux_names:
        setattr(gaussians, n, next(outs))


def to_fused(optimizer):
    """A FusedAdamW over the SAME parameter tensors, groups (incl. "name" and the current lr) and hyper-parameters as an existing
    torch.optim.AdamW, carrying its state over.  With LGR_SELECTIVE_ADAM=1 in the environment at the time of the call, a
    SelectiveAdamW instead (opt-in: inactive Gaussians are not stepped, so results differ from the reference's by design)."""
    if isinstance(optimizer, FusedAdamW):
        return optimizer
    if type(optimizer) is not torch.optim.AdamW:
        raise TypeError(f"to_fused expects torch.optim.AdamW, got {type(optimizer).__name__}")
    skip = {"foreach", "fused", "capturable", "differentiable", "maximize", "amsgrad", "decoupled_weight_decay"}
    for g in optimizer.param_groups:
        if g.get("amsgrad") or g.get("maximize") or g.get("capturable") or g.get("differentiable"):
            raise NotImplementedError("to_fused: amsgrad / maximize / capturable / differentiable groups are not supported")
    groups = [{k: v for k, v in g.items() if k not in skip} for g in optimizer.param_groups]
    cls = SelectiveAdamW if os.environ.get("LGR_SELECTIVE_ADAM", "0") == "1" else FusedAdamW
    fused = cls(groups, **{k: v for k, v in optimizer.defaults.items() if k not in skip})
    for p, st in optimizer.state.items():
        fused.state[p] = st
    return fused


def install(GaussianModel):
    """Make a GaussianModel class (scene/gaussian_model.py) use the fused optimizer step and prune compaction without editing it:
    `training_setup` (:176-224) is wrapped so that the AdamW it builds is replaced by an equivalent FusedAdamW, and `prune_points`
    (:587-600) becomes `optim.prune_points`.  When the class defines `add_densification_stats` and `densify_and_prune` (:745-788),
    they become the native ones of `densify`.  Idempotent."""
    if getattr(GaussianModel, "_lgr_fused_optim", False):
        return GaussianModel
    original_setup = GaussianModel.training_setup

    def training_setup(self, *args, **kwargs):
        out = original_setup(self, *args, **kwargs)
        self.optimizer = to_fused(self.optimizer)
        return out

    training_setup.__wrapped__ = original_setup
    GaussianModel.training_setup = training_setup
    GaussianModel.prune_points = prune_points
    if hasattr(GaussianModel, "add_densification_stats") and hasattr(GaussianModel, "densify_and_prune"):
        from . import densify
        densify.install(GaussianModel)
    GaussianModel._lgr_fused_optim = True
    return GaussianModel
