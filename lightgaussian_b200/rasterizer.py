"""The reference's Python rasterizer surface on top of liblgrast.so.

Mirrors RAST/diff_gaussian_rasterization/__init__.py (RAST = submodules/compress-diff-gaussian-rasterization):
  GaussianRasterizationSettings  (:248-261)  same 13 fields, same order
  GaussianRasterizer             (:263-346)  .forward / .forward_count / .markVisible / .raster_settings
  rasterize_gaussians            (:25-59)    dispatch on raster_settings.f_count
  _C                              pybind module of RAST/ext.cpp:15-20 -> here a namespace with the same four
                                  callables and the same argument order / tuple layouts.

Differences: launches go to torch's *current* stream on the tensors' device (the reference uses the legacy
default stream), gradients are produced without zero-filled temporaries, and the significance outputs of
count mode are exact and deterministic (see include/lgrast.h).
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import os as _os

import torch
import torch.nn as nn

from . import capi, trace


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    f_count: bool


_last_R = [0]
_last_deterministic = [False]


def last_num_rendered() -> int:
    """num_rendered of the most recent forward call in this process (diagnostics / bench.py)."""
    return _last_R[0]


def _apply_deterministic_mode() -> bool:
    """Deterministic mode of a forward, decided at the time of the call (capi.deterministic_requested) and set in the library.
    The autograd nodes record it, and their backward runs in that mode whatever the flag says by then."""
    det = capi.deterministic_requested()
    capi.set_deterministic(det)
    _last_deterministic[0] = det
    return det


def _f32c(t, name):
    """contiguous float32 CUDA view of an input (None for the reference's empty 'absent' tensors)."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    return t.contiguous()


def _make_view(device, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, scale_modifier, degree,
               prefiltered, debug):
    keep = [_f32c(background, "bg"), _f32c(viewmatrix, "viewmatrix"), _f32c(projmatrix, "projmatrix"), _f32c(campos, "campos")]
    for k, n in zip(keep, ("bg", "viewmatrix", "projmatrix", "campos")):
        if k is None:
            raise RuntimeError(f"{n} must be a non-empty CUDA tensor")
    v = capi.LgrView(int(W), int(H), float(tan_fovx), float(tan_fovy), float(scale_modifier), int(degree), int(bool(prefiltered)),
                     int(bool(debug)), keep[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr(), keep[0].data_ptr())
    return v, keep


def _weight_out(count_mode, blend_weight, P, device):
    """The int64 [P] blending-weight output a count forward was given, checked (None when there is none)."""
    if blend_weight is None:
        return None
    if not count_mode:
        raise RuntimeError("blend_weight is a count-mode output")
    if blend_weight.dtype != torch.int64 or tuple(blend_weight.shape) != (P,) or not blend_weight.is_contiguous() or blend_weight.device != device:
        raise RuntimeError(f"blend_weight must be a contiguous int64 [{P}] tensor on {device}")
    return blend_weight


def _forward_native(count_mode, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                    projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug, blend_weight=None):
    """blend_weight: optional int64 [P] output of a count forward, overwritten with this view's fixed-point blending weights
    (lgr_forward_count_weight)."""
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:68-70
    lib = capi.load()
    device = means3D.device
    if not means3D.is_cuda:
        raise RuntimeError("means3D must be a CUDA tensor: this rasterizer has no CPU path")
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    means3D_c = _f32c(means3D, "means3D")
    colors_c, opacity_c = _f32c(colors, "colors_precomp"), _f32c(opacity, "opacities")
    scales_c, rot_c, cov_c, sh_c = _f32c(scales, "scales"), _f32c(rotations, "rotations"), _f32c(cov3D_precomp, "cov3D_precomp"), _f32c(sh, "sh")
    M = 0 if sh_c is None else sh_c.size(1)
    out_color = torch.empty((3, H, W), dtype=torch.float32, device=device)
    radii = torch.empty((P,), dtype=torch.int32, device=device)
    count = score = None
    if count_mode:
        count = torch.empty((P,), dtype=torch.int32, device=device)
        score = torch.empty((P,), dtype=torch.float32, device=device)
    weight = _weight_out(count_mode, blend_weight, P, device)
    _apply_deterministic_mode()
    slots = [capi.BlobSlot(device) for _ in range(3)]
    num_rendered = C.c_int32(0)
    try:
        with torch.cuda.device(device):
            view, keep = _make_view(device, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, scale_modifier,
                                    degree, prefiltered, debug)
            stream = capi.current_stream_ptr(device)
            common = (C.byref(view), P, M, capi.ptr(means3D_c), capi.ptr(sh_c), capi.ptr(colors_c), capi.ptr(opacity_c),
                      capi.ptr(scales_c), capi.ptr(rot_c), capi.ptr(cov_c),
                      capi.ALLOC_CB, slots[0].key, capi.ALLOC_CB, slots[1].key, capi.ALLOC_CB, slots[2].key)
            if weight is not None:
                st = lib.lgr_forward_count_weight(*common, out_color.data_ptr(), capi.ptr(count), capi.ptr(score), capi.ptr(weight),
                                                  capi.ptr(radii), C.byref(num_rendered), stream)
            elif count_mode:
                st = lib.lgr_forward_count(*common, out_color.data_ptr(), capi.ptr(count), capi.ptr(score), capi.ptr(radii),
                                           C.byref(num_rendered), stream)
            else:
                st = lib.lgr_forward(*common, out_color.data_ptr(), capi.ptr(radii), C.byref(num_rendered), stream)
        capi.check(st, "lgr_forward_count_weight" if weight is not None else "lgr_forward_count" if count_mode else "lgr_forward")
    finally:
        for s in slots:
            s.release()
    empty = lambda: torch.empty((0,), dtype=torch.uint8, device=device)  # noqa: E731
    geom, binning, img = (s.tensor if s.tensor is not None else empty() for s in slots)
    _last_R[0] = int(num_rendered.value)
    if P == 0:
        radii = torch.zeros((0,), dtype=torch.int32, device=device)
    return count, score, int(num_rendered.value), out_color, radii, geom, binning, img


class _NativeModule:
    """Stand-in for the reference's pybind module `diff_gaussian_rasterization._C` (RAST/ext.cpp:15-20)."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                            projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug):
        r = _forward_native(False, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                            projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug)
        return r[2:]  # (num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer)

    @staticmethod
    def count_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                        projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug, f_count=True,
                        blend_weight=None):
        """The reference's tuple; blend_weight (int64 [P], optional) also receives the view's fixed-point blending weights."""
        return _forward_native(True, background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                               projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug,
                               blend_weight)

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                                     projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos, geomBuffer, R, binningBuffer,
                                     imageBuffer, debug):
        lib = capi.load()
        device = means3D.device
        P = means3D.size(0)
        H, W = dL_dout_color.size(1), dL_dout_color.size(2)
        means3D_c, colors_c = _f32c(means3D, "means3D"), _f32c(colors, "colors_precomp")
        scales_c, rot_c, cov_c, sh_c = _f32c(scales, "scales"), _f32c(rotations, "rotations"), _f32c(cov3D_precomp, "cov3D_precomp"), _f32c(sh, "sh")
        M = 0 if sh_c is None else sh_c.size(1)
        dpix = _f32c(dL_dout_color, "dL_dout_color")
        mk = lambda *shape: torch.empty(shape, dtype=torch.float32, device=device)  # noqa: E731
        dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D = mk(P, 3), mk(P, 3), mk(P, 1), mk(P, 3)
        dL_dcov3D, dL_dsh, dL_dscales, dL_drot = mk(P, 6), mk(P, M, 3), mk(P, 3), mk(P, 4)
        if P != 0:
            with torch.cuda.device(device):
                view, keep = _make_view(device, background, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, H, W, scale_modifier,
                                        degree, False, debug)
                st = lib.lgr_backward(C.byref(view), P, M, int(R), capi.ptr(means3D_c), capi.ptr(sh_c), capi.ptr(colors_c),
                                      capi.ptr(scales_c), capi.ptr(rot_c), capi.ptr(cov_c), capi.ptr(radii.contiguous()),
                                      geomBuffer.data_ptr(), binningBuffer.data_ptr(), imageBuffer.data_ptr(), dpix.data_ptr(),
                                      dL_dmeans2D.data_ptr(), dL_dcolors.data_ptr(), dL_dopacity.data_ptr(), dL_dmeans3D.data_ptr(),
                                      dL_dcov3D.data_ptr(), capi.ptr(dL_dsh), dL_dscales.data_ptr(), dL_drot.data_ptr(),
                                      capi.current_stream_ptr(device))
            capi.check(st, "lgr_backward")
        return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drot

    @staticmethod
    def mark_visible(means3D, viewmatrix, projmatrix):
        lib = capi.load()
        P = means3D.size(0)
        present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
        if P != 0:
            m, v, p = _f32c(means3D, "means3D"), _f32c(viewmatrix, "viewmatrix"), _f32c(projmatrix, "projmatrix")
            with torch.cuda.device(means3D.device):
                st = lib.lgr_mark_visible(P, m.data_ptr(), v.data_ptr(), p.data_ptr(), present.data_ptr(),
                                          capi.current_stream_ptr(means3D.device))
            capi.check(st, "lgr_mark_visible")
        return present


_C = _NativeModule()


def _pack_args(rs, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh):
    return (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered,
            rs.debug)


class _RasterizeGaussians(torch.autograd.Function):
    """autograd node of the non-count path (RAST/diff_gaussian_rasterization/__init__.py:62-137,192-246)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        args = _pack_args(raster_settings, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh)
        num_rendered, color, radii, geomBuffer, binningBuffer, imgBuffer = _C.rasterize_gaussians(*args)
        ctx.raster_settings = raster_settings
        ctx.num_rendered = num_rendered
        ctx.deterministic = _last_deterministic[0]
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _):
        rs = ctx.raster_settings
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer = ctx.saved_tensors
        capi.set_deterministic(ctx.deterministic)   # the mode of the forward, whatever the flag says now
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = _C.rasterize_gaussians_backward(
            rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, grad_out_color, sh, rs.sh_degree, rs.campos, geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer,
            rs.debug)
        # gradients of absent inputs (empty tensors) must have the inputs' (empty) shape
        def fit(g, ref):
            return g if ref.numel() != 0 else None
        if _exchange["world"] > 1:
            _exchange["stats_record"] = None   # no statistics published: add_densification_stats all-gathers them
            # view-parallel training that left the fused node (override_color, convert_SHs_python / compute_cov3D_python, LGR_FUSED=0,
            # a leaf layout the fused kernels cannot read): the replicas must still step on the SUM over all ranks' views, so the
            # per-Gaussian gradients are all-reduced here (dense NCCL: correct, but ~2x slower than the fused sparse exchange).
            # grad_means2D stays local: it feeds per-view densification statistics, not a parameter.
            _allreduce_unfused([grad_means3D, fit(grad_sh, sh), fit(grad_colors_precomp, colors_precomp), grad_opacities,
                                fit(grad_scales, scales), fit(grad_rotations, rotations), fit(grad_cov3Ds_precomp, cov3Ds_precomp)])
        return (grad_means3D, grad_means2D, fit(grad_sh, sh), fit(grad_colors_precomp, colors_precomp), grad_opacities,
                fit(grad_scales, scales), fit(grad_rotations, rotations), fit(grad_cov3Ds_precomp, cov3Ds_precomp), None)

    @staticmethod
    def forward_count(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, blend_weight=None):
        """No autograd, exactly like the reference (:140-189)."""
        assert raster_settings.f_count
        args = _pack_args(raster_settings, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh)
        gaussians_count, important_score, _, color, radii, _, _, _ = _C.count_gaussians(*args, raster_settings.f_count,
                                                                                        blend_weight=blend_weight)
        return gaussians_count, important_score, color, radii


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                        blend_weight=None):
    if raster_settings.f_count:
        return _RasterizeGaussians.forward_count(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                                 raster_settings, blend_weight)
    if blend_weight is not None:
        raise RuntimeError("blend_weight is a count-mode output (raster_settings.f_count)")
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def _run(self, means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, blend_weight=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        has_sr = scales is not None or rotations is not None
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (has_sr and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        absent = torch.Tensor([])
        shs = absent if shs is None else shs
        colors_precomp = absent if colors_precomp is None else colors_precomp
        scales = absent if scales is None else scales
        rotations = absent if rotations is None else rotations
        cov3D_precomp = absent if cov3D_precomp is None else cov3D_precomp
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   self.raster_settings, blend_weight)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        return self._run(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp)

    def forward_count(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                      cov3D_precomp=None, blend_weight=None):
        """blend_weight: optional int64 [P] tensor that receives this view's fixed-point blending weights (include/lgrast.h,
        lgr_forward_count_weight); the four outputs are unchanged."""
        return self._run(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, blend_weight)


# ------------------------------------------------------------------------------------------------------------------
# Fused-activation path (SURVEY.md section 8f, row N1): the rasterizer consumes GaussianModel's six raw leaves.
# Only gaussian_renderer.render()/count_render() use it; the reference-compatible API above is unchanged.
# ------------------------------------------------------------------------------------------------------------------
def rest_row_stride(rest) -> int:
    """Row stride (floats) of a features_rest leaf the kernels can read in place, or 0 when it has to be copied.
    Dense [P,K,3] tensors, and row-strided views of them -- the distillation student's `_features_rest[:, :8, :]`
    (scene/gaussian_model.py:129-136: stride (45,3,1)) -- qualify: rows start at multiples of the stride, inner layout dense."""
    if rest.dim() != 3 or rest.size(2) != 3:
        return 0
    if rest.is_contiguous():
        return rest.size(1) * 3
    P, K = rest.size(0), rest.size(1)
    if P == 0 or K == 0:
        return 0
    st = rest.stride()
    if st[2] != 1 or st[1] != 3 or st[0] < 3 * K or st[0] > 256:
        return 0
    # whole rows of `stride` floats are staged: the storage must extend that far behind the last row's start
    if rest.storage_offset() + P * st[0] > rest.untyped_storage().nbytes() // 4 or rest.data_ptr() % 16:
        return 0
    return st[0]


def _raw_struct(xyz, dc, rest, scaling, rotation, opacity):
    dense = rest.numel() == 0 or rest.is_contiguous()
    return capi.LgrRawParams(capi.ptr(xyz), capi.ptr(dc), capi.ptr(rest), capi.ptr(scaling), capi.ptr(rotation), capi.ptr(opacity),
                             0 if dense else rest_row_stride(rest))


def _forward_raw_native(count_mode, rs, xyz, dc, rest, scaling, rotation, opacity, blend_weight=None, depth=None):
    """blend_weight: optional int64 [P] output of a count forward (lgr_forward_raw_weight), as in _forward_native.
    depth: optional (depth_mode, out_depth, out_alpha) of lgr_forward_raw_depth, the two planes [H,W]-sized float32 tensors or None."""
    lib = capi.load()
    device = xyz.device
    P, H, W = xyz.size(0), int(rs.image_height), int(rs.image_width)
    M = 1 + rest.size(1)
    leaves = [_f32c(t, n) if t.numel() else t for t, n in
              ((xyz, "xyz"), (dc, "features_dc"), (scaling, "scaling"), (rotation, "rotation"), (opacity, "opacity"))]
    if rest.numel() and not rest.is_contiguous() and rest_row_stride(rest) and rest.dtype == torch.float32 and rest.is_cuda:
        rest_c = rest                      # row-strided view: read in place through features_rest_row_stride
    else:
        rest_c = _f32c(rest, "features_rest") if rest.numel() else rest
    leaves.insert(2, rest_c)
    out_color = torch.empty((3, H, W), dtype=torch.float32, device=device)
    radii = torch.empty((P,), dtype=torch.int32, device=device)
    count = score = None
    if count_mode:
        count = torch.empty((P,), dtype=torch.int32, device=device)
        score = torch.empty((P,), dtype=torch.float32, device=device)
    weight = _weight_out(count_mode, blend_weight, P, device)
    _apply_deterministic_mode()
    slots = [capi.BlobSlot(device) for _ in range(3)]
    num_rendered = C.c_int32(0)
    try:
        with torch.cuda.device(device):
            view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W, rs.scale_modifier,
                                    rs.sh_degree, rs.prefiltered, rs.debug)
            params = _raw_struct(*leaves)
            head = (C.byref(view), P, M, C.byref(params), capi.ALLOC_CB, slots[0].key, capi.ALLOC_CB, slots[1].key, capi.ALLOC_CB, slots[2].key,
                    out_color.data_ptr(), capi.ptr(count), capi.ptr(score))
            tail = (capi.ptr(radii), C.byref(num_rendered), capi.current_stream_ptr(device))
            if weight is not None:
                st = lib.lgr_forward_raw_weight(*head, capi.ptr(weight), *tail)
            elif depth is not None:
                st = lib.lgr_forward_raw_depth(*head, int(depth[0]), capi.ptr(depth[1]), capi.ptr(depth[2]), *tail)
            else:
                st = lib.lgr_forward_raw(*head, *tail)
        capi.check(st, "lgr_forward_raw_weight" if weight is not None else "lgr_forward_raw_depth" if depth is not None else "lgr_forward_raw")
    finally:
        for s_ in slots:
            s_.release()
    empty = lambda: torch.empty((0,), dtype=torch.uint8, device=device)  # noqa: E731
    geom, binning, img = (s_.tensor if s_.tensor is not None else empty() for s_ in slots)
    _last_R[0] = int(num_rendered.value)
    if P == 0:
        radii = torch.zeros((0,), dtype=torch.int32, device=device)
    return count, score, int(num_rendered.value), out_color, radii, geom, binning, img, leaves


def forward_vq_native(count_mode, rs, xyz, store, blend_weight=None):
    """Forward of a resident VQ model (lgr_forward_vq): (count, score, color, radii), count and score None unless count_mode.
    `store` is a vqresident.ResidentVQ; `xyz` its positions ([P,3] float32, the model's _xyz).  No autograd.
    blend_weight: optional int64 [P] output of a count forward (lgr_forward_vq_weight), as in _forward_native."""
    lib = capi.load()
    arrays = (xyz, store.attr, store.slot, store.codebook, store.nonvq)
    if not all(t.is_cuda and t.device == xyz.device and t.is_contiguous() for t in arrays):
        raise RuntimeError("forward_vq_native: xyz and the resident arrays must be contiguous tensors on one CUDA device")
    if xyz.dtype != torch.float32 or tuple(xyz.shape) != (store.P, 3):
        raise RuntimeError("forward_vq_native: xyz must be float32 [P,3] for the store's P Gaussians")
    device = xyz.device
    P, H, W = store.P, int(rs.image_height), int(rs.image_width)
    out_color = torch.empty((3, H, W), dtype=torch.float32, device=device)
    radii = torch.empty((P,), dtype=torch.int32, device=device)
    count = score = None
    if count_mode:
        count = torch.empty((P,), dtype=torch.int32, device=device)
        score = torch.empty((P,), dtype=torch.float32, device=device)
    weight = _weight_out(count_mode, blend_weight, P, device)
    params = capi.LgrVqResidentParams(capi.ptr(xyz), capi.ptr(store.attr), capi.ptr(store.slot), capi.ptr(store.codebook),
                                      capi.ptr(store.nonvq), int(store.attr.dtype == torch.float16),
                                      int(store.nonvq.dtype == torch.float16), store.D, store.Dp, store.K)
    _apply_deterministic_mode()
    slots = [capi.BlobSlot(device) for _ in range(3)]
    num_rendered = C.c_int32(0)
    try:
        with torch.cuda.device(device):
            view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W, rs.scale_modifier,
                                    rs.sh_degree, rs.prefiltered, rs.debug)
            head = (C.byref(view), P, C.byref(params), capi.ALLOC_CB, slots[0].key, capi.ALLOC_CB, slots[1].key, capi.ALLOC_CB, slots[2].key,
                    out_color.data_ptr(), capi.ptr(count), capi.ptr(score))
            tail = (capi.ptr(radii), C.byref(num_rendered), capi.current_stream_ptr(device))
            if weight is not None:
                st = lib.lgr_forward_vq_weight(*head, capi.ptr(weight), *tail)
            else:
                st = lib.lgr_forward_vq(*head, *tail)
        capi.check(st, "lgr_forward_vq_weight" if weight is not None else "lgr_forward_vq")
    finally:
        for s_ in slots:
            s_.release()
    _last_R[0] = int(num_rendered.value)
    return count, score, out_color, radii


# View-parallel gradient exchange (SURVEY.md section 8e).  When enabled, the backward of the fused node returns gradients that
# are already SUMMED over all ranks' views: the dense leaves (xyz, scaling, rotation, opacity: 44 B/Gaussian) go through one
# all-reduce, while the SH gradient (12*M B/Gaussian) is exchanged as its rank-1 factor dRGB (12 B/Gaussian, all-gather) and
# rebuilt locally by lgr_sh_grad_from_views -- ~4x less NVLink traffic than all-reducing the dense gradient at degree 3.
_exchange = {"world": 1, "group": None, "warned_unfused": False, "unfused_calls": 0,
             "densify": False,       # view-parallel densification statistics (densify.add_densification_stats)
             "serial": 0,            # exchanged backwards with statistics so far (the same count on every rank)
             "stats_record": None}   # what the next statistics call reads: the last exchanged backward's buffer, if it published stats


def enable_gradient_exchange(world: int, group=None, *, densification: bool = False):
    """From now on every rasterizer backward in this process returns per-Gaussian gradients SUMMED over the `world` ranks' views:
    the fused node (`render()` on GaussianModel leaves) through the sparse NVLink peer-memory exchange, every other path through a
    dense NCCL all-reduce inside `_RasterizeGaussians.backward` -- no path is left that silently keeps rank-local gradients.
    densification=True (world > 1): GaussianModel.add_densification_stats (as densify.install makes it) also adds every rank's view of
    the step, in rank order, so that every rank takes the same densify-and-prune decisions; the sparse exchange then carries the
    statistics in its slots (DESIGN.md section 6)."""
    _exchange["world"], _exchange["group"] = int(world), group
    _exchange["densify"] = bool(densification) and int(world) > 1
    _exchange["stats_record"] = None


def densification_exchange() -> bool:
    """True when add_densification_stats sums every rank's view (enable_gradient_exchange(world > 1, densification=True))"""
    return _exchange["densify"] and _exchange["world"] > 1


def unfused_exchange_calls() -> int:
    """how many backward passes took the dense all-reduce of the unfused node since start (bench.py / tests: should be 0 on the hot path)"""
    return _exchange["unfused_calls"]


def _allreduce_unfused(grads):
    import torch.distributed as dist
    import warnings
    if not _exchange["warned_unfused"]:
        _exchange["warned_unfused"] = True
        warnings.warn("lightgaussian_b200: view-parallel backward outside the fused render() node -- gradients are summed with a dense "
                      "NCCL all-reduce (correct, slower than the sparse peer-memory exchange of the fused path)", stacklevel=3)
    _exchange["unfused_calls"] += 1
    from . import trace
    trace.bump("unfused_exchange")
    hs = [dist.all_reduce(g, op=dist.ReduceOp.SUM, group=_exchange["group"], async_op=True) for g in grads if g is not None and g.numel()]
    for h in hs:
        h.wait()


def _raw_grads_struct(xyz, dc, rest, scaling, rotation, opacity, rgb=None):
    return capi.LgrRawGrads(capi.ptr(xyz), capi.ptr(dc), capi.ptr(rest), capi.ptr(scaling), capi.ptr(rotation), capi.ptr(opacity),
                            capi.ptr(rgb))


class _RasterizeRawLeaves(torch.autograd.Function):
    """render()'s node when the fused path applies: inputs are the six leaves, gradients come back for the leaves."""

    @staticmethod
    def forward(ctx, xyz, means2D, dc, rest, scaling, rotation, opacity, raster_settings):
        _, _, R, color, radii, geom, binning, img, leaves = _forward_raw_native(False, raster_settings, xyz, dc, rest, scaling, rotation, opacity)
        ctx.raster_settings = raster_settings
        ctx.num_rendered = R
        ctx.deterministic = _last_deterministic[0]
        ctx.save_for_backward(*leaves, radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _):
        rs = ctx.raster_settings
        xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img = ctx.saved_tensors
        capi.set_deterministic(ctx.deterministic)   # the mode of the forward, whatever the flag says now
        world = _exchange["world"]
        exchange = world > 1 and xyz.size(0) != 0 and rest.size(1) > 0
        sparse_single = world == 1 and _os.environ.get("LGR_SPARSE_SINGLE", "0") == "1" and xyz.size(0) != 0 and rest.size(1) > 0
        stats = exchange and _exchange["densify"]
        xs = _sparse_exchange(xyz.device, xyz.size(0), world, _exchange["group"], stats=stats) if (exchange or sparse_single) else None
        if world > 1:
            _exchange["stats_record"] = None   # set again below when this backward publishes statistics
        if xs is not None:
            g, g2d = _backward_raw_sparse(xs, rs, ctx.num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom,
                                          binning, img, world)
        elif not exchange:
            g, g2d, _, _ = backward_raw_native(rs, ctx.num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii,
                                               geom, binning, img, compact=False)
        else:
            g, g2d = _backward_raw_exchange(rs, ctx.num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom,
                                            binning, img, world, _exchange["group"])
        return g[0], g2d, g[1], g[2], g[3], g[4], g[5], None


class _RasterizeRawLeavesAbs(torch.autograd.Function):
    """render()'s fused node under LGR_DENSIFY_GRAD=abs: _RasterizeRawLeaves whose backward goes through lgr_backward_raw_absgrad and
    sets `means2D.absgrad` ([P,2] float32, the sum over pixels of each pixel's |dL/dmean2D| term).  means2D.grad is unchanged."""

    @staticmethod
    def forward(ctx, xyz, means2D, dc, rest, scaling, rotation, opacity, raster_settings):
        color, radii = _RasterizeRawLeaves.forward(ctx, xyz, means2D, dc, rest, scaling, rotation, opacity, raster_settings)
        ctx.means2D = means2D   # render()'s screen-space placeholder, which the caller reads .absgrad from
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _):
        xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img = ctx.saved_tensors
        capi.set_deterministic(ctx.deterministic)   # refused by the forward; the library refuses it again if the flag changed since
        trace.bump("raw_backward_absgrad")
        g, g2d, absgrad = backward_raw_absgrad_native(ctx.raster_settings, ctx.num_rendered, grad_out_color, xyz, dc, rest, scaling,
                                                      rotation, opacity, radii, geom, binning, img)
        ctx.means2D.absgrad = absgrad
        return g[0], g2d, g[1], g[2], g[3], g[4], g[5], None


def absgrad_refusal() -> str | None:
    """Why the fused node cannot compute the absolute-gradient statistic under the current settings, or None.  Checked before any
    launch."""
    if capi.deterministic_requested():
        return "deterministic mode (LGR_DETERMINISTIC=1 or torch.use_deterministic_algorithms) has no absgrad (it needs fixed-order sums)"
    if capi.blend_mode() != 0:
        return "blend mode 1 (the round-1 blend kernels) has no absgrad"
    if _exchange["world"] > 1:
        return "the view-parallel gradient exchange has no absgrad backward"
    if _os.environ.get("LGR_SPARSE_SINGLE", "0") == "1":
        return "LGR_SPARSE_SINGLE=1 (the sparse single-GPU backward) has no absgrad backward"
    return None


def backward_raw_absgrad_native(rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img):
    """lgr_backward_raw_absgrad: six dense leaf gradients, dL/dmeans2D [P,3] and absgrad [P,2]."""
    lib = capi.load()
    device = xyz.device
    P, M = xyz.size(0), 1 + rest.size(1)
    H, W = grad_out_color.size(1), grad_out_color.size(2)
    g2d = torch.empty((P, 3), dtype=torch.float32, device=device)
    absgrad = torch.empty((P, 2), dtype=torch.float32, device=device)
    g = [torch.empty(t.shape, dtype=torch.float32, device=device) for t in (xyz, dc, rest, scaling, rotation, opacity)]
    if P != 0:
        dpix = _f32c(grad_out_color, "grad_out_color")
        with torch.cuda.device(device):
            view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                    rs.scale_modifier, rs.sh_degree, False, rs.debug)
            params, grads = _raw_struct(xyz, dc, rest, scaling, rotation, opacity), _raw_grads_struct(*g)
            st = lib.lgr_backward_raw_absgrad(C.byref(view), P, M, int(num_rendered), C.byref(params), radii.data_ptr(), geom.data_ptr(),
                                              binning.data_ptr(), img.data_ptr(), dpix.data_ptr(), C.byref(grads), g2d.data_ptr(),
                                              absgrad.data_ptr(), capi.current_stream_ptr(device))
        capi.check(st, "lgr_backward_raw_absgrad")
    return g, g2d, absgrad


def rasterize_raw_leaves_absgrad(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity, raster_settings):
    """(color, radii) of the fused node whose backward also sets means2D.absgrad.  Raises RuntimeError before any launch where the
    settings have no absgrad."""
    if raster_settings.f_count:
        raise RuntimeError("LGR_DENSIFY_GRAD=abs: count mode (raster_settings.f_count) has no absgrad")
    why = absgrad_refusal()
    if why is not None:
        raise RuntimeError(f"LGR_DENSIFY_GRAD=abs: {why}")
    return _RasterizeRawLeavesAbs.apply(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity, raster_settings)


DEPTH_MODES = {"z": 1, "inverse": 2}


def depth_alpha_refusal() -> str | None:
    """Why the fused node cannot return depth / alpha under the current settings, or None.  Checked before any launch."""
    if capi.deterministic_requested():
        return "deterministic mode (LGR_DETERMINISTIC=1 or torch.use_deterministic_algorithms) has no depth or alpha output"
    if capi.blend_mode() != 0:
        return "blend mode 1 (the round-1 blend kernels) has no depth or alpha output"
    if _exchange["world"] > 1:
        return "the view-parallel gradient exchange has no depth or alpha backward"
    if _os.environ.get("LGR_SPARSE_SINGLE", "0") == "1":
        return "LGR_SPARSE_SINGLE=1 (the sparse single-GPU backward) has no depth or alpha backward"
    return None


class _RasterizeRawLeavesDepth(torch.autograd.Function):
    """render(depth=..., alpha=...)'s node: _RasterizeRawLeaves plus the depth and alpha planes ([1,H,W] each; an empty placeholder
    for one that was not asked for).  The backward takes the existing lgr_backward_raw when neither plane received a gradient."""

    @staticmethod
    def forward(ctx, xyz, means2D, dc, rest, scaling, rotation, opacity, raster_settings, depth_mode, want_depth, want_alpha):
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        plane = lambda on: torch.empty((1, H, W), dtype=torch.float32, device=xyz.device) if on else None  # noqa: E731
        out_depth, out_alpha = plane(want_depth), plane(want_alpha)
        _, _, R, color, radii, geom, binning, img, leaves = _forward_raw_native(False, raster_settings, xyz, dc, rest, scaling, rotation,
                                                                                opacity, depth=(depth_mode, out_depth, out_alpha))
        ctx.raster_settings = raster_settings
        ctx.num_rendered = R
        ctx.depth_mode = depth_mode
        ctx.save_for_backward(*leaves, radii, geom, binning, img)
        ctx.set_materialize_grads(False)
        empty = lambda: torch.empty((0,), dtype=torch.float32, device=xyz.device)  # noqa: E731
        out_depth = out_depth if out_depth is not None else empty()
        out_alpha = out_alpha if out_alpha is not None else empty()
        ctx.mark_non_differentiable(radii)
        if not want_depth:
            ctx.mark_non_differentiable(out_depth)
        if not want_alpha:
            ctx.mark_non_differentiable(out_alpha)
        return color, radii, out_depth, out_alpha

    @staticmethod
    def backward(ctx, grad_out_color, _, grad_depth, grad_alpha):
        rs = ctx.raster_settings
        xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img = ctx.saved_tensors
        H, W = int(rs.image_height), int(rs.image_width)
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, H, W), dtype=torch.float32, device=xyz.device)
        if grad_depth is not None and grad_depth.numel() == 0:
            grad_depth = None
        if grad_alpha is not None and grad_alpha.numel() == 0:
            grad_alpha = None
        if grad_depth is None and grad_alpha is None:
            trace.bump("raw_backward_plain")
            g, g2d, _, _ = backward_raw_native(rs, ctx.num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii,
                                               geom, binning, img, compact=False)
        else:
            trace.bump("raw_backward_depth")
            g, g2d = backward_raw_depth_native(rs, ctx.num_rendered, grad_out_color, ctx.depth_mode, grad_depth, grad_alpha, xyz, dc,
                                               rest, scaling, rotation, opacity, radii, geom, binning, img)
        return g[0], g2d, g[1], g[2], g[3], g[4], g[5], None, None, None, None


def backward_raw_depth_native(rs, num_rendered, grad_out_color, depth_mode, grad_depth, grad_alpha, xyz, dc, rest, scaling, rotation,
                              opacity, radii, geom, binning, img):
    """lgr_backward_raw_depth: six dense leaf gradients and dL/dmeans2D; grad_depth / grad_alpha [1,H,W] or None (zero)."""
    lib = capi.load()
    device = xyz.device
    P, M = xyz.size(0), 1 + rest.size(1)
    H, W = grad_out_color.size(1), grad_out_color.size(2)
    g2d = torch.empty((P, 3), dtype=torch.float32, device=device)
    g = [torch.empty(t.shape, dtype=torch.float32, device=device) for t in (xyz, dc, rest, scaling, rotation, opacity)]
    if P != 0:
        dpix = _f32c(grad_out_color, "grad_out_color")
        gd = _f32c(grad_depth, "grad_depth") if grad_depth is not None else None
        ga = _f32c(grad_alpha, "grad_alpha") if grad_alpha is not None else None
        with torch.cuda.device(device):
            view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                    rs.scale_modifier, rs.sh_degree, False, rs.debug)
            params, grads = _raw_struct(xyz, dc, rest, scaling, rotation, opacity), _raw_grads_struct(*g)
            st = lib.lgr_backward_raw_depth(C.byref(view), P, M, int(num_rendered), C.byref(params), radii.data_ptr(), geom.data_ptr(),
                                            binning.data_ptr(), img.data_ptr(), dpix.data_ptr(), int(depth_mode), capi.ptr(gd), capi.ptr(ga),
                                            C.byref(grads), g2d.data_ptr(), capi.current_stream_ptr(device))
        capi.check(st, "lgr_backward_raw_depth")
    return g, g2d


def rasterize_raw_leaves_depth(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity, raster_settings, depth=None,
                               alpha=False):
    """(color, radii, depth, alpha) of the fused node: depth [1,H,W] when depth is "z" or "inverse" (else None), alpha [1,H,W] when
    alpha (else None).  Raises RuntimeError before any launch where the settings have no depth or alpha output."""
    if depth is not None and depth not in DEPTH_MODES:
        raise RuntimeError(f"depth={depth!r}: expected None, 'z' or 'inverse'")
    if raster_settings.f_count:
        raise RuntimeError("depth / alpha: count mode (raster_settings.f_count) has no depth or alpha output")
    mode = DEPTH_MODES.get(depth, 0)
    why = depth_alpha_refusal()
    if why is not None:
        raise RuntimeError(f"depth / alpha: {why}")
    color, radii, d, a = _RasterizeRawLeavesDepth.apply(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity,
                                                        raster_settings, mode, depth is not None, bool(alpha))
    return color, radii, (d if depth is not None else None), (a if alpha else None)


_side_streams = {}
_hp_streams = {}
_xtiming = {"on": __import__("os").environ.get("LGR_EXCHANGE_TIMING", "0") == "1", "rows": []}


def exchange_timing_report():
    """mean ms of (blend backward + extract, K7+K8, tail = exposed exchange) per exchange-mode backward (diagnostics)"""
    rows = []
    torch.cuda.synchronize()
    for ev in _xtiming["rows"][5:]:
        rows.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
    if not rows:
        return None
    t = torch.tensor(rows).mean(dim=0).tolist()
    return {"blend_bwd+extract_ms": t[0], "k8_ms": t[1], "exposed_exchange_ms": t[2], "n": len(rows)}


class _SymmExchange:
    """Persistent NVLink symmetric-memory buffers (torch.distributed._symmetric_memory) for the small-leaf all-reduce,
    reduced by OUR peer-memory kernel (lgr_peer_allreduce: P2P loads of this rank's slice from every peer, stores to every
    peer) between two cross-GPU barriers.  Two buffers alternate so that the gradients returned by step k stay valid while
    step k+1 is being written.  Any failure to set this up falls back to NCCL (agreed collectively in _symm_exchange)."""

    def __init__(self, device, P, world, group):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        if world > 8:
            raise RuntimeError("peer-memory all-reduce supports at most 8 ranks (one NVSwitch domain)")
        grp = group if group is not None else dist.group.WORLD
        self.group_name = grp.group_name
        self.capacity = P
        self.n = (P * 11 + 1023) // 1024 * 1024
        self.bufs = [symm_mem.empty(self.n, dtype=torch.float32, device=device) for _ in range(2)]
        self.hdls = [symm_mem.rendezvous(b, self.group_name) for b in self.bufs]
        for b in self.bufs:
            b.zero_()
        self.rank, self.world = int(self.hdls[0].rank), int(self.hdls[0].world_size)
        assert self.world == world
        self.ptr_tables = []
        for h in self.hdls:
            ptrs = [int(p) for p in h.buffer_ptrs]
            assert len(ptrs) == world and all(ptrs)
            self.ptr_tables.append((C.c_void_p * world)(*ptrs))
        self.mc_ptrs = [int(getattr(h, "multicast_ptr", 0) or 0) for h in self.hdls]
        import os
        self.mode = os.environ.get("LGR_EXCHANGE_REDUCE", "peer")
        if self.mode == "multimem" and not all(self.mc_ptrs):
            self.mode = "peer"
        self.turn = 0

    def next(self):
        self.turn ^= 1
        return self.bufs[self.turn]

    def all_reduce_(self, buf, stream):
        k = self.turn
        assert buf.data_ptr() == self.bufs[k].data_ptr()
        h = self.hdls[k]
        h.barrier(channel=0)      # every rank's K7+K8 has written its buffer
        if self.mode == "multimem" and self.mc_ptrs[k]:
            st = capi.load().lgr_multimem_allreduce(self.mc_ptrs[k], self.rank, self.world, self.n, stream.cuda_stream)
        else:
            st = capi.load().lgr_peer_allreduce(self.ptr_tables[k], self.rank, self.world, self.n, stream.cuda_stream)
        capi.check(st, "lgr_peer_allreduce")
        h.barrier(channel=1)      # every peer's stores into this rank's buffer have landed


_symm_cache = {}


def _symm_exchange(device, P, world, group):
    """collectively agreed: either every rank gets symmetric buffers or none does (then NCCL is used)"""
    import os
    import torch.distributed as dist
    # ONE exchange object per (device, world): P changes at every prune / densify event, and keying the cache by P pinned a fresh
    # pair of peer-mapped buffers per value for the life of the process.  The flat buffer is laid out from the call's P, so it is
    # reused exactly while P stays the same and replaced (the old one dropped) when P changes; every rank sees the same P.
    key = (str(device), world)
    cur = _symm_cache.get(key, "none")
    if cur == "none" or (cur is not None and cur.capacity != P):
        _symm_cache.pop(key, None)
        del cur
        xb, ok = None, 1
        # NCCL's all-reduce is the default: for this 132 MB payload the rebuild kernel competes for HBM with whichever reduction
        # runs, so our peer-memory and NVLS multimem kernels have no bandwidth to gain; LGR_EXCHANGE_REDUCE=peer|multimem selects ours.
        if os.environ.get("LGR_EXCHANGE_REDUCE", "nccl") == "nccl":
            ok = 0
        else:
            try:
                xb = _SymmExchange(device, P, world, group)
            except Exception as ex:  # noqa: BLE001  (no multicast / no P2P / API drift: NCCL still works)
                print(f"lightgaussian_b200: peer-memory all-reduce unavailable ({type(ex).__name__}: {ex}); using NCCL", flush=True)
                ok = 0
        flag = torch.tensor([ok], device=device, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        _symm_cache[key] = xb if int(flag.item()) == 1 else None
    return _symm_cache[key]


def _exchange_tables(bases, rank, slot_bytes, push):
    """The pointer tables of one rank of the sparse exchange, per buffer k (bases[k][q] = address of rank q's buffer k, as mapped on
    this rank): (pack_tables, ptr_tables) -- where this rank's packed view goes, and where the accumulate kernel reads view v.
      push: slot `rank` of every rank's buffer; view v is read from slot v of this rank's own buffer.
      pull: slot `rank` of this rank's own buffer only; view v is read from slot v of rank v's buffer."""
    world = len(bases[0])
    r = rank
    if push:
        pack = [(C.c_void_p * world)(*[t[q] + r * slot_bytes for q in range(world)]) for t in bases]
        ptrs = [(C.c_void_p * world)(*[t[r] + v * slot_bytes for v in range(world)]) for t in bases]
    else:
        pack = [(C.c_void_p * 1)(t[r] + r * slot_bytes) for t in bases]
        ptrs = [(C.c_void_p * world)(*[t[v] + v * slot_bytes for v in range(world)]) for t in bases]
    return pack, ptrs


class _SparseExchange:
    """Two alternating exchange buffers per rank in NVLink symmetric memory (torch.distributed._symmetric_memory), each mapped into every
    peer, for the sparse gradient exchange (csrc/lgr_sparse.cuh).  A buffer holds `world` slots; slot v carries view v's packed gradient
    (header | bitmap | prefix | 64-byte rows).
      push (default): rank r WRITES its packed view into slot r of every rank's buffer from inside the pack kernels (posted stores over
                      NVLink, overlapping the slower ranks' blend backward); after one barrier every rank accumulates from LOCAL memory.
      pull (LGR_EXCHANGE_PUSH=0, the round-1 scheme): rank r writes slot r of its OWN buffer only; after the barrier the accumulate
                      kernel loads every peer's slot over NVLink.
    Buffer k of step s is rewritten at step s+2; every rank passes the barrier of step s+1 only after its accumulate kernel of step s
    has finished, so one cross-GPU barrier per step is enough.  world == 1 (tests): plain device tensors, no barrier.
    stats=True: slots of lgr_sparse_exchange_bytes_stats, which also carry each view's densification statistics."""

    def __init__(self, device, P, world, group, stats=False):
        lib = capi.load()
        if world > 8:
            raise RuntimeError("the sparse peer-memory exchange supports at most 8 ranks (one NVSwitch domain)")
        self.world = world
        self.capacity = P          # the layout inside a slot is computed from each call's P <= capacity
        self.stats = bool(stats)
        self.push = world > 1 and _os.environ.get("LGR_EXCHANGE_PUSH", "1") != "0"
        nbytes = lib.lgr_sparse_exchange_bytes_stats(P) if self.stats else lib.lgr_sparse_exchange_bytes(P)
        slot = (int(nbytes) + 255) // 256 * 256
        n = world * slot // 4
        self.ws = torch.empty(int(lib.lgr_sparse_workspace_bytes(P)), dtype=torch.uint8, device=device)
        if world > 1:
            import torch.distributed as dist
            import torch.distributed._symmetric_memory as symm_mem
            grp = group if group is not None else dist.group.WORLD
            self.bufs = [symm_mem.empty(n, dtype=torch.float32, device=device) for _ in range(2)]
            self.hdls = [symm_mem.rendezvous(b, grp.group_name) for b in self.bufs]
            assert int(self.hdls[0].world_size) == world
            self.rank = int(self.hdls[0].rank)
            bases = [[int(p) for p in h.buffer_ptrs] for h in self.hdls]
        else:
            self.bufs = [torch.empty(n, dtype=torch.float32, device=device) for _ in range(2)]
            self.hdls = [None, None]
            self.rank = 0
            bases = [[b.data_ptr()] for b in self.bufs]
        for b in self.bufs:
            b.zero_()
        for t in bases:
            assert len(t) == world and all(t) and all(p % 256 == 0 for p in t)
        self.pack_tables, self.ptr_tables = _exchange_tables(bases, self.rank, slot, self.push)
        self.slot_bytes = slot
        self.turn = 0

    def next(self):
        self.turn ^= 1
        return self.turn

    def rows_published(self) -> int:
        """rows this rank packed in its last backward (diagnostics)"""
        k, r = self.turn, self.rank
        off = r * self.slot_bytes // 4
        return int(self.bufs[k][off + 3:off + 4].view(torch.int32).item())


_sparse_cache = {}


def _sparse_exchange(device, P, world, group, stats=False):
    """collectively agreed: either every rank gets the peer-mapped buffers or none does (then the dense NCCL exchange is used).
    LGR_EXCHANGE=dense selects the dense exchange explicitly.  stats: slots that carry the densification statistics (every rank asks
    for the same, enable_gradient_exchange's densification flag)."""
    # ONE exchange object per (device, world), sized for a capacity >= P (kernels lay the buffer out from the call's P): P shrinks at
    # every prune event and may grow when densifying; only growth beyond the capacity re-allocates (x1.25, the old buffers are
    # dropped first), so a training run no longer pins a new pair of peer-mapped buffers per distinct P.
    key = (str(device), world)
    cur = _sparse_cache.get(key, "none")
    if cur == "none" or (cur is not None and (cur.capacity < P or cur.stats != bool(stats))):
        grow = cur != "none" and cur is not None and cur.capacity < P
        cap = max(int(P * 1.25), P) if grow else (P if cur == "none" else max(P, cur.capacity))
        _sparse_cache.pop(key, None)
        del cur
        xs, ok = None, 1
        if _os.environ.get("LGR_EXCHANGE", "sparse") != "sparse":
            ok = 0
        else:
            try:
                xs = _SparseExchange(device, cap, world, group, stats=stats)
            except Exception as ex:  # noqa: BLE001  (no P2P / API drift: the NCCL path still works)
                print(f"lightgaussian_b200: sparse peer-memory exchange unavailable ({type(ex).__name__}: {ex}); using the dense NCCL exchange", flush=True)
                ok = 0
        if world > 1:
            import torch.distributed as dist
            flag = torch.tensor([ok], device=device, dtype=torch.int32)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
            ok = int(flag.item())
        _sparse_cache[key] = xs if ok == 1 else None
    return _sparse_cache[key]


def exchange_info(world):
    """("sparse-p2p" | "dense-nccl" | "none", rows published by this rank in its last backward or None) -- diagnostics for bench.py"""
    if world <= 1:
        return "none", None
    for (dev, w), xs in _sparse_cache.items():
        if w == world and xs is not None:
            return ("sparse-p2p-push" if xs.push else "sparse-p2p"), xs.rows_published()
    return "dense-nccl", None


def _backward_raw_sparse(xs, rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img, world):
    """View-parallel backward with the sparse exchange: blend backward | flag + scan + per-Gaussian backward of the ~13 % of Gaussians with a
    non-zero gradient, published in peer-mapped memory | one cross-GPU barrier | every rank reads all views' rows over NVLink and writes the
    dense, summed leaf gradients (bit-identical on every rank).  No NCCL call, no host synchronisation."""
    device = xyz.device
    P = xyz.size(0)
    g2d = torch.empty((P, 3), dtype=torch.float32, device=device)
    g = [torch.empty(t.shape, dtype=torch.float32, device=device) for t in (xyz, dc, rest, scaling, rotation, opacity)]
    k = xs.next()
    serial = None
    if xs.stats:
        # densification statistics ride in the slots; the statistics call of this step reads buffer k before the next step's barrier
        _exchange["serial"] = serial = (_exchange["serial"] + 1) & 0xFFFFFFFF
    with torch.cuda.device(device):
        _sparse_pack(xs, k, rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img, g2d,
                     serial=serial)
        if world > 1:
            xs.hdls[k].barrier(channel=0)          # every rank's rows of this step are published
        _sparse_accumulate(xs, k, int(rs.sh_degree), world, xyz, rest, g)
    if serial is not None:
        _exchange["stats_record"] = dict(xs=xs, k=k, serial=serial, P=P, device=device)
    return g, g2d


def _sparse_pack(xs, k, rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img, g2d,
                 serial=None):
    """First half of the sparse backward, on the current stream of xyz's device: blend backward, then flag + scan + per-Gaussian backward
    of the flagged Gaussians into this rank's slot of exchange buffer k (every rank's, in push mode).  Writes this view's dL/dmeans2D
    into g2d [P,3].  serial (an exchange built with stats=True): the slot also carries this view's densification statistics, stamped
    with the step serial."""
    lib = capi.load()
    device = xyz.device
    P, M = xyz.size(0), 1 + rest.size(1)
    H, W = grad_out_color.size(1), grad_out_color.size(2)
    dpix = _f32c(grad_out_color, "grad_out_color")
    stream = capi.current_stream_ptr(device)
    view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W, rs.scale_modifier,
                            rs.sh_degree, False, rs.debug)
    st = lib.lgr_backward_raw_begin(C.byref(view), P, int(num_rendered), radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                                    img.data_ptr(), dpix.data_ptr(), None, stream)
    capi.check(st, "lgr_backward_raw_begin")
    params = _raw_struct(xyz, dc, rest, scaling, rotation, opacity)
    if serial is None:
        st = lib.lgr_backward_raw_sparse_pack_push(C.byref(view), P, M, C.byref(params), radii.data_ptr(), geom.data_ptr(), xs.pack_tables[k],
                                                   len(xs.pack_tables[k]), xs.rank if xs.push else 0, xs.ws.data_ptr(), g2d.data_ptr(), stream)
        capi.check(st, "lgr_backward_raw_sparse_pack_push")
        return
    stats = capi.LgrSparseStats(int(serial) & 0xFFFFFFFF)
    st = lib.lgr_backward_raw_sparse_pack_push_ex(C.byref(view), P, M, C.byref(params), radii.data_ptr(), geom.data_ptr(), xs.pack_tables[k],
                                                  len(xs.pack_tables[k]), xs.rank if xs.push else 0, xs.ws.data_ptr(), g2d.data_ptr(),
                                                  C.byref(stats), stream)
    capi.check(st, "lgr_backward_raw_sparse_pack_push_ex")


def _sparse_accumulate(xs, k, sh_degree, world, xyz, rest, g):
    """Second half, once every rank's view is in buffer k: the six dense leaf gradients g (list of [P,...] float32 tensors), summed
    over the `world` views in rank order."""
    lib = capi.load()
    P, M = xyz.size(0), 1 + rest.size(1)
    grads = _raw_grads_struct(*g)
    st = lib.lgr_backward_raw_sparse_accumulate(P, M, int(sh_degree), world, xs.ptr_tables[k], xyz.data_ptr(), C.byref(grads),
                                                capi.current_stream_ptr(xyz.device))
    capi.check(st, "lgr_backward_raw_sparse_accumulate")


def _exchange_chunks(P):
    """[(first, count)] ranges of Gaussians, boundaries at multiples of 256.  LGR_EXCHANGE_CHUNKS ranges; default 1 = one all-reduce
    after the whole K7+K8: with more ranges the NCCL kernels of the earlier ranges take SMs and HBM bandwidth from the ranges still
    being computed."""
    import os
    n = max(1, int(os.environ.get("LGR_EXCHANGE_CHUNKS", "1")))
    blocks = (P + 255) // 256
    n = min(n, blocks)
    out, b0 = [], 0
    for c in range(n):
        b1 = blocks * (c + 1) // n
        if b1 > b0:
            out.append((b0 * 256, min(P, b1 * 256) - b0 * 256))
        b0 = b1
    return out


def _backward_raw_exchange(rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img, world, grp):
    """The view-parallel backward: every collective is issued as early as its input exists so that it overlaps kernels.

        main stream :  blend backward + dRGB extract | K7+K8 (small leaves -> flat)            | wait
        NCCL stream :                                | all-gather dRGB, campos | all-reduce flat |
        side stream :                                                          | rebuild SH gradient from all views |
    """
    import torch.distributed as dist
    lib = capi.load()
    device = xyz.device
    P, M = xyz.size(0), 1 + rest.size(1)
    H, W = grad_out_color.size(1), grad_out_color.size(2)
    g2d = torch.empty((P, 3), dtype=torch.float32, device=device)
    xb = _symm_exchange(device, P, world, grp)
    flat_full = xb.next() if xb is not None else torch.empty(P * 11, dtype=torch.float32, device=device)
    flat = flat_full[:P * 11]                                         # rotation first: keeps it 16-byte aligned
    g_rot, g_xyz = flat[:4 * P].view(P, 4), flat[4 * P:7 * P].view(P, 3)
    g_scal, g_op = flat[7 * P:10 * P].view(P, 3), flat[10 * P:].view(P, 1)
    d_rgb = torch.empty((P, 3), dtype=torch.float32, device=device)
    all_rgb = torch.empty((world, P, 3), dtype=torch.float32, device=device)
    all_cam = torch.empty((world, 3), dtype=torch.float32, device=device)
    d_dc, d_rest = torch.empty(dc.shape, dtype=torch.float32, device=device), torch.empty(rest.shape, dtype=torch.float32, device=device)
    dpix = _f32c(grad_out_color, "grad_out_color")
    main = torch.cuda.current_stream(device)
    side = _side_streams.setdefault(str(device), torch.cuda.Stream(device=device))
    with torch.cuda.device(device):
        view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W, rs.scale_modifier,
                                rs.sh_degree, False, rs.debug)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)] if _xtiming["on"] else None
        if ev:
            ev[0].record(main)
        st = lib.lgr_backward_raw_begin(C.byref(view), P, int(num_rendered), radii.data_ptr(), geom.data_ptr(), binning.data_ptr(),
                                        img.data_ptr(), dpix.data_ptr(), d_rgb.data_ptr(), main.cuda_stream)
        capi.check(st, "lgr_backward_raw_begin")
        if ev:
            ev[1].record(main)
        w_rgb = dist.all_gather_into_tensor(all_rgb, d_rgb, group=grp, async_op=True)          # overlaps K7+K8 below
        w_cam = dist.all_gather_into_tensor(all_cam, keep[3].reshape(1, 3), group=grp, async_op=True)
        params = _raw_struct(xyz, dc, rest, scaling, rotation, opacity)
        grads = _raw_grads_struct(g_xyz, None, None, g_scal, g_rot, g_op, rgb=None)
        # optional (LGR_EXCHANGE_CHUNKS > 1, measured slower, see _exchange_chunks): K7+K8 in ranges of Gaussians, the all-reduce of one
        # range's small-leaf gradients (four slices of the flat buffer, coalesced into one NCCL launch) overlapping the next range
        chunks = _exchange_chunks(P) if xb is None else [(0, P)]
        w_flat = []
        for (c0, cn) in chunks:
            st = lib.lgr_backward_raw_end_range(C.byref(view), P, M, C.byref(params), radii.data_ptr(), geom.data_ptr(), C.byref(grads),
                                                g2d.data_ptr(), c0, cn, main.cuda_stream)
            capi.check(st, "lgr_backward_raw_end_range")
            if xb is None:
                if len(chunks) == 1:
                    w_flat.append(dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=grp, async_op=True))
                else:
                    with dist.distributed_c10d._coalescing_manager(group=grp, device=device, async_ops=True) as cm:
                        for t in (g_rot, g_xyz, g_scal, g_op):
                            dist.all_reduce(t[c0:c0 + cn], op=dist.ReduceOp.SUM, group=grp)
                    w_flat.append(cm)
        if ev:
            ev[2].record(main)
        # critical path first: the small-leaf reduction runs on a HIGH-priority stream so that its blocks are scheduled ahead
        # of the bandwidth-hungry rebuild kernel that overlaps it
        if xb is not None:
            hp = _hp_streams.setdefault(str(device), torch.cuda.Stream(device=device, priority=-1))
            hp.wait_stream(main)
            with torch.cuda.stream(hp):
                xb.all_reduce_(flat_full, hp)  # our peer-memory reduction over NVLink
        with torch.cuda.stream(side):                                                            # overlaps the all-reduce
            w_rgb.wait()
            w_cam.wait()
            st = lib.lgr_sh_grad_from_views(P, M, int(rs.sh_degree), world, xyz.data_ptr(), all_cam.data_ptr(), all_rgb.data_ptr(),
                                            d_dc.data_ptr(), d_rest.data_ptr(), side.cuda_stream)
            capi.check(st, "lgr_sh_grad_from_views")
        if xb is not None:
            main.wait_stream(hp)
        else:
            for w in w_flat:
                w.wait()
        main.wait_stream(side)
        if ev:
            ev[3].record(main)
            _xtiming["rows"].append(ev)
    return [g_xyz, d_dc, d_rest, g_scal, g_rot, g_op], g2d


def backward_raw_native(rs, num_rendered, grad_out_color, xyz, dc, rest, scaling, rotation, opacity, radii, geom, binning, img,
                        compact=False):
    """lgr_backward_raw.  compact=False: six dense leaf gradients.  compact=True: the SH leaves are NOT written; instead the
    clamp-masked dL/dRGB [P,3] of this view is returned, and the four small leaves live in one flat buffer (one all-reduce)."""
    lib = capi.load()
    device = xyz.device
    P, M = xyz.size(0), 1 + rest.size(1)
    H, W = grad_out_color.size(1), grad_out_color.size(2)
    g2d = torch.empty((P, 3), dtype=torch.float32, device=device)
    flat = d_rgb = None
    if compact:
        flat = torch.empty(P * 11, dtype=torch.float32, device=device)   # rotation first: keeps it 16-byte aligned
        g_rot, g_xyz = flat[:4 * P].view(P, 4), flat[4 * P:7 * P].view(P, 3)
        g_scal, g_op = flat[7 * P:10 * P].view(P, 3), flat[10 * P:].view(P, 1)
        d_rgb = torch.empty((P, 3), dtype=torch.float32, device=device)
        g = [g_xyz, None, None, g_scal, g_rot, g_op]
    else:
        g = [torch.empty(t.shape, dtype=torch.float32, device=device) for t in (xyz, dc, rest, scaling, rotation, opacity)]
    if P != 0:
        dpix = _f32c(grad_out_color, "grad_out_color")
        with torch.cuda.device(device):
            view, keep = _make_view(device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H, W,
                                    rs.scale_modifier, rs.sh_degree, False, rs.debug)
            params, grads = _raw_struct(xyz, dc, rest, scaling, rotation, opacity), _raw_grads_struct(*g, rgb=d_rgb)
            st = lib.lgr_backward_raw(C.byref(view), P, M, int(num_rendered), C.byref(params), radii.data_ptr(), geom.data_ptr(),
                                      binning.data_ptr(), img.data_ptr(), dpix.data_ptr(), C.byref(grads), g2d.data_ptr(),
                                      capi.current_stream_ptr(device))
        capi.check(st, "lgr_backward_raw")
    return g, g2d, d_rgb, flat


def sh_grad_from_views(xyz, campos_all, d_rgb_all, dc_like, rest_like, sh_degree):
    """sum over views of basis(dir_v) (x) dRGB_v  ->  (d_features_dc, d_features_rest)   (lgr_sh_grad_from_views)"""
    lib = capi.load()
    P, M = xyz.size(0), 1 + rest_like.size(1)
    d_dc, d_rest = torch.empty_like(dc_like), torch.empty_like(rest_like)
    if P != 0:
        with torch.cuda.device(xyz.device):
            st = lib.lgr_sh_grad_from_views(P, M, int(sh_degree), int(campos_all.size(0)), xyz.data_ptr(), campos_all.contiguous().data_ptr(),
                                            d_rgb_all.contiguous().data_ptr(), d_dc.data_ptr(), d_rest.data_ptr(),
                                            capi.current_stream_ptr(xyz.device))
        capi.check(st, "lgr_sh_grad_from_views")
    return d_dc, d_rest


def rasterize_raw_leaves(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity, raster_settings, blend_weight=None):
    """(color, radii) or, in count mode, (gaussians_count, important_score, color, radii) -- same as rasterize_gaussians."""
    if raster_settings.f_count:
        count, score, _, color, radii, _, _, _, _ = _forward_raw_native(True, raster_settings, xyz.detach(), features_dc.detach(),
                                                                        features_rest.detach(), scaling.detach(), rotation.detach(),
                                                                        opacity.detach(), blend_weight)
        return count, score, color, radii
    if blend_weight is not None:
        raise RuntimeError("blend_weight is a count-mode output (raster_settings.f_count)")
    return _RasterizeRawLeaves.apply(xyz, means2D, features_dc, features_rest, scaling, rotation, opacity, raster_settings)


_fused_ok = {}


def fused_activations_match_torch(device) -> bool:
    """One-time self-check per device: the in-kernel activations are only used when they reproduce this torch build's
    exp / sigmoid / F.normalize bit for bit (otherwise render() silently keeps the unfused path)."""
    key = str(device)
    if key not in _fused_ok:
        g = torch.Generator().manual_seed(1)
        P = 4096
        raw = dict(xyz=torch.randn(P, 3, generator=g), dc=torch.randn(P, 1, 3, generator=g), rest=torch.randn(P, 15, 3, generator=g) * 0.2,
                   scaling=torch.randn(P, 3, generator=g) * 0.5 - 4.0, rotation=torch.randn(P, 4, generator=g), opacity=torch.randn(P, 1, generator=g) * 2)
        raw = {k: v.to(device) for k, v in raw.items()}
        eye = torch.eye(4, device=device)
        view = eye.clone(); view[3, 2] = 4.0
        proj = view.clone(); proj[2, 3] = 1.0
        rs = GaussianRasterizationSettings(64, 64, 0.6, 0.6, torch.zeros(3, device=device), 1.0, view, proj, 3, torch.zeros(3, device=device),
                                           False, False, False)
        with torch.no_grad():
            a = _forward_raw_native(False, rs, raw["xyz"], raw["dc"], raw["rest"], raw["scaling"], raw["rotation"], raw["opacity"])
            act = (rs.bg, raw["xyz"], torch.Tensor([]), torch.sigmoid(raw["opacity"]), torch.exp(raw["scaling"]),
                   torch.nn.functional.normalize(raw["rotation"]), 1.0, torch.Tensor([]), view, proj, 0.6, 0.6, 64, 64,
                   torch.cat((raw["dc"], raw["rest"]), dim=1), 3, rs.campos, False, False)
            b = _C.rasterize_gaussians(*act)
        _fused_ok[key] = bool(torch.equal(a[3], b[1]) and torch.equal(a[4], b[2]) and a[2] == b[0])
    return _fused_ok[key]
