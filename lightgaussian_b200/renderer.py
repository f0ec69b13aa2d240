"""render() / count_render() with the reference's signatures and return dictionaries
(reference gaussian_renderer/__init__.py:22-124 and :127-229).  The two differ only in f_count and the two
extra outputs, so both go through one helper here.

`pc` is anything with GaussianModel's getters (scene/gaussian_model.py:98-118): get_xyz, get_opacity,
get_scaling, get_rotation, get_features, active_sh_degree, max_sh_degree and, for
pipe.compute_cov3D_python, get_covariance(scaling_modifier).
"""
from __future__ import annotations

import math

import torch

import os

import torch.nn.functional as F

from . import trace

from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_raw_leaves, fused_activations_match_torch,
                         rest_row_stride, forward_vq_native, rasterize_raw_leaves_depth, depth_alpha_refusal, DEPTH_MODES,
                         rasterize_raw_leaves_absgrad, absgrad_refusal, camera_grad_refusal)

_LEAVES = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")

SIGNIFICANCE_MODES = ("count", "blend_weight")
WEIGHT_SCALE = 2.0 ** -32   # resolution of the fixed-point blending weight (include/lgrast.h, lgr_forward_count_weight)


def significance_mode() -> str:
    """LGR_SIGNIFICANCE, read at call time: "count" (unset; the reference's opacity * count) or "blend_weight" (sum of alpha * T)."""
    mode = os.environ.get("LGR_SIGNIFICANCE", "count")
    if mode not in SIGNIFICANCE_MODES:
        raise RuntimeError(f"LGR_SIGNIFICANCE={mode!r}: expected one of {', '.join(SIGNIFICANCE_MODES)}")
    return mode


DENSIFY_GRAD_MODES = ("grad", "abs")


def densify_grad_mode() -> str:
    """LGR_DENSIFY_GRAD, read at call time: "grad" (unset; the reference's ||sum_p dL_p/dmean2D||) or "abs" (AbsGS / gsplat absgrad:
    render() sets viewspace_points.absgrad = sum_p |dL_p/dmean2D| and add_densification_stats accumulates its norm)."""
    mode = os.environ.get("LGR_DENSIFY_GRAD", "grad")
    if mode not in DENSIFY_GRAD_MODES:
        raise RuntimeError(f"LGR_DENSIFY_GRAD={mode!r}: expected one of {', '.join(DENSIFY_GRAD_MODES)}")
    return mode


def weight_score(blend_weight_fx: torch.Tensor) -> torch.Tensor:
    """float32 score of int64 fixed-point blending weights: float32(float64(fx) * 2^-32)."""
    return (blend_weight_fx.to(torch.float64) * WEIGHT_SCALE).to(torch.float32)


def _can_fuse(pc, pipe, override_color, dense_copies=False) -> bool:
    """The fused path needs GaussianModel-style raw leaves with the standard activations
    (scene/gaussian_model.py:35-43: exp / sigmoid / normalize) and the default pipeline flags.  dense_copies: the caller hands
    non-contiguous leaves to the fused node as contiguous copies (_dense_leaves), so their layout does not matter."""
    if os.environ.get("LGR_FUSED", "1") == "0" or override_color is not None:
        return False
    if pipe.convert_SHs_python or pipe.compute_cov3D_python:
        return False
    if not all(hasattr(pc, n) for n in _LEAVES):
        return False
    if getattr(pc, "scaling_activation", torch.exp) is not torch.exp:
        return False
    if getattr(pc, "opacity_activation", torch.sigmoid) is not torch.sigmoid:
        return False
    if getattr(pc, "rotation_activation", F.normalize) is not F.normalize:
        return False
    t = pc._xyz
    # every leaf dense, except that _features_rest may be a row-strided view: the distillation student's
    # `_features_rest[:, :8, :]` (scene/gaussian_model.py:129-136) is read in place through its row stride
    if not (t.is_cuda and all(getattr(pc, n).dtype == torch.float32
                              and (dense_copies or getattr(pc, n).is_contiguous() or n == "_features_rest") for n in _LEAVES)):
        return False
    if pc._features_rest.dim() != 3 or pc._features_dc.shape[1] != 1 or pc._features_rest.shape[1] < 1:
        return False
    if not dense_copies and not pc._features_rest.is_contiguous() and rest_row_stride(pc._features_rest) == 0:
        return False
    if (pc.active_sh_degree + 1) ** 2 > 1 + pc._features_rest.shape[1]:
        return False
    return fused_activations_match_torch(t.device)

def _dense_leaves(pc):
    """the six leaves for the fused node, each non-contiguous one (create_from_pcd's permuted _xyz) as a contiguous copy whose gradient
    autograd routes back to the leaf; a row-strided _features_rest the kernels read in place stays as it is"""
    out = []
    for n in _LEAVES:
        t = getattr(pc, n)
        keep = t.is_contiguous() or (n == "_features_rest" and rest_row_stride(t) != 0)
        out.append(t if keep else t.contiguous())
    return out


def _resident_store(pc, pipe, override_color):
    """The resident VQ store of `pc` (vqresident.py) when this call can render the compressed model in place: a forward without
    gradients, default pipeline flags, SH colours and the standard activations.  Looks only at `pc._vq_resident` and `pc._xyz`, so
    the deferred leaves stay unread; in every other case the caller's first read of a leaf materialises them."""
    store = getattr(pc, "_vq_resident", None)
    if store is None or torch.is_grad_enabled() or override_color is not None:
        return None
    if os.environ.get("LGR_FUSED", "1") == "0" or pipe.convert_SHs_python or pipe.compute_cov3D_python:
        return None
    if (getattr(pc, "scaling_activation", torch.exp) is not torch.exp or getattr(pc, "opacity_activation", torch.sigmoid) is not torch.sigmoid
            or getattr(pc, "rotation_activation", F.normalize) is not F.normalize):
        return None
    xyz = pc._xyz
    if not (xyz.is_cuda and xyz.dtype == torch.float32 and xyz.is_contiguous() and tuple(xyz.shape) == (store.P, 3)
            and xyz.device == store.slot.device):
        return None
    if (pc.active_sh_degree + 1) ** 2 > store.D // 3:
        return None
    return store if fused_activations_match_torch(xyz.device) else None


_SH_C0 = 0.28209479177387814
_SH_C1 = 0.4886025119029199
_SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435)


def eval_sh_torch(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """PyTorch SH evaluation for pipe.convert_SHs_python (the role of utils/sh_utils.py:57-120).
    sh: [..., C, (max_deg+1)^2], dirs: [..., 3] unit vectors -> [..., C]."""
    out = _SH_C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        out = out - _SH_C1 * y * sh[..., 1] + _SH_C1 * z * sh[..., 2] - _SH_C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            out = (out + _SH_C2[0] * xy * sh[..., 4] + _SH_C2[1] * yz * sh[..., 5] + _SH_C2[2] * (2.0 * zz - xx - yy) * sh[..., 6]
                   + _SH_C2[3] * xz * sh[..., 7] + _SH_C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                out = (out + _SH_C3[0] * y * (3 * xx - yy) * sh[..., 9] + _SH_C3[1] * xy * z * sh[..., 10]
                       + _SH_C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + _SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                       + _SH_C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + _SH_C3[5] * z * (xx - yy) * sh[..., 14]
                       + _SH_C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return out


def _unfused_reason(pc, pipe, override_color) -> str:
    """why _can_fuse refused, for the depth / alpha error message"""
    if override_color is not None:
        return "override_color"
    if os.environ.get("LGR_FUSED", "1") == "0":
        return "LGR_FUSED=0"
    if pipe.convert_SHs_python or pipe.compute_cov3D_python:
        return "pipe.convert_SHs_python / pipe.compute_cov3D_python"
    return "a model without GaussianModel's raw float32 CUDA leaves and standard activations (exp / sigmoid / normalize)"


def _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, f_count, weight=False, depth=None, alpha=False,
            camera_grad=False):
    planes = depth is not None or alpha
    # LGR_DENSIFY_GRAD=abs: the training render's backward also produces viewspace_points.absgrad; checked before anything is read
    absgrad = not f_count and densify_grad_mode() == "abs" and torch.is_grad_enabled()
    # camera_grad: the camera tensors become inputs of the fused node (only meaningful with gradients); checked before any launch
    cam_grad = bool(camera_grad) and torch.is_grad_enabled()
    if cam_grad:
        if absgrad:
            raise RuntimeError("render(camera_grad=True): LGR_DENSIFY_GRAD=abs has no camera gradients")
        if not _can_fuse(pc, pipe, override_color):
            raise RuntimeError(f"render(camera_grad=True) needs the fused path, which {_unfused_reason(pc, pipe, override_color)} rules out")
        why = camera_grad_refusal(viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform,
                                  viewpoint_camera.camera_center)
        if why is not None:
            raise RuntimeError(f"render(camera_grad=True): {why}")
    if absgrad:
        if planes:
            raise RuntimeError("LGR_DENSIFY_GRAD=abs cannot be combined with render(depth=..., alpha=...)")
        if not _can_fuse(pc, pipe, override_color, dense_copies=True):
            raise RuntimeError(f"LGR_DENSIFY_GRAD=abs needs the fused path, which {_unfused_reason(pc, pipe, override_color)} rules out")
        why = absgrad_refusal()
        if why is not None:
            raise RuntimeError(f"LGR_DENSIFY_GRAD=abs: {why}")
    if planes:
        # checked before anything is read or launched; a resident VQ model takes the leaf path below (its leaves materialise)
        if depth is not None and depth not in DEPTH_MODES:
            raise RuntimeError(f"render(depth={depth!r}): expected None, 'z' or 'inverse'")
        if not _can_fuse(pc, pipe, override_color):
            raise RuntimeError(f"render(depth=..., alpha=...) needs the fused path, which {_unfused_reason(pc, pipe, override_color)} rules out")
        why = depth_alpha_refusal()
        if why is not None:
            raise RuntimeError(f"render(depth=..., alpha=...): {why}")
    xyz = pc.get_xyz
    # weight: count mode that also returns the view's fixed-point blending weights (int64 [P], fully written by the forward)
    blend_weight = torch.empty((xyz.shape[0],), dtype=torch.int64, device=xyz.device) if weight else None
    # grad placeholder for the screen-space means, as the reference builds it (:37-46)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass

    settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height),
        image_width=int(viewpoint_camera.image_width),
        tanfovx=math.tan(viewpoint_camera.FoVx * 0.5),
        tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
        bg=bg_color,
        scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform,
        projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=pc.active_sh_degree,
        campos=viewpoint_camera.camera_center,
        prefiltered=False,
        debug=pipe.debug,
        f_count=f_count,
    )
    if absgrad:
        trace.bump("render_fused")
        trace.bump("render_absgrad")
        xyz_, dc, rest, scaling, rotation, opacity = _dense_leaves(pc)
        outputs = rasterize_raw_leaves_absgrad(xyz_, screenspace_points, dc, rest, scaling, rotation, opacity, settings)
        return _package(outputs, screenspace_points, f_count)
    if planes or cam_grad:
        if planes:
            trace.bump("render_depth_alpha")
        if cam_grad:
            trace.bump("render_camera_grad")
        color, radii, d, a = rasterize_raw_leaves_depth(pc._xyz, screenspace_points, pc._features_dc, pc._features_rest, pc._scaling,
                                                        pc._rotation, pc._opacity, settings, depth, alpha, cam_grad)
        result = _package((color, radii), screenspace_points, False)
        if d is not None:
            result["depth"] = d
        if a is not None:
            result["alpha"] = a
        return result
    store = _resident_store(pc, pipe, override_color)
    if store is not None:
        trace.bump("render_vq_resident")
        count, score, color, radii = forward_vq_native(f_count, settings, pc._xyz.detach(), store, blend_weight)
        return _package((count, score, color, radii) if f_count else (color, radii), screenspace_points, f_count, blend_weight)
    if _can_fuse(pc, pipe, override_color):
        trace.bump("render_fused")
        if not pc._features_rest.is_contiguous():
            trace.bump("render_fused_strided_rest")
        outputs = rasterize_raw_leaves(pc._xyz, screenspace_points, pc._features_dc, pc._features_rest, pc._scaling, pc._rotation,
                                       pc._opacity, settings, blend_weight)
        return _package(outputs, screenspace_points, f_count, blend_weight)

    trace.bump("render_unfused")
    rasterizer = GaussianRasterizer(raster_settings=settings)

    geometry = dict(scales=None, rotations=None, cov3D_precomp=None)
    if pipe.compute_cov3D_python:
        geometry["cov3D_precomp"] = pc.get_covariance(scaling_modifier)
    else:
        geometry["scales"], geometry["rotations"] = pc.get_scaling, pc.get_rotation

    appearance = dict(shs=None, colors_precomp=None)
    if override_color is not None:
        appearance["colors_precomp"] = override_color
    elif pipe.convert_SHs_python:
        feats = pc.get_features
        shs_view = feats.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
        dirs = xyz - viewpoint_camera.camera_center.repeat(feats.shape[0], 1)
        dirs = dirs / dirs.norm(dim=1, keepdim=True)
        appearance["colors_precomp"] = torch.clamp_min(eval_sh_torch(pc.active_sh_degree, shs_view, dirs) + 0.5, 0.0)
    else:
        appearance["shs"] = pc.get_features

    if blend_weight is not None:
        outputs = rasterizer.forward_count(means3D=xyz, means2D=screenspace_points, opacities=pc.get_opacity, **appearance, **geometry,
                                           blend_weight=blend_weight)
    else:
        outputs = rasterizer(means3D=xyz, means2D=screenspace_points, opacities=pc.get_opacity, **appearance, **geometry)
    return _package(outputs, screenspace_points, f_count, blend_weight)


def _package(outputs, screenspace_points, f_count, blend_weight=None):
    if f_count:
        gaussians_count, important_score, rendered_image, radii = outputs
    else:
        rendered_image, radii = outputs
    result = {
        "render": rendered_image,
        "viewspace_points": screenspace_points,
        "visibility_filter": radii > 0,
        "radii": radii,
    }
    if f_count:
        result["gaussians_count"] = gaussians_count
        result["important_score"] = important_score
    if blend_weight is not None:
        result["important_score"] = weight_score(blend_weight)
        result["blend_weight_fx"] = blend_weight
    return result


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, *, depth=None, alpha=False,
           camera_grad=False):
    """Render the scene.  Background tensor (bg_color) must be on the GPU.
    depth="z" / "inverse" adds "depth", and alpha=True adds "alpha", to the result: [1,H,W] float32 planes with gradients to the
    leaves, sum_i alpha_i*T_i*z_i (z, or 1/z: view-space depth; background 0, not divided by alpha) and 1 - final T (DESIGN.md
    section 7).  They come from the fused path only: override_color, the pipe's Python flags, LGR_FUSED=0, non-standard activations,
    deterministic mode, blend mode 1, the view-parallel exchange and LGR_SPARSE_SINGLE=1 raise RuntimeError before any launch.  A
    resident VQ model asked for them renders from its leaves, which materialise as on any call that needs them.
    With LGR_DENSIFY_GRAD=abs (read at each call) and gradients enabled, the backward also sets `viewspace_points.absgrad` ([P,2], the
    sum over pixels of each pixel's |dL/dmean2D| term, DESIGN.md section 7) for add_densification_stats; the same paths, depth= and
    alpha= then raise RuntimeError before any launch.  Without gradients the variable changes nothing.
    camera_grad=True (with gradients enabled) makes viewpoint_camera's world_view_transform, full_proj_transform and camera_center
    tensor inputs of the fused node: those that require grad receive dL/d themselves in the backward (DESIGN.md section 7, "Camera
    gradients"; the intrinsics get none).  It needs float32 CUDA tensors of shapes [4,4], [4,4], [3] and the fused path; the unfused
    paths, LGR_DENSIFY_GRAD=abs, the view-parallel exchange and LGR_SPARSE_SINGLE=1 raise RuntimeError before any launch.  It works in
    deterministic mode (bit-identical camera gradients run to run) and with depth= / alpha=.  Without gradients it changes nothing."""
    return _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, False, depth=depth, alpha=alpha,
                   camera_grad=camera_grad)


def count_render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None):
    """render() plus per-Gaussian `gaussians_count` and `important_score` for this view (prune.py:133-157).
    With LGR_SIGNIFICANCE=blend_weight (read at each call), `important_score` is instead the Gaussian's blending weight in this view,
    the sum of alpha * T over the pixels that blend it, and the dict gains `blend_weight_fx`, the same sums as exact int64 in units
    of 2^-32 (DESIGN.md section 3).  `gaussians_count` is the same in both modes."""
    weight = significance_mode() == "blend_weight"
    return _render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, override_color, True, weight)
