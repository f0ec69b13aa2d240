"""ctypes binding of the C-ABI in include/lgrast.h.  torch is used only for device memory
(`tensor.data_ptr()`) and the current stream; no torch type crosses into liblgrast.so.

There is deliberately NO fallback: if liblgrast.so is missing or fails to load, importing the
rasterizer raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

from . import build as _build

LGR_OK = 0
ABI_VERSION = 2   # LGR_ABI_VERSION of include/lgrast.h this binding was written against


class LgrView(C.Structure):
    """struct lgr_view (include/lgrast.h)"""
    _fields_ = [
        ("image_width", C.c_int32), ("image_height", C.c_int32),
        ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float),
        ("sh_degree", C.c_int32), ("prefiltered", C.c_int32), ("debug", C.c_int32),
        ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p), ("background", C.c_void_p),
    ]


_SIX_LEAVES = [("xyz", C.c_void_p), ("features_dc", C.c_void_p), ("features_rest", C.c_void_p), ("scaling", C.c_void_p),
               ("rotation", C.c_void_p), ("opacity", C.c_void_p)]


class LgrRawParams(C.Structure):
    """struct lgr_raw_params: six leaf pointers + the row stride (floats) of features_rest (0 = dense)"""
    _fields_ = _SIX_LEAVES + [("features_rest_row_stride", C.c_int32)]


class LgrRawGrads(C.Structure):
    """struct lgr_raw_grads: the six (dense) leaf gradients + the optional compact dL/dRGB factor"""
    _fields_ = _SIX_LEAVES + [("rgb", C.c_void_p)]


class LgrVqResidentParams(C.Structure):
    """struct lgr_vq_resident_params: the resident arrays of a VecTree-compressed model"""
    _fields_ = [("xyz", C.c_void_p), ("attr", C.c_void_p), ("slot", C.c_void_p), ("codebook", C.c_void_p), ("nonvq", C.c_void_p),
                ("attr_half", C.c_int32), ("nonvq_half", C.c_int32), ("D", C.c_int32), ("Dp", C.c_int32), ("K", C.c_int32)]


class LgrAdamwTensor(C.Structure):
    """struct lgr_adamw_tensor"""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_int64), ("lr", C.c_double), ("step", C.c_double), ("row_elems", C.c_int64), ("param_row_stride", C.c_int64)]


class LgrAdamwRowTensor(C.Structure):
    """struct lgr_adamw_row_tensor"""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("width", C.c_int64),
                ("param_row_stride", C.c_int64), ("param_col_stride", C.c_int64), ("grad_row_stride", C.c_int64), ("grad_col_stride", C.c_int64),
                ("exp_avg_row_stride", C.c_int64), ("exp_avg_col_stride", C.c_int64),
                ("exp_avg_sq_row_stride", C.c_int64), ("exp_avg_sq_col_stride", C.c_int64), ("lr", C.c_double), ("step", C.c_double)]


class LgrCompactTensor(C.Structure):
    """struct lgr_compact_tensor"""
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("row_words", C.c_int32)]


class LgrDensifyTensor(C.Structure):
    """struct lgr_densify_tensor"""
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("row_words", C.c_int32), ("role", C.c_int32)]


DENSIFY_COPY, DENSIFY_XYZ, DENSIFY_SCALING, DENSIFY_MOMENT, DENSIFY_ZERO = range(5)   # LGR_DENSIFY_* roles


class LgrSparseStats(C.Structure):
    """struct lgr_sparse_stats"""
    _fields_ = [("serial", C.c_uint32)]


SPARSE_STATS_ERR_HEADER, SPARSE_STATS_ERR_FILTER, SPARSE_STATS_ERR_GRAD = 1, 2, 4   # bits of lgr_densify_stats_exchanged's error word


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)

_lib = None
_lib_lock = threading.Lock()


def lib_path() -> str:
    return _build.LIB_PATH


def load():
    """Load (building first if the sources are newer and nvcc is present) and type the library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        # rebuild when the sources are newer than the binary and nvcc is here (build_library returns early when up to date);
        # on a box without nvcc the shipped binary is used as is
        path = _build.LIB_PATH
        if not os.path.exists(path) or (_build.have_nvcc() and _build._stale()):
            path = _build.build_library()
        lib = C.CDLL(path)
        if lib.lgr_abi_version() != ABI_VERSION:
            raise RuntimeError("liblgrast.so ABI version mismatch")
        vp, i32 = C.c_void_p, C.c_int
        fwd_common = [C.POINTER(LgrView), i32, i32] + [vp] * 7 + [ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp]
        lib.lgr_forward.restype = i32
        lib.lgr_forward.argtypes = fwd_common + [vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_forward_count.restype = i32
        lib.lgr_forward_count.argtypes = fwd_common + [vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_backward.restype = i32
        lib.lgr_backward.argtypes = [C.POINTER(LgrView), i32, i32, i32] + [vp] * 20
        lib.lgr_forward_raw.restype = i32
        lib.lgr_forward_raw.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp,
                                        vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_forward_vq.restype = i32
        lib.lgr_forward_vq.argtypes = [C.POINTER(LgrView), i32, C.POINTER(LgrVqResidentParams), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp,
                                       vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        # the *_weight forwards: their sibling's arguments with int64_t* blend_weight behind important_score
        lib.lgr_forward_count_weight.restype = i32
        lib.lgr_forward_count_weight.argtypes = fwd_common + [vp, vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_forward_raw_weight.restype = i32
        lib.lgr_forward_raw_weight.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN,
                                               vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_forward_vq_weight.restype = i32
        lib.lgr_forward_vq_weight.argtypes = [C.POINTER(LgrView), i32, C.POINTER(LgrVqResidentParams), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN,
                                              vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_backward_raw.restype = i32
        lib.lgr_backward_raw.argtypes = [C.POINTER(LgrView), i32, i32, i32, C.POINTER(LgrRawParams), vp, vp, vp, vp, vp,
                                         C.POINTER(LgrRawGrads), vp, vp]
        # depth and alpha planes: lgr_forward_raw's arguments with (depth_mode, out_depth, out_alpha) behind important_score, and
        # lgr_backward_raw's with (depth_mode, dL_ddepth, dL_dalpha) behind dL_dout_color
        lib.lgr_forward_raw_depth.restype = i32
        lib.lgr_forward_raw_depth.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN,
                                              vp, vp, vp, vp, i32, vp, vp, vp, C.POINTER(C.c_int32), vp]
        lib.lgr_backward_raw_depth.restype = i32
        lib.lgr_backward_raw_depth.argtypes = [C.POINTER(LgrView), i32, i32, i32, C.POINTER(LgrRawParams), vp, vp, vp, vp, vp,
                                               i32, vp, vp, C.POINTER(LgrRawGrads), vp, vp]
        # absolute-gradient densification statistic: lgr_backward_raw's arguments with dL_dmeans2D_abs behind dL_dmeans2D
        lib.lgr_backward_raw_absgrad.restype = i32
        lib.lgr_backward_raw_absgrad.argtypes = [C.POINTER(LgrView), i32, i32, i32, C.POINTER(LgrRawParams), vp, vp, vp, vp, vp,
                                                 C.POINTER(LgrRawGrads), vp, vp, vp]
        # camera gradients: lgr_backward_raw_depth's arguments with (dL_dviewmatrix, dL_dprojmatrix, dL_dcampos, workspace,
        # workspace_bytes) behind dL_dmeans2D
        lib.lgr_camera_grad_workspace_bytes.restype = C.c_size_t
        lib.lgr_camera_grad_workspace_bytes.argtypes = [i32]
        lib.lgr_backward_raw_camera.restype = i32
        lib.lgr_backward_raw_camera.argtypes = [C.POINTER(LgrView), i32, i32, i32, C.POINTER(LgrRawParams), vp, vp, vp, vp, vp,
                                                i32, vp, vp, C.POINTER(LgrRawGrads), vp, vp, vp, vp, vp, C.c_size_t, vp]
        lib.lgr_backward_raw_begin.restype = i32
        lib.lgr_backward_raw_begin.argtypes = [C.POINTER(LgrView), i32, i32, vp, vp, vp, vp, vp, vp, vp]
        lib.lgr_backward_raw_end.restype = i32
        lib.lgr_backward_raw_end.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), vp, vp, C.POINTER(LgrRawGrads), vp, vp]
        lib.lgr_backward_raw_end_range.restype = i32
        lib.lgr_backward_raw_end_range.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), vp, vp, C.POINTER(LgrRawGrads), vp, i32, i32, vp]
        lib.lgr_peer_allreduce.restype = i32
        lib.lgr_peer_allreduce.argtypes = [C.POINTER(C.c_void_p), i32, i32, C.c_size_t, vp]
        lib.lgr_image_loss_workspace_bytes.restype = C.c_size_t
        lib.lgr_image_loss_workspace_bytes.argtypes = [i32, i32, i32]
        lib.lgr_image_loss_forward.restype = i32
        lib.lgr_image_loss_forward.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp, vp]
        lib.lgr_image_l1_forward.restype = i32
        lib.lgr_image_l1_forward.argtypes = [vp, vp, i32, i32, i32, vp, vp, vp]
        lib.lgr_image_loss_backward.restype = i32
        lib.lgr_image_loss_backward.argtypes = [vp, vp, vp, i32, i32, i32, C.c_float, C.c_float, vp, vp, vp]
        lib.lgr_adamw_step.restype = i32
        lib.lgr_adamw_step.argtypes = [i32, C.POINTER(LgrAdamwTensor), C.c_double, C.c_double, C.c_double, C.c_double, vp]
        lib.lgr_adamw_step_selective.restype = i32
        lib.lgr_adamw_step_selective.argtypes = [i32, C.POINTER(LgrAdamwRowTensor), C.c_longlong, C.c_double, C.c_double, C.c_double,
                                                 C.c_double, vp]
        lib.lgr_compact_workspace_bytes.restype = C.c_size_t
        lib.lgr_compact_workspace_bytes.argtypes = [i32]
        lib.lgr_compact_plan.restype = i32
        lib.lgr_compact_plan.argtypes = [i32, vp, vp, vp, C.c_size_t, C.POINTER(C.c_int32), vp]
        lib.lgr_compact_rows.restype = i32
        lib.lgr_compact_rows.argtypes = [i32, vp, i32, C.POINTER(LgrCompactTensor), vp]
        lib.lgr_sparse_exchange_bytes.restype = C.c_size_t
        lib.lgr_sparse_exchange_bytes.argtypes = [i32]
        lib.lgr_sparse_workspace_bytes.restype = C.c_size_t
        lib.lgr_sparse_workspace_bytes.argtypes = [i32]
        lib.lgr_backward_raw_sparse_pack.restype = i32
        lib.lgr_backward_raw_sparse_pack.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), vp, vp, vp, vp, vp, vp]
        lib.lgr_backward_raw_sparse_pack_push.restype = i32
        lib.lgr_backward_raw_sparse_pack_push.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), vp, vp, C.POINTER(C.c_void_p), i32, i32,
                                                          vp, vp, vp]
        lib.lgr_sparse_exchange_bytes_stats.restype = C.c_size_t
        lib.lgr_sparse_exchange_bytes_stats.argtypes = [i32]
        lib.lgr_backward_raw_sparse_pack_push_ex.restype = i32
        lib.lgr_backward_raw_sparse_pack_push_ex.argtypes = [C.POINTER(LgrView), i32, i32, C.POINTER(LgrRawParams), vp, vp, C.POINTER(C.c_void_p),
                                                             i32, i32, vp, vp, C.POINTER(LgrSparseStats), vp]
        lib.lgr_densify_stats_exchanged.restype = i32
        lib.lgr_densify_stats_exchanged.argtypes = [i32, i32, i32, C.POINTER(C.c_void_p), C.c_uint32, vp, i32, vp, vp, vp, vp, vp]
        lib.lgr_densify_stats_encode.restype = i32
        lib.lgr_densify_stats_encode.argtypes = [i32, vp, i32, vp, vp, vp]
        lib.lgr_densify_stats_add_views.restype = i32
        lib.lgr_densify_stats_add_views.argtypes = [i32, i32, vp, vp, vp, vp]
        lib.lgr_backward_raw_sparse_accumulate.restype = i32
        lib.lgr_backward_raw_sparse_accumulate.argtypes = [i32, i32, i32, i32, C.POINTER(C.c_void_p), vp, C.POINTER(LgrRawGrads), vp]
        lib.lgr_vq_workspace_bytes.restype = C.c_size_t
        lib.lgr_vq_workspace_bytes.argtypes = [C.c_int64]
        lib.lgr_vq_assign.restype = i32
        lib.lgr_vq_assign.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.lgr_vq_ema_update.restype = i32
        lib.lgr_vq_ema_update.argtypes = [i32, i32, C.c_double, C.c_double, vp, vp, vp, vp, vp, vp]
        lib.lgr_vq_gather.restype = i32
        lib.lgr_vq_gather.argtypes = [i32, i32, vp, vp, vp, vp]
        lib.lgr_vq_pack_indices.restype = i32
        lib.lgr_vq_pack_indices.argtypes = [C.c_int64, i32, vp, vp, vp]
        lib.lgr_vq_unpack_indices.restype = i32
        lib.lgr_vq_unpack_indices.argtypes = [C.c_int64, i32, vp, vp, vp]
        lib.lgr_multimem_allreduce.restype = i32
        lib.lgr_multimem_allreduce.argtypes = [vp, i32, i32, C.c_size_t, vp]
        lib.lgr_sh_grad_from_views.restype = i32
        lib.lgr_sh_grad_from_views.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        lib.lgr_knn_workspace_bytes.restype = C.c_size_t
        lib.lgr_knn_workspace_bytes.argtypes = [i32]
        lib.lgr_knn_mean_dist3.restype = i32
        lib.lgr_knn_mean_dist3.argtypes = [i32, vp, vp, vp, C.c_size_t, vp]
        lib.lgr_densify_stats.restype = i32
        lib.lgr_densify_stats.argtypes = [i32, vp, i32, vp, vp, vp, vp]
        lib.lgr_densify_workspace_bytes.restype = C.c_size_t
        lib.lgr_densify_workspace_bytes.argtypes = [i32]
        lib.lgr_densify_plan.restype = i32
        lib.lgr_densify_plan.argtypes = [i32, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, i32, i32, vp, C.c_size_t,
                                         C.POINTER(C.c_int32), vp]
        lib.lgr_densify_split_inputs.restype = i32
        lib.lgr_densify_split_inputs.argtypes = [i32, vp, C.POINTER(C.c_int32), vp, vp, vp, vp, vp, vp]
        lib.lgr_densify_rows.restype = i32
        lib.lgr_densify_rows.argtypes = [i32, vp, C.POINTER(C.c_int32), vp, vp, i32, C.POINTER(LgrDensifyTensor), vp]
        lib.lgr_mark_visible.restype = i32
        lib.lgr_mark_visible.argtypes = [i32, vp, vp, vp, vp, vp]
        lib.lgr_last_error.restype = C.c_char_p
        lib.lgr_launch_count.restype = C.c_uint64
        lib.lgr_binning_overflows.restype = C.c_uint64
        lib.lgr_forward_stream_syncs.restype = C.c_uint64
        lib.lgr_set_binning_estimate.restype = None
        lib.lgr_set_binning_estimate.argtypes = [C.c_uint64]
        for name in ("lgr_geometry_layout", "lgr_image_layout", "lgr_binning_layout"):
            getattr(lib, name).restype = C.c_size_t
        lib.lgr_geometry_layout.argtypes = [i32, C.POINTER(C.c_size_t), i32]
        lib.lgr_image_layout.argtypes = [i32, i32, C.POINTER(C.c_size_t), i32]
        lib.lgr_binning_layout.argtypes = [i32, i32, i32, C.POINTER(C.c_size_t), i32]
        lib.lgr_profile_stage_name.restype = C.c_char_p
        lib.lgr_profile_collect.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_uint64), i32]
        _lib = lib
    return _lib


class LgrError(RuntimeError):
    pass


def check(status: int, what: str):
    if status != LGR_OK:
        msg = load().lgr_last_error()
        raise LgrError(f"{what} failed (status {status}): {msg.decode() if msg else ''}")


# ---- allocator callback -------------------------------------------------------------------------
# One C callback for all calls; `user` is a small integer naming a slot that receives the tensor.
_slots = {}
_slot_lock = threading.Lock()
_next_slot = [1]


class BlobSlot:
    """Receives one opaque state blob (a uint8 torch tensor) from the library's allocator callback."""

    def __init__(self, device):
        self.device = device
        self.tensor = None
        with _slot_lock:
            self.key = _next_slot[0]
            _next_slot[0] += 1
            _slots[self.key] = self

    def release(self):
        with _slot_lock:
            _slots.pop(self.key, None)


def _alloc(user, nbytes):
    slot = _slots.get(user)
    if slot is None:
        return None
    try:
        t = torch.empty(int(nbytes), dtype=torch.uint8, device=slot.device)
    except Exception:  # out of memory -> NULL -> LGR_ERR_ALLOC
        return None
    slot.tensor = t
    return t.data_ptr()


ALLOC_CB = ALLOC_FN(_alloc)


def ptr(t):
    """Device pointer of a tensor, or NULL for None / empty tensors (the reference's 'input absent')."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def current_stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def launch_count() -> int:
    return int(load().lgr_launch_count())


def geometry_layout(P: int):
    out = (C.c_size_t * 8)()
    total = load().lgr_geometry_layout(P, out, 8)
    names = ["depth", "means2D", "conic_opacity", "rgb", "cov3D", "clamped", "tiles_touched", "sorted_ids"]
    return dict(zip(names, list(out))), int(total)


def image_layout(W: int, H: int):
    out = (C.c_size_t * 3)()
    total = load().lgr_image_layout(W, H, out, 3)
    return dict(zip(["final_T", "n_contrib", "ranges"], list(out))), int(total)


def binning_layout(R: int, W: int, H: int):
    out = (C.c_size_t * 1)()
    total = load().lgr_binning_layout(R, W, H, out, 1)
    return dict(point_list=int(out[0])), int(total)


_blend_mode = [0]


def set_blend_mode(mode: int) -> None:
    """0 = ring kernels (default), 1 = round-1 kernels (A/B measurements)"""
    check(load().lgr_set_blend_mode(int(mode)), "lgr_set_blend_mode")
    _blend_mode[0] = int(mode)


def blend_mode() -> int:
    """the blend kernels set_blend_mode selected last in this process (0 until it is called)"""
    return _blend_mode[0]


DEFAULT_BINNING_MODE = 2


def set_binning_mode(mode: int) -> None:
    """2 = library radix sorts + scan (default, fastest measured), 0 = hand-written binning kernels (no library); both size the
    binning blob from an estimate (no GPU idle on the host), 1 = hand-written kernels with an exact size (one stream sync)"""
    check(load().lgr_set_binning_mode(int(mode)), "lgr_set_binning_mode")


def binning_overflows() -> int:
    """views whose binning blob estimate was too small (binning + blend repeated) since load"""
    return int(load().lgr_binning_overflows())


def forward_stream_syncs() -> int:
    """forwards that synchronised the stream to size the binning blob exactly since load (deterministic mode, binning mode 1,
    LGR_BINNING_SYNC=1); the default forward takes none"""
    return int(load().lgr_forward_stream_syncs())


def set_vq_mode(mode: int) -> None:
    """VecTree nearest-code search: 0 = tensor-core coarse pass + exact FP32 rescore (default), 1 = FP32 kernel only"""
    check(load().lgr_set_vq_mode(int(mode)), "lgr_set_vq_mode")


def deterministic_requested() -> bool:
    """The rule every op of this package applies at call time: deterministic mode is on when torch's
    `torch.use_deterministic_algorithms(True)` is in effect or the environment sets LGR_DETERMINISTIC=1."""
    return bool(torch.are_deterministic_algorithms_enabled()) or os.environ.get("LGR_DETERMINISTIC", "0") == "1"


def set_deterministic(on: bool) -> None:
    """lgr_set_deterministic: fixed-order reductions in place of the float atomics (process-wide)"""
    check(load().lgr_set_deterministic(int(bool(on))), "lgr_set_deterministic")


def set_kback_mode(mode: int) -> None:
    """fused K7+K8 of the raw backward: 0 = zero-fill + compacted list (default), 1 = dense kernel (A/B measurements)"""
    check(load().lgr_set_kback_mode(int(mode)), "lgr_set_kback_mode")


def set_binning_estimate(instances: int) -> None:
    """overwrite the running instance estimate of binning modes 0 and 2 (tests; 0 = forget it)"""
    load().lgr_set_binning_estimate(C.c_uint64(int(instances)))


def set_tile_culling(on: bool):
    """exact tile-level culling at binning time (default on); off = per-tile lists identical to the reference's"""
    check(load().lgr_set_tile_culling(int(on)), "lgr_set_tile_culling")


def profile_enable(on: bool):
    load().lgr_profile_enable(int(on))


def profile_collect():
    """{stage name: (total ms, launches)} since the last collect; synchronises the device."""
    lib = load()
    n = lib.lgr_profile_stage_count()
    ms = (C.c_double * n)()
    cnt = (C.c_uint64 * n)()
    check(lib.lgr_profile_collect(ms, cnt, n), "lgr_profile_collect")
    return {lib.lgr_profile_stage_name(k).decode(): (float(ms[k]), int(cnt[k])) for k in range(n)}
