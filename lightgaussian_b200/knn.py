"""distCUDA2 of submodules/simple-knn (spatial.cu:15-26): the mean squared distance of every point to its three nearest other points,
which GaussianModel.create_from_pcd turns into the initial scales (scene/gaussian_model.py:152-156).  Computed by lgr_knn_mean_dist3
(csrc/lgr_knn.cuh), bit-identical to the reference's extension, on the current stream without a host synchronisation."""
from __future__ import annotations

import torch

from . import capi


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """points: CUDA float32 [P, 3] -> CUDA float32 [P].  With fewer than three other points the missing neighbours count as
    FLT_MAX, as in the reference (+inf for P = 1 and 2, FLT_MAX / 3 for P = 3)."""
    if not isinstance(points, torch.Tensor) or points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("distCUDA2: points must be a tensor of shape (P, 3)")
    if points.dtype != torch.float32:
        raise RuntimeError(f"distCUDA2: points must be float32, got {points.dtype}")
    if not points.is_cuda:
        raise RuntimeError("distCUDA2: points must be a CUDA tensor: there is no CPU path")
    P = points.shape[0]
    if P >= 2 ** 31 - 32:
        raise RuntimeError("distCUDA2: too many points")
    out = torch.empty((P,), dtype=torch.float32, device=points.device)
    if P == 0:
        return out
    pts = points.contiguous()   # spatial.cu:23
    lib = capi.load()
    with torch.cuda.device(points.device):
        ws = torch.empty((int(lib.lgr_knn_workspace_bytes(P)),), dtype=torch.uint8, device=points.device)
        capi.check(lib.lgr_knn_mean_dist3(P, pts.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                          capi.current_stream_ptr(points.device)), "lgr_knn_mean_dist3")
    return out
