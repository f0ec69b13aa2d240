"""View-parallel execution of the hot path: one process per GPU (torchrun), cameras partitioned across ranks,
Gaussians replicated.  The path has exactly one exchange step per use (SURVEY.md section 8e):

  training      all-reduce(sum) of the per-Gaussian gradients after each rank's backward  -> allreduce_grads()
  significance  all-reduce(sum) of the exact int64 per-Gaussian counts over all views    -> sharded_prune_list()

The reference has no multi-GPU path at all (utils/general_utils.py:151 pins cuda:0); semantics here are
"world_size views per optimizer step, gradients summed" for training, and bit-identical results for any
partition for the significance pass (integer sums commute).
"""
from __future__ import annotations

import os
from typing import List, Sequence

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None):
    """Returns (rank, world, local_rank).  Single-process when WORLD_SIZE is unset."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_views(n_views: int, rank: int, world: int) -> List[int]:
    """camera indices {i : i mod world == rank} (SURVEY.md section 8e)."""
    return list(range(rank, n_views, world))


def balanced_view_schedule(costs: Sequence[float], world: int) -> List[List[int]]:
    """Steps of `world` views each with SIMILAR cost inside a step.  A view-parallel step lasts as long as its slowest rank, so the views
    of one step should cost the same: views are ordered by cost (e.g. the instance count `num_rendered` of the previous epoch) and cut
    into consecutive groups of `world`; group g is step g, its k-th view goes to rank (k + g) mod world so that no rank always gets the
    heavier end of its groups.  Every view appears exactly once; a last incomplete group is padded by repeating its own views.
    Deterministic in `costs`, so all ranks compute the same schedule without talking to each other.  Returns schedule[step][rank]."""
    order = sorted(range(len(costs)), key=lambda i: (-float(costs[i]), i))
    steps = []
    for g in range(0, len(order), world):
        grp = order[g:g + world]
        while len(grp) < world:
            grp = grp + grp[:world - len(grp)]
        r = (g // world) % world
        steps.append([grp[(k - r) % world] for k in range(world)])
    return steps


class FlatGrads:
    """One contiguous fp32 buffer holding every parameter's gradient, with `.grad` of each parameter a view into
    it, so the per-step exchange is a single NCCL all-reduce over NVLink instead of one per tensor."""

    def __init__(self, params: Sequence[torch.Tensor]):
        self.params = list(params)
        n = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.params[0].device)
        off = 0
        for p in self.params:
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()

    def zero(self):
        self.flat.zero_()

    def allreduce(self, world: int, average: bool = False):
        if world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            if average:
                self.flat.div_(world)

    @property
    def nbytes(self) -> int:
        return self.flat.numel() * 4


def enable_gradient_exchange(world: int, group=None, *, densification: bool = False):
    """Training on `world` ranks: after this call the backward of render()'s fused node returns gradients already summed
    over all ranks' views.  The four small leaves (44 B/Gaussian) go through ONE all-reduce; the SH gradient, which is
    rank-1 per Gaussian and view, is exchanged as its 12 B/Gaussian factor (all-gather) and rebuilt locally
    (lgr_sh_grad_from_views) -- about 4x less NVLink traffic than all-reducing the dense 12*M B/Gaussian tensor.
    densification=True: add_densification_stats (the native one, densify.install) adds every rank's view of the step in rank order,
    so the statistics, and with them every densify_and_prune decision and the model size, stay identical on every rank."""
    from . import rasterizer
    rasterizer.enable_gradient_exchange(world, group, densification=densification)


def allreduce_counts(count: torch.Tensor, world: int) -> torch.Tensor:
    """exact, order-independent sum of per-Gaussian hit counts (int64)."""
    c = count.to(torch.int64)
    if world > 1:
        dist.all_reduce(c, op=dist.ReduceOp.SUM)
    return c


# the int64 sum of the fixed-point blending weights cannot overflow below this many pixel-views: each pixel adds at most 0.99 * 2^32
WEIGHT_PIXEL_VIEWS_MAX = 2 ** 31


def check_weight_bound(cameras) -> int:
    """Pixel-views of `cameras` (sum of W * H); raises before anything runs when their blending weights could overflow int64."""
    n = sum(int(c.image_width) * int(c.image_height) for c in cameras)
    if n >= WEIGHT_PIXEL_VIEWS_MAX:
        raise RuntimeError(f"blend_weight significance: {n} pixel-views over {len(cameras)} cameras; the exact int64 sum is only "
                           f"guaranteed below 2^31 pixel-views (about 1000 views at 1080p)")
    return n


def sharded_prune_list(gaussians, cameras, pipe, background, count_render_fn, rank: int = 0, world: int = 1):
    """prune.prune_list (reference prune.py:133-157) with the camera loop partitioned over ranks.
    Returns (gaussian_list int64[P], imp_list float32[P]) identical on every rank and for every world size:
    counts are summed as integers, and the score is opacity * total count (opacity does not change inside
    the loop -- there is no optimizer step in prune_list).
    With LGR_SIGNIFICANCE=blend_weight, imp_list is the total blending weight instead: each view's int64 `blend_weight_fx` is
    summed as integers, all-reduced once next to the counts, and converted to float32 once, so it is as partition-independent."""
    from .renderer import significance_mode, weight_score
    weight = significance_mode() == "blend_weight"
    if weight:
        check_weight_bound(cameras)
    total = wtotal = None
    for i in shard_views(len(cameras), rank, world):
        pkg = count_render_fn(cameras[i], gaussians, pipe, background)
        c = pkg["gaussians_count"].to(torch.int64)
        total = c if total is None else total + c
        if weight:
            w = pkg["blend_weight_fx"].to(torch.int64)
            wtotal = w if wtotal is None else wtotal + w
    if total is None:
        total = torch.zeros(gaussians.get_xyz.shape[0], dtype=torch.int64, device=gaussians.get_xyz.device)
    if weight:
        if wtotal is None:
            wtotal = torch.zeros_like(total)
        both = allreduce_counts(torch.stack([total, wtotal]), world)
        return both[0], weight_score(both[1])
    total = allreduce_counts(total, world)
    imp = gaussians.get_opacity.detach().reshape(-1) * total.to(torch.float32)
    return total, imp
