"""Where the host and the GPU wait on each other in one training view of the bench workload: 3M Gaussians, SH degree 3, 1920x1080,
16 cameras, train_view with the fused L1 (what bench.py times).

  (1) step time: CUDA events around windows of --steps views, median over --windows windows;
  (2) host enqueue time per step: a host clock around the same windows, stopped before the closing synchronise;
  (3) per-stage native kernel times (the library's event profile) of the binning stages, in a window of their own;
  (4) in a separate run under torch.profiler (CUDA activities; trace written to --out-dir): the GPU's idle time between device
      activities per step, split into (a) the gaps between the depth-order scan's last kernel and the next emit_kernel -- the
      forward's wait for the instance count, when there is one -- and (b) all other gaps.

Prints the card's name, power limit and SM clock next to the numbers.
Run: python scripts/time_forward_wait.py [--out-dir DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightgaussian_b200 import capi  # noqa: E402
from lightgaussian_b200.loss import l1_loss  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import render  # noqa: E402
from lightgaussian_b200.synth import make_scene, make_cameras  # noqa: E402
from lightgaussian_b200.trainstep import train_view  # noqa: E402

BIN_STAGES = ("depth_sort(cub)", "scan(cub)", "emit_kernel", "tile_sort(cub)", "ranges_kernel", "blend_forward_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def idle_gaps(events, steps):
    """GPU idle time per step from the profiler's device activities: the union of all kernel / memcpy / memset intervals, its gaps
    split into those between a scan kernel's end and the next emit_kernel's start, and the rest"""
    acts = sorted((e.time_range.start, e.time_range.end, e.name) for e in events
                  if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start)
    wait_us = other_us = pending = 0.0
    n_wait = 0
    busy_end, after_scan = None, False
    for start, end, name in acts:
        gap = start - busy_end if busy_end is not None and start > busy_end else 0.0
        if after_scan:
            pending += gap               # every gap from the scan's end to the next emit is part of the wait
        else:
            other_us += gap
        if after_scan and "emit_kernel" in name:
            wait_us += pending
            n_wait += 1
            after_scan = False
        elif "DeviceScanKernel" in name:
            other_us += pending
            after_scan, pending = True, 0.0
        busy_end = end if busy_end is None else max(busy_end, end)
    if after_scan:
        other_us += pending
    return dict(wait_gap_ms_per_step=wait_us / 1e3 / steps, other_gaps_ms_per_step=other_us / 1e3 / steps,
                waits_seen=n_wait, steps=steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--steps", type=int, default=32, help="views per timed window")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--out-dir", default="bench_out/forward_wait")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_forward_wait.py measures on a CUDA device; none is present")
    dev = torch.device("cuda", 0)
    scene = make_scene(a.P, sh_degree=3, seed=0)
    pc = GaussianParams(scene["raw"], 3, dev)
    params = pc.parameters()
    cams = [TorchCamera(c, dev) for c in make_cameras(a.cams, a.width, a.height)]
    gen = torch.Generator().manual_seed(1234)
    targets = [torch.rand(3, a.height, a.width, generator=gen).to(dev) for _ in range(min(a.cams, 8))]
    pipe, bg = pipeline_params(), torch.zeros(3, device=dev)
    capi.load()

    def step(s):
        for p in params:
            p.grad = None
        i = s % len(cams)
        train_view(render, cams[i], pc, pipe, bg, targets[i % len(targets)], l1_loss)

    for s in range(2 * a.cams):                                   # warm-up of every camera
        step(s)
    torch.cuda.synchronize()
    overflows0 = capi.binning_overflows()

    # (1) + (2)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gpu_ms, host_ms = [], []
    for w in range(a.windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        for s in range(a.steps):
            step(w * a.steps + s)
        e1.record()
        t1 = time.perf_counter()
        e1.synchronize()
        gpu_ms.append(e0.elapsed_time(e1) / a.steps)
        host_ms.append((t1 - t0) * 1e3 / a.steps)
    overflows = capi.binning_overflows() - overflows0

    # (3) the binning stages' device times
    capi.profile_collect()
    capi.profile_enable(True)
    for s in range(a.cams):
        step(s)
    prof_rows = capi.profile_collect()
    capi.profile_enable(False)
    stages = {k: ms / n for k, (ms, n) in prof_rows.items() if n > 0 and k in BIN_STAGES}
    native_ms = sum(ms for ms, n in prof_rows.values() if n > 0) / a.cams

    # (4) idle gaps from a trace of its own
    os.makedirs(a.out_dir, exist_ok=True)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        for s in range(a.cams):
            step(s)
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(a.out_dir, "train_view.pt.trace.json"))
    gaps = idle_gaps(prof.events(), a.cams)

    res = dict(card=card(), P=a.P, width=a.width, height=a.height, cams=a.cams,
               step_ms=dict(median=float(np.median(gpu_ms)), min=float(np.min(gpu_ms)), max=float(np.max(gpu_ms)), windows=gpu_ms),
               host_enqueue_ms_per_step=dict(median=float(np.median(host_ms)), windows=host_ms),
               views_per_s=1000.0 / float(np.median(gpu_ms)), repeats_for_capacity_in_timed_windows=overflows,
               stage_ms_per_view=stages, native_ms_per_view=native_ms, idle=gaps)
    print(json.dumps(res, indent=1))
    with open(os.path.join(a.out_dir, "time_forward_wait.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
