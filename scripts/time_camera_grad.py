"""Cost of the camera gradients (render(..., camera_grad=True)) against the default render, on the bench scene: 3M Gaussians, SH degree 3,
1920x1080, 16 cameras.

  (a) forward + backward to the leaves (and the camera): render() and the backward of an L1 loss, default and camera_grad alternated view
      by view, CUDA events;
  (b) K7+K8 (the per-Gaussian backward, stage "preprocess_backward_kernel" of the library's event profile) and the finish kernel
      ("camera_grad_finish_kernel"), rounds of each mode alternated.

Prints the card's name, power limit and SM clock next to the numbers.  Run: python scripts/time_camera_grad.py [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightgaussian_b200 import capi  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import render  # noqa: E402
from lightgaussian_b200.synth import make_scene, make_cameras  # noqa: E402

MODES = ("default", "camera")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_camera_grad.py measures on a CUDA device; none is present")
    scene = make_scene(a.P, sh_degree=3, seed=0)
    pc = GaussianParams(scene["raw"], 3, "cuda")
    del scene
    cams = [TorchCamera(c) for c in make_cameras(16, a.width, a.height)]
    for c in cams:   # camera tensors that want gradients, as a pose-refinement loop builds them
        for n in ("world_view_transform", "full_proj_transform", "camera_center"):
            setattr(c, n, getattr(c, n).clone().requires_grad_(True))
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    target = torch.rand(3, a.height, a.width, generator=torch.Generator().manual_seed(1234)).cuda()

    def step(cam, mode):
        for p in pc.parameters():
            p.grad = None
        pkg = render(cam, pc, pipe, bg, camera_grad=(mode == "camera"))
        (pkg["render"] - target).abs().mean().backward()

    for cam in cams[:4]:                      # warm-up of every shape, both modes
        for m in MODES:
            step(cam, m)
    torch.cuda.synchronize()

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fb = {m: [] for m in MODES}
    for r in range(a.rounds):
        for i, cam in enumerate(cams):
            for m in (MODES if (r + i) % 2 == 0 else MODES[::-1]):
                ev[0].record()
                step(cam, m)
                ev[1].record()
                ev[1].synchronize()
                fb[m].append(ev[0].elapsed_time(ev[1]))

    k8 = {m: [] for m in MODES}
    fin = []
    capi.profile_enable(True)
    capi.profile_collect()
    for r in range(a.rounds):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):
            for cam in cams:
                step(cam, m)
            prof = capi.profile_collect()
            k8[m].append(prof.get("preprocess_backward_kernel", (0.0, 0))[0] / len(cams))
            if m == "camera":
                ms, n = prof.get("camera_grad_finish_kernel", (0.0, 0))
                fin.append(ms / max(n, 1))
    capi.profile_enable(False)

    def summary(x):
        x = np.asarray(x)
        return dict(median_ms=float(np.median(x)), p10_ms=float(np.percentile(x, 10)), p90_ms=float(np.percentile(x, 90)), n=int(x.size))
    res = dict(card=card(), P=a.P, width=a.width, height=a.height, cameras=len(cams),
               forward_backward={m: summary(fb[m]) for m in MODES}, k7k8_per_view={m: summary(k8[m]) for m in MODES},
               finish_kernel=summary(fin))
    for k in ("forward_backward", "k7k8_per_view"):
        res[k]["camera_over_default"] = res[k]["camera"]["median_ms"] / res[k]["default"]["median_ms"]
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
