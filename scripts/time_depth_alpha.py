"""Cost of the depth and alpha planes (render(depth="z", alpha=True)) against colour only, on the bench scene: 3M Gaussians, SH degree 3,
1920x1080, 16 cameras.

  (a) forward: render() under no_grad, colour only and colour + depth + alpha alternated view by view, CUDA events around each call;
  (b) forward + backward: render() and the backward of an L1 loss on every plane the call returns, alternated the same way;
  (c) the blend forward and backward kernels (stages of the library's event profile), rounds of each variant alternated.

Prints the card's name, power limit and SM clock next to the numbers.  Run: python scripts/time_depth_alpha.py [--out FILE.json]"""
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

VARIANTS = ("color", "color+depth+alpha")


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
        sys.exit("time_depth_alpha.py measures on a CUDA device; none is present")
    scene = make_scene(a.P, sh_degree=3, seed=0)
    pc = GaussianParams(scene["raw"], 3, "cuda")
    del scene
    cams = [TorchCamera(c) for c in make_cameras(16, a.width, a.height)]
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    g = torch.Generator().manual_seed(1234)
    target = torch.rand(3, a.height, a.width, generator=g).cuda()
    tplane = torch.rand(1, a.height, a.width, generator=g).cuda()

    def forward(cam, v):
        if v == "color":
            return render(cam, pc, pipe, bg)
        return render(cam, pc, pipe, bg, depth="z", alpha=True)

    def step(cam, v):
        for p in pc.parameters():
            p.grad = None
        pkg = forward(cam, v)
        loss = (pkg["render"] - target).abs().mean()
        if v != "color":
            loss = loss + (pkg["depth"] - tplane).abs().mean() + (pkg["alpha"] - tplane).abs().mean()
        loss.backward()

    def fwd_only(cam, v):
        with torch.no_grad():
            forward(cam, v)

    for cam in cams[:4]:                      # warm-up of every shape, both variants
        for v in VARIANTS:
            fwd_only(cam, v)
            step(cam, v)
    torch.cuda.synchronize()

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def alternate(fn):
        per = {v: [] for v in VARIANTS}
        for r in range(a.rounds):
            for i, cam in enumerate(cams):
                for v in (VARIANTS if (r + i) % 2 == 0 else VARIANTS[::-1]):
                    ev[0].record()
                    fn(cam, v)
                    ev[1].record()
                    ev[1].synchronize()
                    per[v].append(ev[0].elapsed_time(ev[1]))
        return per

    fwd = alternate(fwd_only)
    fb = alternate(step)

    kernels = {v: {"blend_forward_kernel": [], "blend_backward_kernel": [], "preprocess_backward_kernel": []} for v in VARIANTS}
    capi.profile_enable(True)
    capi.profile_collect()
    for r in range(a.rounds):
        for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):
            for cam in cams:
                step(cam, v)
            prof = capi.profile_collect()
            for k in kernels[v]:
                ms, n = prof.get(k, (0.0, 0))
                kernels[v][k].append(ms / len(cams))
    capi.profile_enable(False)

    def stats(x):
        x = np.asarray(x)
        return dict(median_ms=float(np.median(x)), p10_ms=float(np.percentile(x, 10)), p90_ms=float(np.percentile(x, 90)), n=int(x.size))
    res = dict(card=card(), P=a.P, width=a.width, height=a.height, cameras=len(cams),
               forward={v: stats(fwd[v]) for v in VARIANTS}, forward_backward={v: stats(fb[v]) for v in VARIANTS},
               kernels_per_view={v: {k: stats(x) for k, x in kernels[v].items()} for v in VARIANTS})
    for k in ("forward", "forward_backward"):
        res[k]["planes_over_color"] = res[k][VARIANTS[1]]["median_ms"] / res[k][VARIANTS[0]]["median_ms"]
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
