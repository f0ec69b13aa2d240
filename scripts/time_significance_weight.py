"""Cost of the blending-weight significance (LGR_SIGNIFICANCE=blend_weight) against the default opacity * count, on the bench scene:
3M Gaussians, SH degree 3, 1920x1080.

  (a) count_render views/s, default and opt-in alternated view by view, CUDA events around each call;
  (b) the count blend kernel's time (stage "blend_forward_kernel<count>" of the library's event profile), in separate rounds of each mode;
  (c) parallel.sharded_prune_list over 16 cameras, each mode, alternated.

Prints the card's name, power limit and SM clock next to the numbers.  Run: python scripts/time_significance_weight.py [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightgaussian_b200 import capi, parallel  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import count_render  # noqa: E402
from lightgaussian_b200.synth import make_scene, make_cameras  # noqa: E402

MODES = ("count", "blend_weight")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_significance_weight.py measures on a CUDA device; none is present")
    scene = make_scene(a.P, sh_degree=3, seed=0)
    pc = GaussianParams(scene["raw"], 3, "cuda", requires_grad=False)
    cams = [TorchCamera(c) for c in make_cameras(16, a.width, a.height)]
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")

    def call(cam, mode):
        os.environ["LGR_SIGNIFICANCE"] = mode
        with torch.no_grad():
            return count_render(cam, pc, pipe, bg)

    for cam in cams[:4]:                      # warm-up of every shape, both modes
        for m in MODES:
            call(cam, m)
    torch.cuda.synchronize()

    # (a) views/s, alternating per view
    per = {m: [] for m in MODES}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for r in range(a.rounds):
        for i, cam in enumerate(cams):
            order = MODES if (r + i) % 2 == 0 else MODES[::-1]
            for m in order:
                ev[0].record()
                call(cam, m)
                ev[1].record()
                ev[1].synchronize()
                per[m].append(ev[0].elapsed_time(ev[1]))

    # (b) blend kernel time from the library's event profile, rounds of each mode alternated
    blend = {m: [] for m in MODES}
    capi.profile_enable(True)
    capi.profile_collect()
    for r in range(a.rounds):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):
            for cam in cams:
                call(cam, m)
            ms, n = capi.profile_collect()["blend_forward_kernel<count>"]
            blend[m].append(ms / max(n, 1))
    capi.profile_enable(False)

    # (c) sharded_prune_list over the 16 cameras
    prune = {m: [] for m in MODES}
    for r in range(max(a.rounds // 2, 3)):
        for m in (MODES if r % 2 == 0 else MODES[::-1]):
            os.environ["LGR_SIGNIFICANCE"] = m
            ev[0].record()
            with torch.no_grad():
                parallel.sharded_prune_list(pc, cams, pipe, bg, count_render)
            ev[1].record()
            ev[1].synchronize()
            prune[m].append(ev[0].elapsed_time(ev[1]))
    os.environ.pop("LGR_SIGNIFICANCE", None)

    def stats(v):
        v = np.asarray(v)
        return dict(median_ms=float(np.median(v)), p10_ms=float(np.percentile(v, 10)), p90_ms=float(np.percentile(v, 90)), n=int(v.size))
    res = dict(card=card(), P=a.P, width=a.width, height=a.height,
               count_render={m: stats(per[m]) for m in MODES}, blend_fwd_count={m: stats(blend[m]) for m in MODES},
               sharded_prune_list_16={m: stats(prune[m]) for m in MODES})
    for k in ("count_render", "blend_fwd_count", "sharded_prune_list_16"):
        c, w = res[k]["count"]["median_ms"], res[k]["blend_weight"]["median_ms"]
        res[k]["weight_over_count"] = w / c
    res["views_per_s"] = {m: 1000.0 / res["count_render"][m]["median_ms"] for m in MODES}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
