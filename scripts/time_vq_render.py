"""Render a VecTree-compressed model in place (lightgaussian_b200/vqresident.py) against the dense leaves GaussianModel.load_vq
builds from the same files: 3M Gaussians, SH degree 3, 1080p, make_scene data encoded by our Quantization with the reference's
parameters (8192 codes, vq_ratio 0.6, half; fewer k-means iterations than the reference's 1000, which do not change the sizes).
Prints forward and count_render views/s (CUDA events, alternating rounds), the preprocess kernel time of each path (library stage
timers, a separate pass), the bytes each load leaves allocated and its peak, and the card name and power limit.

    python scripts/time_vq_render.py [--rounds 5] [--views 20] [--out DIR]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lightgaussian_b200 import capi  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import count_render, render  # noqa: E402
from lightgaussian_b200.synth import make_cameras, make_scene  # noqa: E402
from lightgaussian_b200.vectree import Quantization  # noqa: E402
from lightgaussian_b200.vqresident import ResidentVQ  # noqa: E402

P, W, H = 3_000_000, 1920, 1080


class Resident:
    def __init__(self, store):
        self._vq_resident, self._xyz = store, store.xyz
        self.max_sh_degree = self.active_sh_degree = 3

    @property
    def get_xyz(self):
        return self._xyz


def measured_load(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base


def views_per_s(fn, model, cams, bg):
    pipe = pipeline_params()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for c in cams:
        fn(c, model, pipe, bg)
    e.record()
    e.synchronize()
    return len(cams) / (s.elapsed_time(e) / 1000.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--iters", type=int, default=20, help="k-means iterations of the encoding")
    ap.add_argument("--out", default=None, help="directory for the result JSON")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name()

    raw = make_scene(P, sh_degree=3, seed=0)["raw"]
    table = np.concatenate([raw["xyz"], np.zeros((P, 3), np.float32), raw["features_dc"].reshape(P, 3),
                            raw["features_rest"].transpose(0, 2, 1).reshape(P, -1), raw["opacity"], raw["scaling"], raw["rotation"]], axis=1)
    imp = np.random.default_rng(1).random(P)
    work = tempfile.mkdtemp(prefix="time_vq_render_")
    torch.manual_seed(0)
    Quantization(table, importance=imp, sh_degree=3, save_path=work, codebook_size=8192, iteration_num=args.iters, vq_ratio=0.6,
                 vq_way="half", device="cuda").quantize()
    del table, raw

    store, res_held, res_peak = measured_load(lambda: ResidentVQ.load(work, 3, "cuda"))
    shell = type("Shell", (), {})()
    shell.path, shell.max_sh_degree, shell.xyz = work, 3, store.xyz

    def dense_load():
        pc = GaussianParams.__new__(GaussianParams)
        for n, t in ResidentVQ.materialize(shell).items():
            setattr(pc, n, t)
        pc.max_sh_degree = pc.active_sh_degree = 3
        return pc

    dense, den_held, den_peak = measured_load(dense_load)
    resident = Resident(store)
    cams = [TorchCamera(c) for c in make_cameras(args.views, W, H)]
    bg = torch.zeros(3, device="cuda")
    rates = {k: [] for k in ("render_resident", "render_dense", "count_resident", "count_dense")}
    with torch.no_grad():
        for fn in (render, count_render):       # warm-up of every shape
            for m in (resident, dense):
                views_per_s(fn, m, cams[:3], bg)
        for _ in range(args.rounds):
            rates["render_resident"].append(views_per_s(render, resident, cams, bg))
            rates["render_dense"].append(views_per_s(render, dense, cams, bg))
            rates["count_resident"].append(views_per_s(count_render, resident, cams, bg))
            rates["count_dense"].append(views_per_s(count_render, dense, cams, bg))
        pre = {}
        for name, m in (("resident", resident), ("dense", dense)):
            capi.profile_collect()
            capi.profile_enable(True)
            views_per_s(render, m, cams, bg)
            stages = capi.profile_collect()
            capi.profile_enable(False)
            ms, n = stages["preprocess_kernel"]
            pre[name] = ms / max(n, 1)
    result = dict(card=card, P=P, W=W, H=H, views=args.views, rounds=args.rounds,
                  views_per_s={k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for k, v in rates.items()},
                  preprocess_ms=pre, resident_bytes=dict(store=store.nbytes(), held_after_load=res_held, peak_during_load=res_peak),
                  dense_bytes=dict(held_after_load=den_held, peak_during_load=den_peak))
    shutil.rmtree(work, ignore_errors=True)
    print(json.dumps(result, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_vq_render.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
