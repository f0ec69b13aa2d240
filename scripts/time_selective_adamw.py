"""SelectiveAdamW against FusedAdamW on the bench scene: 3M Gaussians, SH degree 3, the six parameter groups of GaussianModel, CUDA
events, dense and selective timed in alternating rounds.

  (a) gradients of one real 1080p view (fused render, 0.8 L1 + 0.2 DSSIM, backward) -- and their measured active-row fraction;
  (b) synthetic gradients whose active rows are a random 0, 1, 13, 50 and 100 % of the Gaussians;
  (c) the whole iteration with each optimizer (render, loss, backward, step, zero_grad).

Bytes per step, from shapes: dense 28 B per element (read p, g, m, v; write p, m, v); selective 4 B per element for the gradient read
plus 24 B per element of the active rows.  Prints the card's name and power limit.  Run: python scripts/time_selective_adamw.py
[--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lightgaussian_b200 import loss as fused_loss  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.optim import FusedAdamW, SelectiveAdamW  # noqa: E402
from lightgaussian_b200.renderer import render  # noqa: E402
from lightgaussian_b200.synth import make_scene, make_cameras  # noqa: E402

NAMES = ["_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"]
LRS = [1.6e-4, 2.5e-3, 2.5e-3 / 20, 0.05, 0.005, 0.001]          # arguments/__init__.py OptimizationParams


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def make_opt(cls, pc):
    return cls([{"params": [getattr(pc, n)], "lr": lr, "name": n} for n, lr in zip(NAMES, LRS)], lr=0.0, eps=1e-15)


def time_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def alternate(arms, n, rounds):
    """{name: median ms per call} over `rounds` alternating rounds of `n` calls per arm"""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            out[k].append(time_ms(fn, n))
    return {k: float(np.median(v)) for k, v in out.items()}, {k: (float(min(v)), float(max(v))) for k, v in out.items()}


def active_fraction(pc):
    P = pc._xyz.shape[0]
    act = torch.zeros(P, dtype=torch.bool, device="cuda")
    for n in NAMES:
        act |= (getattr(pc, n).grad.reshape(P, -1) != 0).any(dim=1)
    return float(act.float().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=3_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--steps", type=int, default=20, help="optimizer steps per round and arm")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_selective_adamw.py needs a GPU")
    P, W, H = args.P, args.width, args.height
    res = {"card": card(), "P": P, "image": [W, H]}
    print(f"# {res['card']}")
    scene = make_scene(P, sh_degree=3, seed=0)                    # the bench scene (bench.py)
    cams = [TorchCamera(c, "cuda") for c in make_cameras(16, W, H)]
    gen = torch.Generator().manual_seed(1234)
    targets = [torch.rand(3, H, W, generator=gen).cuda() for _ in range(8)]
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    pc = GaussianParams(scene["raw"], 3, "cuda")
    n_el = sum(getattr(pc, n).numel() for n in NAMES)
    dense, sel = make_opt(FusedAdamW, pc), make_opt(SelectiveAdamW, pc)
    arms = {"dense": dense.step, "selective": sel.step}

    def row(label, frac):
        med, spread = alternate(arms, args.steps, args.rounds)
        b_dense, b_sel = 28 * n_el, 4 * n_el + 24 * n_el * frac
        r = {"case": label, "active_rows": frac, "dense_ms": med["dense"], "selective_ms": med["selective"],
             "speedup": med["dense"] / med["selective"], "dense_gbs": b_dense / med["dense"] / 1e6, "selective_gbs": b_sel / med["selective"] / 1e6,
             "spread_ms": spread}
        print(f"{label:>24s}  active {100 * frac:6.2f} %  dense {med['dense']:.3f} ms ({r['dense_gbs']:.0f} GB/s)  "
              f"selective {med['selective']:.3f} ms ({r['selective_gbs']:.0f} GB/s)  x{r['speedup']:.2f}", flush=True)
        return r

    # (a) one real view
    img = render(cams[0], pc, pipe, bg)["render"]
    fused_loss.l1_ssim_loss(img, targets[0], 0.2).backward()
    res["real_view"] = row("real 1080p view", active_fraction(pc))
    # (b) synthetic active-row densities
    res["synthetic"] = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in (0.0, 0.01, 0.13, 0.5, 1.0):
        keep = torch.rand(P, generator=g, device="cuda") < d
        for n in NAMES:
            p = getattr(pc, n)
            x = torch.randn(p.shape, generator=g, device="cuda") * 1e-3
            p.grad = x * keep.view((P,) + (1,) * (p.dim() - 1))
        res["synthetic"].append(row(f"synthetic {100 * d:g} %", active_fraction(pc)))
    # (c) whole iteration, one fresh model per optimizer (the steps above have moved pc far from the scene: its render costs differ)
    del dense, sel, arms, pc
    models = {"dense": (GaussianParams(scene["raw"], 3, "cuda"), FusedAdamW), "selective": (GaussianParams(scene["raw"], 3, "cuda"), SelectiveAdamW)}
    its = {}
    for name, (m, cls) in models.items():
        opt, state = make_opt(cls, m), {"i": 0}

        def it(m=m, opt=opt, state=state):
            i = state["i"] % len(cams)
            state["i"] += 1
            img = render(cams[i], m, pipe, bg)["render"]
            fused_loss.l1_ssim_loss(img, targets[i % len(targets)], 0.2).backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
        its[name] = it
    for fn in its.values():                                        # every camera once: states exist, allocator warm
        for _ in range(len(cams)):
            fn()
    med, spread = alternate(its, len(cams), args.rounds)
    res["iteration"] = {"dense_ms": med["dense"], "selective_ms": med["selective"], "dense_its": 1e3 / med["dense"],
                        "selective_its": 1e3 / med["selective"], "spread_ms": spread}
    print(f"{'whole iteration':>24s}  dense {med['dense']:.3f} ms ({1e3 / med['dense']:.1f} it/s)  selective {med['selective']:.3f} ms "
          f"({1e3 / med['selective']:.1f} it/s)", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
