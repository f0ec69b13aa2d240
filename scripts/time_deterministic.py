"""What deterministic mode costs: bench.py's scene (3M Gaussians, SH degree 3, 1920x1080, camera 0 of 16, black background), timed
in default and deterministic mode in alternating rounds with CUDA events, warm-up first:
  * forward   : render() of the fused path;
  * backward  : the backward of that render against a fixed upstream gradient (retain_graph, the same forward every time);
  * iteration : render, 0.8 L1 + 0.2 DSSIM (lgr_image_loss), backward, FusedAdamW step;
  * VecTree   : one weighted EMA k-means iteration at 80 000 samples x 8192 codes x 27 dims (VectorQuantize in training mode), on
                random samples, and in the worst case for the per-code sums: every sample in one tight cluster far from the initial
                codebook, so all 80 000 samples fall on one code and one warp adds them all.
Prints the card name and its power limit with the numbers, and the memory the deterministic binning blob holds (from shapes).

    python scripts/time_deterministic.py [--rounds 10] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lightgaussian_b200 import capi, loss as fused_loss, optim as fused_optim  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params  # noqa: E402
from lightgaussian_b200.renderer import render  # noqa: E402
from lightgaussian_b200.synth import make_scene, make_cameras  # noqa: E402
from lightgaussian_b200.vectree import VectorQuantize  # noqa: E402

P, W, H = 3_000_000, 1920, 1080


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def set_mode(on):
    os.environ["LGR_DETERMINISTIC"] = "1" if on else "0"


def timed(fn, reps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    dev = "cuda"
    scene = make_scene(P, sh_degree=3, seed=0)
    pc = GaussianParams(scene["raw"], 3, dev)
    del scene
    cam = TorchCamera(make_cameras(16, W, H)[0], dev)
    bg = torch.zeros(3, device=dev)
    pipe = pipeline_params()
    target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(1234)).to(dev)
    dpix = torch.randn(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev) * 1e-7
    names = ["_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"]
    lrs = [1.6e-4, 2.5e-3, 2.5e-3 / 20, 0.05, 0.005, 0.001]
    opt = fused_optim.FusedAdamW([{"params": [getattr(pc, n)], "lr": lr, "name": n} for n, lr in zip(names, lrs)], lr=0.0, eps=1e-15)

    def fwd():
        with torch.no_grad():
            render(cam, pc, pipe, bg)

    held = {}

    def prepare_bwd():
        held["pkg"] = render(cam, pc, pipe, bg)

    def bwd():
        held["pkg"]["render"].backward(dpix, retain_graph=True)

    def iteration():
        pkg = render(cam, pc, pipe, bg)
        loss = fused_loss.l1_ssim_loss(pkg["render"], target, 0.2)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    g = torch.Generator(device=dev).manual_seed(0)
    feats = torch.randn(320_000, 27, device=dev, generator=g)
    imp = torch.rand(320_000, device=dev, generator=g) + 0.01
    torch.manual_seed(0)
    vq = VectorQuantize(dim=27, codebook_size=8192, decay=0.8, commitment_weight=0.0).to(dev)
    vq.train()
    sel = torch.randint(0, 320_000, (80_000,), device=dev, generator=g)
    x, w = feats[sel].unsqueeze(0), imp[sel].reshape(1, -1, 1)

    xc = 5.0 + 0.05 * torch.randn(80_000, 27, device=dev, generator=g)
    torch.manual_seed(0)
    vqc = VectorQuantize(dim=27, codebook_size=8192, decay=0.8, commitment_weight=0.0).to(dev)
    vqc.train()
    state = (vqc._codebook.embed.clone(), vqc._codebook.cluster_size.clone())

    def vq_iter():
        vq(x, weight=w)

    def vq_clustered():
        vqc._codebook.embed.copy_(state[0])
        vqc._codebook.cluster_size.copy_(state[1])
        vqc(xc.unsqueeze(0), weight=w)

    arms = {"forward": (None, fwd), "backward": (prepare_bwd, bwd), "iteration": (None, iteration), "vectree": (None, vq_iter),
            "vectree_one_code": (None, vq_clustered)}
    times = {(k, m): [] for k in arms for m in (False, True)}
    for on in (False, True):       # warm-up of every shape in both modes
        set_mode(on)
        for k, (prep, fn) in arms.items():
            if prep:
                prep()
            fn()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            set_mode(on)
            for k, (prep, fn) in arms.items():
                if prep:
                    prep()
                times[(k, on)].append(timed(fn, args.reps))
    set_mode(False)
    capi.set_deterministic(False)

    # memory held between forward and backward: the binning blob of one forward in each mode (partial rows + bitmap in deterministic mode)
    from lightgaussian_b200.rasterizer import _forward_raw_native, GaussianRasterizationSettings
    import math
    rs = GaussianRasterizationSettings(H, W, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), bg, 1.0, cam.world_view_transform,
                                       cam.full_proj_transform, 3, cam.camera_center, False, False, False)
    blob = {}
    for on in (False, True):
        set_mode(on)
        with torch.no_grad():
            r = _forward_raw_native(False, rs, *[p.detach() for p in pc.parameters()])
        blob[on] = (int(r[6].numel()), int(r[5][:4].view(torch.int32)[0].item()))
    set_mode(False)
    capi.set_deterministic(False)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out = {"card": card(), "P": P, "image": f"{W}x{H}", "rounds": args.rounds, "reps": args.reps, "ms_median": {}}
    for k in arms:
        d, t = med[(k, False)], med[(k, True)]
        spread = (max(times[(k, False)]) - min(times[(k, False)])) / d
        out["ms_median"][k] = {"default": round(d, 4), "deterministic": round(t, 4), "ratio": round(t / d, 3),
                               "default_spread": round(spread, 3)}
    from lightgaussian_b200.vectree import vq_assign
    idx = vq_assign(xc, state[0][0])
    out["vectree_one_code_largest_cluster"] = int(torch.bincount(idx.long(), minlength=8192).max())
    out["binning_blob_bytes"] = {"default": blob[False][0], "deterministic": blob[True][0], "instances_listed": blob[True][1]}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
