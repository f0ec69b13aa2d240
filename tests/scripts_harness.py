"""Harness for running the reference's scripts UNMODIFIED on a GPU (tests/test_gpu_scripts.py).

Two import stacks over the same verbatim copy of the reference's Python tree (oracle/_ref/stock/LightGaussian, staged by
oracle/stage_reference.py when build() finds the reference checkout):

  ours   PYTHONPATH = <repo>/dropin : <repo> : oracle/_ref/stock/LightGaussian          -> our rasterizer / loss / optimizer
  stock  PYTHONPATH = oracle/_ref/stock : oracle/_ref/stock/shims : oracle/_ref/stock/LightGaussian
                                                                                     -> the reference's own pybind extension (built
                                                                                        from RAST/setup.py), gaussian_renderer, loss, AdamW

The synthetic scene (SURVEY.md section 8d): seeded random Gaussians, cameras on a Fibonacci sphere, ground-truth images rendered
from the scene itself, written as a COLMAP-layout dataset; checkpoints in the reference's `capture()` layout made by the
reference's own GaussianModel (tests/helpers/make_checkpoint.py).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "oracle", "_ref", "stock")
TREE = os.path.join(REFDIR, "LightGaussian")
HELPERS = os.path.join(ROOT, "tests", "helpers")


def stacks_available() -> str | None:
    """None when both stacks can run, else the reason."""
    if not os.path.isfile(os.path.join(TREE, "prune_finetune.py")):
        return "oracle/_ref/stock/LightGaussian is not staged (oracle/stage_reference.py needs the reference checkout)"
    ext = os.path.join(REFDIR, "diff_gaussian_rasterization")
    if not (os.path.isdir(ext) and any(f.startswith("_C") and f.endswith(".so") for f in os.listdir(ext))):
        return "oracle/_ref/stock/diff_gaussian_rasterization (the reference's own extension) is not built"
    if not os.path.isdir(os.path.join(REFDIR, "shims")):
        return "oracle/_ref/stock/shims is not staged"
    return None


def stack_env(stack: str, trace: str | None = None) -> dict:
    if stack == "ours":
        path = [os.path.join(ROOT, "dropin"), ROOT, TREE]
    elif stack == "stock":
        path = [REFDIR, os.path.join(REFDIR, "shims"), TREE]
    else:
        raise ValueError(stack)
    # PYTHONSAFEPATH (python -P, >= 3.11): do NOT put the script's own directory at sys.path[0] -- otherwise `python prune_finetune.py`
    # finds the reference's gaussian_renderer/ package next to the script before PYTHONPATH is consulted, and our drop-in never loads
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(path), PYTHONSAFEPATH="1", PYTHONHASHSEED="0",
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    # torch >= 2.6 defaults torch.load to weights_only=True; the reference's checkpoints are tuples of Parameters + an optimizer
    # state_dict written by the torch of its day.  Same setting for both stacks.
    env["TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD"] = "1"
    env.pop("LGR_TRACE", None)
    if trace:
        env["LGR_TRACE"] = trace
    return env


def run(stack: str, argv: list, cwd: str | None = None, trace: str | None = None, timeout: int = 900) -> subprocess.CompletedProcess:
    """python <argv> under the stack's import path; cwd defaults to the reference tree (its scripts import top-level siblings)."""
    out = subprocess.run([sys.executable] + argv, env=stack_env(stack, trace), cwd=cwd or TREE, capture_output=True, text=True, timeout=timeout)
    if out.returncode != 0:
        raise RuntimeError(f"[{stack}] {' '.join(argv[:2])} failed ({out.returncode})\n--- stdout\n{out.stdout[-3000:]}\n--- stderr\n{out.stderr[-6000:]}")
    return out


def render_ground_truth(raw: dict, cams, device="cuda"):
    """GT images of the synthetic scene: our render() of the full scene, black background, one [3,H,W] float32 array per camera."""
    import torch
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    pc = GaussianParams(raw, 3, device, requires_grad=False)
    bg = torch.zeros(3, device=device)
    pipe = pipeline_params()
    imgs = []
    with torch.no_grad():
        for c in cams:
            imgs.append(render(TorchCamera(c, device), pc, pipe, bg)["render"].clamp(0, 1).cpu().numpy())
    return imgs


def build_workdir(base: str, P=20000, W=320, H=240, n_views=24, seed=5, scale_mult=1.5, iteration=30000) -> dict:
    """dataset + checkpoint for the script runs.  Returns the paths and the scene."""
    from lightgaussian_b200.synth import make_scene, make_cameras, write_colmap_dataset
    scene = make_scene(P, sh_degree=3, seed=seed, scale_mult=scale_mult)
    cams = make_cameras(n_views, W, H)
    gt = render_ground_truth(scene["raw"], cams)
    data = os.path.join(base, "data")
    write_colmap_dataset(data, list(zip(cams, gt)))
    raw_path = os.path.join(base, "raw.npz")
    # cameras_extent of this rig: 1.1 x the largest distance of a camera from the centroid of the cameras (getNerfppNorm)
    np.savez(raw_path, spatial_lr_scale=np.float32(3.3), **scene["raw"])
    ckpt = os.path.join(base, f"chkpnt{iteration}.pth")
    run("stock", [os.path.join(HELPERS, "make_checkpoint.py"), raw_path, ckpt, str(iteration)])
    return dict(base=base, data=data, ckpt=ckpt, raw=scene["raw"], act=scene["act"], cams=cams, gt=gt, W=W, H=H, P=P, iteration=iteration)


def read_scalars(model_dir: str, tag: str) -> dict:
    """{step: value} of a tensorboard scalar the scripts log through utils/logger_utils.py:56-59."""
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(model_dir, size_guidance={"scalars": 0})
    acc.Reload()
    return {e.step: e.value for e in acc.Scalars(tag)}


def load_checkpoint_leaves(path: str) -> dict:
    """numpy leaves of a `capture()` checkpoint (scene/gaussian_model.py:62-76)"""
    import torch
    (cap, it) = torch.load(path, weights_only=False, map_location="cpu")
    names = ["xyz", "features_dc", "features_rest", "scaling", "rotation", "opacity"]
    leaves = {n: np.ascontiguousarray(t.detach().float().numpy()) for n, t in zip(names, cap[1:7])}
    return dict(active_sh_degree=int(cap[0]), iteration=int(it), leaves=leaves)


def psnr_of_leaves(leaves: dict, sh_degree: int, cams, gt, device="cuda") -> float:
    """mean PSNR over the cameras of the model `leaves` against the GT images, rendered by OUR renderer for both stacks' results
    (utils/image_utils.py psnr: 20 log10(1/sqrt(mse)) per image)."""
    import torch
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    pc = GaussianParams(leaves, int(round((leaves["features_rest"].shape[1] + 1) ** 0.5)) - 1, device, requires_grad=False)
    pc.active_sh_degree = sh_degree
    bg = torch.zeros(3, device=device)
    vals = []
    with torch.no_grad():
        for c, g in zip(cams, gt):
            img = render(TorchCamera(c, device), pc, pipeline_params(), bg)["render"].clamp(0, 1)
            mse = ((img - torch.from_numpy(g).to(device)) ** 2).mean().item()
            vals.append(20.0 * np.log10(1.0 / np.sqrt(max(mse, 1e-12))))
    return float(np.mean(vals))


def read_trace(path: str) -> dict:
    with open(path) as f:
        return json.load(f)
