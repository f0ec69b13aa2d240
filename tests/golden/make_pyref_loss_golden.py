"""Generates tests/golden/pyref_loss.npz by IMPORTING the reference's own loss module (/root/reference/utils/loss_utils.py)
on CPU: l1_loss, ssim and the autograd gradient of the training loss (1-l)*l1 + l*(1-ssim) (prune_finetune.py:160-164).
Needs the reference checkout:  python tests/golden/make_pyref_loss_golden.py"""
import importlib.util
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("ref_loss_utils", "/root/reference/utils/loss_utils.py")
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

rng = np.random.default_rng(77)
out = {}
for name, (H, W) in {"a": (37, 53), "b": (64, 40), "c": (11, 9)}.items():
    yy, xx = np.mgrid[0:H, 0:W]
    base = 0.5 + 0.4 * np.sin(xx / 7.0)[None] * np.cos(yy / 5.0)[None] * np.array([1.0, 0.7, 0.4])[:, None, None]
    x = np.clip(base + 0.1 * rng.standard_normal((3, H, W)), 0, 1.5).astype(np.float32)
    y = np.clip(base + 0.05 * rng.standard_normal((3, H, W)), 0, 1).astype(np.float32)
    xt = torch.from_numpy(x).requires_grad_(True)
    yt = torch.from_numpy(y)
    l1, ss = ref.l1_loss(xt, yt), ref.ssim(xt, yt)
    lam = 0.2
    loss = (1.0 - lam) * l1 + lam * (1.0 - ss)
    loss.backward()
    out.update({f"{name}_x": x, f"{name}_y": y, f"{name}_l1": np.float32(l1.item()), f"{name}_ssim": np.float32(ss.item()),
                f"{name}_loss": np.float32(loss.item()), f"{name}_grad": xt.grad.numpy().copy()})
np.savez_compressed(os.path.join(HERE, "pyref_loss.npz"), **out)
print({k: (v.shape if hasattr(v, "shape") and v.shape else float(v)) for k, v in out.items() if not k.endswith(("_x", "_y", "_grad"))})
