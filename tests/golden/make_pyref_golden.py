"""Generates tests/golden/pyref_sh.npz by IMPORTING the reference's own Python SH evaluator
(/root/reference/utils/sh_utils.py:57-120, the `convert_SHs_python` path of gaussian_renderer/__init__.py:79-96)
on CPU.  Needs the reference checkout; the .npz is committed.

    python tests/golden/make_pyref_golden.py
"""
import importlib.util
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
spec = importlib.util.spec_from_file_location("ref_sh_utils", "/root/reference/utils/sh_utils.py")
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

rng = np.random.default_rng(2024)
N = 512
means = rng.uniform(-1, 1, (N, 3)).astype(np.float32)
campos = np.array([0.4, -2.5, 1.1], np.float32)
shs = np.concatenate([rng.standard_normal((N, 1, 3)), 0.3 * rng.standard_normal((N, 15, 3))], axis=1).astype(np.float32)  # [N,16,3]
out = dict(means=means, campos=campos, shs=shs)
feats = torch.from_numpy(shs)
for deg in range(4):
    shs_view = feats.transpose(1, 2).view(-1, 3, 16)               # gaussian_renderer/__init__.py:82-84
    d = torch.from_numpy(means) - torch.from_numpy(campos).repeat(N, 1)
    d = d / d.norm(dim=1, keepdim=True)
    rgb = torch.clamp_min(ref.eval_sh(deg, shs_view, d) + 0.5, 0.0)  # :89-90
    out[f"rgb_deg{deg}"] = rgb.numpy().astype(np.float32)
np.savez_compressed(os.path.join(HERE, "pyref_sh.npz"), **out)
print("wrote pyref_sh.npz", {k: v.shape for k, v in out.items()})
