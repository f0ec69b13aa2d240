"""Deterministic GaussianModel states for tests/test_gpu_densify.py, built the same way under both stacks: leaves of synth.make_scene,
seeded Adam moments, densification statistics from a file (real render() + backward views) or seeded.  Case options: `sh_degree`
keeps (degree+1)^2 - 1 rows of _features_rest (0 rows at degree 0); `wide_scales` spreads the log-scales by a seeded per-row offset
in [-3, 3), so that clone, split and the world-space size prune all find rows on both sides of their thresholds."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.append(ROOT)

from lightgaussian_b200.synth import make_scene  # noqa: E402

ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
        "rotation": "_rotation"}
RAW = {"xyz": "xyz", "f_dc": "features_dc", "f_rest": "features_rest", "opacity": "opacity", "scaling": "scaling", "rotation": "rotation"}
STEP = 120.0


def build(case: dict) -> dict:
    P = case["P"]
    scene = make_scene(case["P_base"], sh_degree=3, seed=case["seed"], scale_mult=1.5)
    st = {name: torch.from_numpy(scene["raw"][RAW[name]][:P].copy()) for name in ATTR}
    if "sh_degree" in case:
        st["f_rest"] = st["f_rest"][:, :(case["sh_degree"] + 1) ** 2 - 1].contiguous()
    if case.get("wide_scales"):
        st["scaling"] += torch.rand((P, 1), generator=torch.Generator().manual_seed(case["seed"] + 1)) * 6 - 3
    g = torch.Generator().manual_seed(case["seed"])
    for name in ATTR:
        st["m_" + name] = torch.randn(st[name].shape, generator=g) * 1e-4
        st["v_" + name] = torch.rand(st[name].shape, generator=g) * 1e-8
    if case.get("stats"):
        d = torch.load(case["stats"])
        st["accum"], st["denom"] = d["accum"][:P].clone(), d["denom"][:P].clone()
    else:
        st["denom"] = torch.randint(0, 6, (P, 1), generator=g).float()
        st["accum"] = torch.rand((P, 1), generator=g) * st["denom"] * 4e-4
    st["max_radii2D"] = torch.randint(0, 40, (P,), generator=g).float()
    k = case.get("zero_denom_every", 0)
    if k:
        st["accum"][::k] = 0
        st["denom"][::k] = 0
    return st
