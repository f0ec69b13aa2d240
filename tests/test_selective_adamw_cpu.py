"""SelectiveAdamW without a GPU: the kernel's resources in the built library (no spills, TMA bulk copies for the gradient slices),
the [rows, width] description of each layout, the checks that refuse a step before anything changes, and the opt-in switches."""
import os
import re
import subprocess
import sys

import pytest
import torch

from lightgaussian_b200 import build, optim
from tests.test_deterministic_sass import CUOBJDUMP, _find, sass  # noqa: F401  (module fixture: the library's SASS by kernel name)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_kernel_has_no_spills_and_stages_gradients_with_bulk_copies(sass):  # noqa: F811
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", build.build_library()], check=True, capture_output=True, text=True).stdout
    usage = re.findall(r"Function (\S*adamw_selective_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert usage, "adamw_selective_kernel not in the library"
    for name, reg, stack, local in usage:
        assert int(stack) == 0 and int(local) == 0, (name, stack, local)
        assert int(reg) <= 64, (name, reg)          # four 256-thread blocks per SM
    for name in _find(sass, "adamw_selective_kernel"):
        assert "UBLKCP" in sass[name]


def test_row_view_of_each_layout():
    P = 7
    assert optim._row_view(torch.zeros(P, 15, 3)) == (45, 1)
    assert optim._row_view(torch.zeros(P, 1)) == (1, 1)
    xyz = torch.zeros(3, P).t()                                      # create_from_pcd
    assert optim._row_view(xyz) == (1, P)
    assert optim._row_view(torch.zeros(P, 15, 3)[:, :8, :]) == (45, 1)
    assert optim._row_view(torch.zeros(P, 8, 3), like=torch.zeros(P, 15, 3)[:, :8, :]) == (24, 1)
    assert optim._row_view(torch.zeros(P, 4, 6)[:, :, ::2]) == (24, 2)    # one column stride of 2
    with pytest.raises(RuntimeError, match="rows, width"):
        optim._row_view(torch.zeros(P, 4, 6)[:, :, :3])                  # columns 0-2 of each 6: no single stride


def test_refused_steps_change_nothing():
    a = torch.nn.Parameter(torch.zeros(10, 3))
    b = torch.nn.Parameter(torch.zeros(11, 1))
    opt = optim.SelectiveAdamW([{"params": [a], "lr": 0.1}, {"params": [b], "lr": 0.1}], lr=0.0, eps=1e-15)
    opt.step()                                                       # no gradients: nothing to do, no library needed
    a.grad, b.grad = torch.ones_like(a), torch.ones_like(b)
    with pytest.raises(RuntimeError, match="number of rows"):
        opt.step()
    assert len(opt.state) == 0
    b.grad = None
    with pytest.raises(RuntimeError, match="CUDA"):                  # no CPU path
        opt.step()
    c = torch.nn.Parameter(torch.zeros(10, 4))
    opt2 = optim.SelectiveAdamW([{"params": [a], "lr": 0.1}, {"params": [c], "lr": 0.1, "weight_decay": 0.0}], lr=0.0)
    c.grad = torch.ones_like(c)
    with pytest.raises(NotImplementedError, match="weight_decay"):
        opt2.step()


def test_to_fused_opts_in_through_the_environment(monkeypatch):
    p = torch.nn.Parameter(torch.zeros(5, 3))
    make = lambda: torch.optim.AdamW([{"params": [p], "lr": 1e-4, "name": "xyz"}], lr=0.0, eps=1e-15)  # noqa: E731
    monkeypatch.delenv("LGR_SELECTIVE_ADAM", raising=False)
    assert type(optim.to_fused(make())) is optim.FusedAdamW
    monkeypatch.setenv("LGR_SELECTIVE_ADAM", "1")
    sel = optim.to_fused(make())
    assert type(sel) is optim.SelectiveAdamW and sel.param_groups[0]["name"] == "xyz" and sel.param_groups[0]["eps"] == 1e-15


def test_dropin_refuses_selective_without_the_fused_optimizer():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]), LGR_SELECTIVE_ADAM="1", LGR_FUSED_OPTIM="0")
    r = subprocess.run([sys.executable, "-c", "import gaussian_renderer"], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "LGR_SELECTIVE_ADAM=1" in r.stderr, r.stderr[-2000:]
    env["LGR_FUSED_OPTIM"] = "1"
    r = subprocess.run([sys.executable, "-c", "import gaussian_renderer"], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
