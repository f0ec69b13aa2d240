"""The drop-in packages keep the reference's import surface: with <repo>/dropin and <repo> ahead of the reference checkout
on sys.path, the reference's own modules (scene.gaussian_model, prune, gaussian_renderer users) import unmodified.
The parts that need the reference's Python tree use the verbatim copy oracle/stage_reference.py stages under oracle/_ref/stock and
skip where it was not staged."""
import importlib
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "stock", "LightGaussian")


def test_plyfile_shim_roundtrip(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    try:
        plyfile = importlib.import_module("plyfile")
        names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "rot_0"]
        data = np.empty(17, dtype=[(n, "f4") for n in names])
        rng = np.random.default_rng(0)
        for n in names:
            data[n] = rng.standard_normal(17).astype(np.float32)
        path = str(tmp_path / "pc.ply")
        plyfile.PlyData([plyfile.PlyElement.describe(data, "vertex")]).write(path)
        back = plyfile.PlyData.read(path)
        assert [p.name for p in back.elements[0].properties] == names
        for n in names:
            np.testing.assert_array_equal(np.asarray(back.elements[0][n]), data[n])
        np.testing.assert_array_equal(back["vertex"]["x"], data["x"])
    finally:
        sys.path.remove(os.path.join(ROOT, "dropin"))
        sys.modules.pop("plyfile", None)


@pytest.mark.skipif(not os.path.isdir(REF), reason="oracle/_ref/stock/LightGaussian is not staged")
def test_reference_modules_import_against_the_dropins():
    """`scene.gaussian_model` (needs simple_knn._C, plyfile), `prune` (needs gaussian_renderer.count_render, icecream) and the
    GaussianModel getters work on top of our packages -- in a clean interpreter with the documented PYTHONPATH order."""
    code = r"""
import sys, torch
import gaussian_renderer, diff_gaussian_rasterization
assert gaussian_renderer.__file__.startswith(%r), gaussian_renderer.__file__
assert diff_gaussian_rasterization.__file__.startswith(%r)
from gaussian_renderer import render, count_render, network_gui, GaussianModel
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
import prune                                   # reference module: `from gaussian_renderer import render, count_render`, `from icecream import ic`
from scene.gaussian_model import GaussianModel as GM
assert GM is GaussianModel
g = GM(3)
assert g.scaling_activation is torch.exp and g.opacity_activation is torch.sigmoid
assert g.rotation_activation is torch.nn.functional.normalize
from arguments import PipelineParams
from lightgaussian_b200 import optim
assert GM.prune_points is optim.prune_points and GM.training_setup.__wrapped__ is not None     # row N3 installed by the drop-in
import vectree.utils, vectree.vq, lightgaussian_b200.vectree                                    # row N4 overlay
assert vectree.utils.load_vqgaussian is lightgaussian_b200.vectree.load_vqgaussian
assert vectree.utils.write_ply_data.__code__.co_filename.startswith(%r) and vectree.vq.__file__.startswith(%r)
import scene.gaussian_model as sgm
assert sgm.load_vqgaussian is lightgaussian_b200.vectree.load_vqgaussian                       # what GaussianModel.load_vq calls (:420-422)
print("ok")
""" % (os.path.join(ROOT, "dropin"), os.path.join(ROOT, "dropin"), REF + os.sep, REF + os.sep)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, REF]))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]


@pytest.mark.skipif(not os.path.isdir(REF), reason="oracle/_ref/stock/LightGaussian is not staged")
def test_reference_scripts_import_unmodified_against_the_dropins():
    """prune_finetune.py, distill_train.py, train_densify_prune.py, render.py, render_video.py, prune.py and metrics.py -- the callers of the hot
    path (SURVEY.md section 8a) -- import with the documented PYTHONPATH order: every `from gaussian_renderer / diff_gaussian_rasterization /
    utils.loss_utils / vectree.utils / scene import ...` they do resolves (to ours where we replace it, to the reference's file otherwise)."""
    code = r"""
import sys, importlib
sys.argv = ["x"]
for m in ["prune_finetune", "distill_train", "train_densify_prune", "render", "render_video", "prune", "metrics"]:
    mod = importlib.import_module(m)
    assert mod.__file__.startswith(%r), mod.__file__
import prune_finetune, metrics
import lightgaussian_b200.renderer as ours, lightgaussian_b200.loss as ours_loss
assert prune_finetune.render is ours.render
assert prune_finetune.l1_loss.__module__ == "utils.loss_utils" and prune_finetune.l1_loss.__code__.co_filename.startswith(%r)
assert metrics.ssim.__code__.co_filename.startswith(%r)
print("ok")
""" % (REF + os.sep, os.path.join(ROOT, "dropin"), os.path.join(ROOT, "dropin"))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT, REF]))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600, cwd=tempfile.gettempdir())
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]
