"""Run with a stack's PYTHONPATH (tests/scripts_harness.py): build the reference's Scene(dataset, GaussianModel(3)) from a COLMAP
dataset, as prune_finetune.py / train_densify_prune.py do without load_iteration, so that GaussianModel.create_from_pcd sets the
initial scales from distCUDA2 (scene/gaussian_model.py:152-156); save _scaling as .npy."""
import sys
from argparse import ArgumentParser

import numpy as np

from arguments import ModelParams
from scene import Scene
from scene.gaussian_model import GaussianModel
import simple_knn._C  # after torch (scene imports it): the reference's extension links libc10

source, model_dir, out_path = sys.argv[1], sys.argv[2], sys.argv[3]
parser = ArgumentParser()
lp = ModelParams(parser)
dataset = lp.extract(parser.parse_args(["-s", source, "-m", model_dir]))
g = GaussianModel(3)
Scene(dataset, g)
np.save(out_path, g._scaling.detach().cpu().numpy())
print("scaling", tuple(g._scaling.shape))
print("distCUDA2 from", simple_knn._C.__file__)
