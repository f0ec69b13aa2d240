"""Drop-in for the reference's `simple_knn._C` extension (submodules/simple-knn).  scene/gaussian_model.py:20 imports it at module
import time, and GaussianModel.create_from_pcd calls distCUDA2 whenever a Scene is built from a dataset's point cloud (every script
that constructs Scene(dataset, gaussians) without load_iteration).  The native kernel is lightgaussian_b200/csrc/lgr_knn.cuh; importing
this module loads neither liblgrast.so nor a GPU, the first call does."""


def distCUDA2(points):
    from lightgaussian_b200.knn import distCUDA2 as native
    return native(points)
