"""lightgaussian_b200 -- H100 (sm_90a) implementation of LightGaussian's rasterizer hot path.

Public surface (same names as the reference):
    GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians   (diff_gaussian_rasterization)
    render, count_render                                                      (gaussian_renderer)
Importing the rasterizer requires the native library liblgrast.so; there is no CPU fallback.
"""
__version__ = "0.1.0"


def __getattr__(name):  # lazy: `import lightgaussian_b200.synth` must not pull in torch
    if name in ("GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"):
        from . import rasterizer
        return getattr(rasterizer, name)
    if name in ("render", "count_render"):
        from . import renderer
        return getattr(renderer, name)
    raise AttributeError(name)
