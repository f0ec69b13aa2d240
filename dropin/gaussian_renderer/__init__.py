"""Drop-in for the reference's `gaussian_renderer` package (render, count_render, network_gui, GaussianModel)."""
from lightgaussian_b200.renderer import render, count_render  # noqa: F401
from . import network_gui  # noqa: F401

import os as _os

try:  # render.py:22 / render_video.py:23 do `from gaussian_renderer import GaussianModel`
    from scene.gaussian_model import GaussianModel  # noqa: F401
except Exception:  # reference checkout not on the path: the name is simply absent
    GaussianModel = None

from lightgaussian_b200.renderer import significance_mode as _significance_mode  # noqa: E402
_significance_mode()   # an unknown LGR_SIGNIFICANCE fails here, not at the first prune
from lightgaussian_b200.renderer import densify_grad_mode as _densify_grad_mode  # noqa: E402
if _densify_grad_mode() == "abs" and _os.environ.get("LGR_FUSED_OPTIM", "1") == "0":
    # LGR_FUSED_OPTIM=0 keeps the class's own add_densification_stats, which would silently accumulate the reference's statistic
    raise RuntimeError("LGR_DENSIFY_GRAD=abs needs the native densification: it cannot be combined with LGR_FUSED_OPTIM=0")
if _os.environ.get("LGR_SELECTIVE_ADAM", "0") == "1" and _os.environ.get("LGR_FUSED_OPTIM", "1") == "0":
    raise RuntimeError("LGR_SELECTIVE_ADAM=1 needs the fused optimizer: it cannot be combined with LGR_FUSED_OPTIM=0")
if GaussianModel is not None and _os.environ.get("LGR_FUSED_OPTIM", "1") != "0":
    # row N3: the AdamW built by GaussianModel.training_setup becomes FusedAdamW (bit-identical updates, one launch per step)
    # and prune_points uses the fused compaction; LGR_FUSED_OPTIM=0 keeps torch.optim.AdamW and the reference's surgery.
    # LGR_SELECTIVE_ADAM=1 makes it a SelectiveAdamW (opt-in: only Gaussians with a non-zero gradient row are stepped).
    from lightgaussian_b200 import optim as _optim
    _optim.install(GaussianModel)
if GaussianModel is not None and hasattr(GaussianModel, "load_vq") and _os.environ.get("LGR_FUSED", "1") != "0":
    # render.py / render_video.py --load_vq: the compressed model stays resident and render() reads it in place; the five leaves
    # other than _xyz are built only when something reads or assigns one.  LGR_FUSED=0 keeps the reference's dense load_vq.
    from lightgaussian_b200 import vqresident as _vqresident
    _vqresident.install(GaussianModel)
if GaussianModel is None:
    del GaussianModel
