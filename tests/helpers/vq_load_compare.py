"""Under our stack: the reference's GaussianModel with the patched load_vq against the class's own load_vq on the same files.
argv: <model dir with extreme_saving/> <result.json>"""
import json
import sys

import torch
import torch.nn.functional as F

from gaussian_renderer import GaussianModel, render
from lightgaussian_b200 import trace
from lightgaussian_b200.model import TorchCamera, pipeline_params
from lightgaussian_b200.synth import make_cameras

model_dir, out = sys.argv[1], sys.argv[2]
NAMES = ["_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"]
res = {"patched": bool(getattr(GaussianModel.load_vq, "_lgr_resident", False))}


def fresh(dense=False):
    g = GaussianModel(3)
    (GaussianModel.load_vq._lgr_dense if dense else GaussianModel.load_vq)(g, model_dir)
    return g


def same(x, y):
    return (type(x) is type(y) and x.dtype == y.dtype and x.shape == y.shape and x.stride() == y.stride()
            and x.is_contiguous() == y.is_contiguous() and x.requires_grad == y.requires_grad and torch.equal(x.detach(), y.detach()))


ref = fresh(dense=True)
a = fresh()
res["deferred_before_read"] = "_vq_resident" in a.__dict__ and type(a) is not GaussianModel
res["leaves_equal"] = [n for n in NAMES if same(getattr(a, n), getattr(ref, n))]
res["class_restored"] = type(a) is GaussianModel and "_vq_resident" not in a.__dict__

cam = TorchCamera(make_cameras(3, 96, 64)[1])
bg = torch.zeros(3, device="cuda")
pipe = pipeline_params()

# a grad-mode render straight after load: materialises, then the fused backward of the dense path
grads = {}
for key, g in (("ref", ref), ("ref_again", fresh(dense=True)), ("ours", fresh())):
    img = render(cam, g, pipe, bg)["render"]
    img.abs().mean().backward()
    grads[key] = [getattr(g, n).grad for n in NAMES]
# the blend backward sums with float atomics: where two dense runs already differ, ours may differ from either by as much
res["grad_spread"] = max(float((x - y).abs().max()) for x, y in zip(grads["ref"], grads["ref_again"]))
res["grads_equal"] = all(x is not None and (torch.equal(x, y) if res["grad_spread"] == 0.0 else
                                            float((x - y).abs().max()) <= 2 * res["grad_spread"])
                         for x, y in zip(grads["ours"], grads["ref"]))

with torch.no_grad():
    colors = torch.sigmoid(ref._xyz * 3.0)
    o = render(cam, fresh(), pipe, bg, override_color=colors)
    r = render(cam, ref, pipe, bg, override_color=colors)
    res["override_color_equal"] = torch.equal(o["render"], r["render"]) and torch.equal(o["radii"], r["radii"])
    cov_pipe = pipeline_params(compute_cov3D_python=True)
    o = render(cam, fresh(), cov_pipe, bg)
    r = render(cam, ref, cov_pipe, bg)
    res["cov3D_python_equal"] = torch.equal(o["render"], r["render"]) and torch.equal(o["radii"], r["radii"])
    g = fresh()
    res["capture_equal"] = (torch.equal(g.get_features, ref.get_features) and torch.equal(g.get_scaling, ref.get_scaling)
                            and torch.equal(g.get_rotation, F.normalize(ref._rotation)))
res["trace"] = dict(trace.counters)
with open(out, "w") as f:
    json.dump(res, f)
