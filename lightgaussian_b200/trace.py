"""Process-wide path counters.  The reference's scripts are run UNMODIFIED, so a test cannot ask them which of our code paths they
took; with LGR_TRACE=<file> set, the counters below are written to that file (JSON) when the interpreter exits:
    render_fused / render_unfused      gaussian_renderer.render()/count_render() calls through the raw-leaf kernels / the plain API
    render_fused_strided_rest          ... of which with a row-strided _features_rest (the distillation student)
    render_vq_resident / vq_materialize  calls that rendered a resident VQ model in place / resident models whose leaves were built
    adamw_steps / adamw_strided_params FusedAdamW.step() calls / row-strided parameters updated in place
    adamw_selective_steps              SelectiveAdamW.step() calls
    unfused_exchange                   view-parallel backward passes that took the dense all-reduce of the unfused node
    render_depth_alpha                 render(depth=..., alpha=...) calls (the fused node with the depth and alpha planes)
    raw_backward_depth / raw_backward_plain  backwards of that node through lgr_backward_raw_depth / through lgr_backward_raw, the
                                       latter when neither plane received a gradient
    render_absgrad / raw_backward_absgrad  render() calls through the fused node that also computes the absolute-gradient
                                       densification statistic (LGR_DENSIFY_GRAD=abs) / its backwards (lgr_backward_raw_absgrad)
    densify_stats_absgrad              add_densification_stats calls that added ||absgrad|| (LGR_DENSIFY_GRAD=abs)
Cost when LGR_TRACE is unset: one dict increment per call."""
from __future__ import annotations

import atexit
import json
import os

counters: dict = {}


def bump(name: str, by: int = 1) -> None:
    counters[name] = counters.get(name, 0) + by


def _dump() -> None:
    path = os.environ.get("LGR_TRACE")
    if path:
        try:
            with open(path, "w") as f:
                json.dump(counters, f)
        except OSError:
            pass


atexit.register(_dump)
