#!/usr/bin/env python
"""bench.py -- training views/sec of the rasterizer hot path (BASELINE.json metric) on N GPUs of one node.

  python bench.py --gpus 1 --steps 20 --warmup 5                       # our sm_90a path
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
         bench.py --gpus N --steps K --warmup W                         # view-parallel, one rank per GPU
  python bench.py --impl reference ...                                  # the reference's own CUDA kernels (oracle/_ref)

A "step" is one training view per rank through the public API: gaussian_renderer.render() (activations, SH
concatenation, rasterizer forward) -> L1 image loss -> backward to the six raw parameter leaves; for N > 1 the
per-Gaussian gradients are then summed across ranks with ONE NCCL all-reduce (the path's only exchange).
Workload = BASELINE.json configs[2]: 3M synthetic Gaussians, SH degree 3, 1920x1080, synthetic cameras.
Prints ONE JSON line on rank 0.  --dump-outputs DIR also writes what the last timed step computed (the loss and a fixed, seeded
sample of 65 536 rows of every leaf gradient) as DIR/<name>.npy, so that two builds can be compared output for output.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

METRIC = "training views/sec at 3M Gaussians 1080p"
UNIT = "views/s"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", choices=["ours", "reference", "reference-kernels"], default="ours",
                    help="reference = the UNMODIFIED reference stack from oracle/_ref/stock (its pybind extension built from RAST/setup.py, its "
                         "gaussian_renderer.render, its GaussianModel, its l1_loss); reference-kernels = the reference's kernels behind our "
                         "own harness (oracle/_ref shim)")
    ap.add_argument("--mode", choices=["train", "distill"], default="train",
                    help="train = the headline step (render + L1 + backward); distill = one distill_train.py iteration "
                         "(student M=9 strided leaf + teacher M=16 renders, 0.8 L1 + 0.2 DSSIM, backward, AdamW step)")
    ap.add_argument("--P", type=int, default=3_000_000, help="number of Gaussians (default: the 3M workload)")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--cams", type=int, default=16, help="distinct synthetic cameras cycled through")
    ap.add_argument("--blend-mode", type=int, default=0, help="DIAGNOSTIC: 0 = ring blend kernels (default), 1 = the round-1 blend kernels")
    ap.add_argument("--bin-mode", type=int, default=2, help="binning: 2 = library radix sorts + scan (default, fastest measured), 0 = hand-written "
                    "kernels, blob sized from an estimate, no host sync, 1 = hand-written kernels, exact blob size (one stream sync)")
    ap.add_argument("--kback-mode", type=int, default=0, help="DIAGNOSTIC: fused K7+K8 of the raw backward: 0 = rows cleared inside the blend "
                    "backward + compacted list (default), 1 = dense kernel, 2 = separate zero-fill kernel + compacted list")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-exchange", action="store_true", help="DIAGNOSTIC ONLY (invalid for the metric): N>1 without any gradient exchange")
    ap.add_argument("--dense-allreduce", action="store_true", help="N>1: all-reduce the dense gradients instead of the compact SH exchange")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's loss and a seeded sample of its leaf gradients as DIR/<name>.npy")
    return ap.parse_args()


# ------------------------------------------------------------------------------------------------
# clocks, sampled DURING the timed region
# ------------------------------------------------------------------------------------------------
class ClockSampler:
    """nvidia-smi polled every 50 ms from construction on; every line is stamped on arrival, and only the lines that arrived
    between begin() and end() (the timed region, plus -- when that region is shorter than two polls -- an untimed continuation of
    the same steps, flagged in "window") are reported."""
    Q = "index,clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.lines = []
        self.proc = None
        self.t0 = self.t1 = None
        self.window = "timed region"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50",
                                          "-i", str(self.idx)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append((time.perf_counter(), line.strip()))

    def begin(self):
        self.t0 = time.perf_counter()

    def end(self):
        self.t1 = time.perf_counter()

    def in_window(self):
        return [ln for (t, ln) in list(self.lines) if self.t0 is not None and t >= self.t0 and (self.t1 is None or t <= self.t1)]

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        lines = self.in_window()
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for ln in lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[1]))
                mx.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None, "samples": len(sm),
                "reasons": sorted(reasons), "window": self.window}


# ------------------------------------------------------------------------------------------------
# the reference's kernels behind the same autograd surface (only for --impl reference)
# ------------------------------------------------------------------------------------------------
def make_reference_render():
    """render() whose rasterizer is the reference's own CUDA code (oracle/_ref/libref_rasterizer.so: forward.cu,
    backward.cu, rasterizer_impl.cu compiled unmodified).  Allocation behaviour follows the reference's torch binding
    (zero-filled outputs, RAST/rasterize_points.cu:79-80,254-262)."""
    import ctypes as C
    path = os.path.join(ROOT, "oracle", "_ref", "libref_rasterizer.so")
    if not os.path.exists(path):
        return None
    lib = C.CDLL(path)
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    lib.ref_state_create.restype = vp
    lib.ref_forward.restype = i
    lib.ref_forward.argtypes = [vp, i, i, i, i, vp, i, i, vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp, vp]
    lib.ref_backward.restype = None
    lib.ref_backward.argtypes = [vp, i, i, i, vp, i, i, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, vp, vp] + [vp] * 9
    state = lib.ref_state_create()

    class RefRasterize(torch.autograd.Function):
        @staticmethod
        def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, cam, bg, tanx, tany, H, W, deg):
            P, M = means3D.shape[0], sh.shape[1]
            color = torch.full((3, H, W), 0.0, dtype=torch.float32, device=means3D.device)
            radii = torch.full((P,), 0, dtype=torch.int32, device=means3D.device)
            ms, shc, op, sc, ro = means3D.contiguous(), sh.contiguous(), opacities.contiguous(), scales.contiguous(), rotations.contiguous()
            lib.ref_forward(state, 0, P, deg, M, bg.data_ptr(), W, H, ms.data_ptr(), shc.data_ptr(), None, op.data_ptr(), sc.data_ptr(),
                            1.0, ro.data_ptr(), None, cam.world_view_transform.data_ptr(), cam.full_proj_transform.data_ptr(),
                            cam.camera_center.data_ptr(), tanx, tany, 0, color.data_ptr(), radii.data_ptr(), None, None)
            ctx.save_for_backward(ms, shc, sc, ro, radii, bg)
            ctx.cam, ctx.meta = cam, (tanx, tany, H, W, deg)
            return color, radii

        @staticmethod
        def backward(ctx, g_color, _):
            ms, shc, sc, ro, radii, bg = ctx.saved_tensors
            tanx, tany, H, W, deg = ctx.meta
            cam = ctx.cam
            P, M = ms.shape[0], shc.shape[1]
            z = lambda *s: torch.zeros(s, dtype=torch.float32, device=ms.device)  # noqa: E731
            d2, dcon, dop, dcol, d3, dcov, dsh, dsc, dro = z(P, 3), z(P, 2, 2), z(P, 1), z(P, 3), z(P, 3), z(P, 6), z(P, M, 3), z(P, 3), z(P, 4)
            g = g_color.contiguous()
            lib.ref_backward(state, P, deg, M, bg.data_ptr(), W, H, ms.data_ptr(), shc.data_ptr(), None, sc.data_ptr(), 1.0, ro.data_ptr(),
                             None, cam.world_view_transform.data_ptr(), cam.full_proj_transform.data_ptr(), cam.camera_center.data_ptr(),
                             tanx, tany, radii.data_ptr(), g.data_ptr(), d2.data_ptr(), dcon.data_ptr(), dop.data_ptr(), dcol.data_ptr(),
                             d3.data_ptr(), dcov.data_ptr(), dsh.data_ptr(), dsc.data_ptr(), dro.data_ptr())
            return d3, d2, dsh, dop, dsc, dro, None, None, None, None, None, None, None

    def render(cam, pc, pipe, bg):
        xyz = pc.get_xyz
        ssp = torch.zeros_like(xyz, requires_grad=True) + 0
        img, radii = RefRasterize.apply(xyz, ssp, pc.get_features, pc.get_opacity, pc.get_scaling, pc.get_rotation, cam, bg,
                                        math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), int(cam.image_height),
                                        int(cam.image_width), pc.active_sh_degree)
        return {"render": img, "viewspace_points": ssp, "visibility_filter": radii > 0, "radii": radii}
    return render


def make_stock_reference(raw, dev):
    """The reference's own public path, UNMODIFIED (BASELINE.md section 2.1): `gaussian_renderer.render` + `scene.gaussian_model.GaussianModel`
    + the pybind extension `diff_gaussian_rasterization._C` built from RAST/setup.py (rasterize_points.cu:46-299), all from oracle/_ref/stock
    (staged by oracle/stage_reference.py).  Returns (render_fn, gaussians, l1_loss, AdamW-factory) or None when it is not staged."""
    ref = os.path.join(ROOT, "oracle", "_ref", "stock")
    tree = os.path.join(ref, "LightGaussian")
    ext = os.path.join(ref, "diff_gaussian_rasterization")
    if not (os.path.isfile(os.path.join(tree, "gaussian_renderer", "__init__.py")) and os.path.isdir(ext)
            and any(f.startswith("_C") and f.endswith(".so") for f in os.listdir(ext))):
        return None
    for p_ in (tree, os.path.join(ref, "shims"), ref):
        sys.path.insert(0, p_)
    for name in [m for m in sys.modules if m.split(".")[0] in ("gaussian_renderer", "diff_gaussian_rasterization", "utils", "scene")]:
        del sys.modules[name]
    import diff_gaussian_rasterization as dgr
    import gaussian_renderer as gr
    from scene.gaussian_model import GaussianModel
    from utils.loss_utils import l1_loss
    assert dgr.__file__.startswith(ref) and gr.__file__.startswith(tree), (dgr.__file__, gr.__file__)
    from torch import nn
    g = GaussianModel(3)
    leaf = lambda a: nn.Parameter(torch.from_numpy(np.ascontiguousarray(a)).float().to(dev).requires_grad_(True))  # noqa: E731
    g._xyz, g._features_dc, g._features_rest = leaf(raw["xyz"]), leaf(raw["features_dc"]), leaf(raw["features_rest"])
    g._scaling, g._rotation, g._opacity = leaf(raw["scaling"]), leaf(raw["rotation"]), leaf(raw["opacity"])
    g.active_sh_degree = 3
    g.parameters = lambda: [g._xyz, g._features_dc, g._features_rest, g._scaling, g._rotation, g._opacity]
    return gr.render, g, l1_loss


# ------------------------------------------------------------------------------------------------
def cpu_oracle_sample(scene, cam, W, H):
    """the CPU port (oracle/lgo.c, single thread) on ONE view of the same workload: forward + backward."""
    from oracle.lgo import Oracle, View
    act = scene["act"]
    v = View(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform, cam.camera_center,
             np.zeros(3, np.float32), 3, 1.0)
    o = Oracle()
    rng = np.random.default_rng(0)
    dpix = rng.standard_normal((3, H, W)).astype(np.float32)
    t0 = time.perf_counter()
    f = o.forward(v, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    o.backward(v, f, dpix, act["means3D"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    dt = time.perf_counter() - t0
    return 1.0 / dt, dt


def make_torch_reference_loss(dev):
    """(1-l)*l1_loss + l*(1-ssim) with l = 0.2 exactly as utils/loss_utils.py:18-85 composes it from torch ops (5 depthwise conv2d +
    elementwise + autograd): what the reference's training loops launch per iteration (prune_finetune.py:160-164)."""
    import torch.nn.functional as F
    g1 = torch.tensor([math.exp(-((k - 5) ** 2) / (2 * 1.5 ** 2)) for k in range(11)], device=dev)
    g1 = g1 / g1.sum()
    w2 = (g1[:, None] * g1[None, :]).expand(3, 1, 11, 11).contiguous()

    def torch_loss(x, y):
        cv = lambda t: F.conv2d(t[None], w2, padding=5, groups=3)[0]  # noqa: E731
        mu1, mu2 = cv(x), cv(y)
        s1, s2, s12 = cv(x * x) - mu1 * mu1, cv(y * y) - mu2 * mu2, cv(x * y) - mu1 * mu2
        m = ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))
        return 0.8 * (x - y).abs().mean() + 0.2 * (1.0 - m.mean())
    return torch_loss



def main_distill(args, rank, world, dev):
    """--mode distill: one distill_train.py iteration per step and rank (distill_train.py:124-166 with the C4 flags --new_max_sh 2
    --enable_covariance): student render (M = 9, _features_rest the NON-contiguous [P,8,3] view onedownSHdegree() leaves,
    scene/gaussian_model.py:129-136; opacity frozen), teacher render (M = 16, leaves require grad, image detached),
    0.8 L1 + 0.2 (1 - SSIM), backward, AdamW.step, zero_grad.  N > 1: each rank takes its own camera, student gradients summed."""
    from lightgaussian_b200 import parallel
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.synth import make_scene, make_cameras
    P, W, H = args.P, args.width, args.height
    scene = make_scene(P, sh_degree=3, seed=0)
    cams = [TorchCamera(c, dev) for c in make_cameras(args.cams, W, H)]
    bg = torch.zeros(3, device=dev)
    pipe = pipeline_params()
    names = ["_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"]
    lrs = [1.6e-4, 2.5e-3, 2.5e-3 / 20, 0.05, 0.005, 0.001]
    launches0 = 0
    if args.impl == "ours":
        from lightgaussian_b200 import capi, loss as fused_loss, optim as fused_optim, rasterizer
        from lightgaussian_b200.renderer import render as render_fn
        capi.load()
        teacher = GaussianParams(scene["raw"], 3, dev)
        student = GaussianParams(scene["raw"], 3, dev)
        student._features_rest = student._features_rest.clone().detach()[:, :8, :]      # onedownSHdegree(), verbatim
        student._features_rest.requires_grad = True
        student.max_sh_degree = student.active_sh_degree = 2
        student._opacity.requires_grad = False                                           # no --enable_opacity
        loss_fn = lambda x, y: fused_loss.l1_ssim_loss(x, y, 0.2)  # noqa: E731
        opt = fused_optim.FusedAdamW([{"params": [getattr(student, n)], "lr": lr, "name": n} for n, lr in zip(names, lrs)], lr=0.0, eps=1e-15)
        if world > 1:
            parallel.enable_gradient_exchange(world)
        kind = "fused kernels (strided student leaf read and updated in place)"
    else:
        stock = make_stock_reference(scene["raw"], dev)
        if stock is None:
            print(json.dumps({"impl": args.impl, "unavailable": "oracle/_ref/stock (stock reference stack) is not staged"}))
            return 0
        render_fn, teacher, _ = stock
        import copy
        student = copy.deepcopy(teacher)
        student.max_sh_degree = 2
        student.onedownSHdegree()
        student._opacity.requires_grad = False
        torch_loss = make_torch_reference_loss(dev)
        loss_fn = torch_loss
        opt = torch.optim.AdamW([{"params": [getattr(student, n)], "lr": lr, "name": n} for n, lr in zip(names, lrs)], lr=0.0, eps=1e-15)
        kind = "stock reference stack (oracle/_ref/stock) + torch loss composition + torch.optim.AdamW"
    assert not student._features_rest.is_contiguous()

    def step(k):
        cam = cams[(k * world + rank) % len(cams)]
        s_img = render_fn(cam, student, pipe, bg)["render"]
        t_img = render_fn(cam, teacher, pipe, bg)["render"].detach()
        loss_fn(s_img, t_img).backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    for k in range(args.warmup):
        step(k)
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    if args.impl == "ours":
        launches0 = capi.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(args.steps):
        step(args.warmup + k)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
    ms = float(ms.item())
    if rank == 0:
        line = {"metric": "distillation iterations/sec at 3M Gaussians 1080p (student SH2 + teacher SH3, views sharded over GPUs)",
                "value": args.steps * world / (ms * 1e-3), "unit": "views/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                "config": {"workload": f"{P} Gaussians, {W}x{H}, distill_train.py iteration: student SH degree 2 (strided [P,8,3] leaf) + teacher SH degree 3, "
                                       "0.8 L1 + 0.2 DSSIM, backward, AdamW", "gaussians": P, "resolution": [W, H], "cameras": len(cams)},
                "run": {"views_per_step": world, "path": kind},
                "gpu_launches": (capi.launch_count() - launches0) if args.impl == "ours" else 0}
        if args.impl != "ours":
            line["impl"] = args.impl
        elif world > 1:
            line["run"]["unfused_exchange_calls"] = rasterizer.unfused_exchange_calls()
        print(json.dumps(line))
    if world > 1:
        torch.distributed.destroy_process_group()
    return 0


def main():
    args = parse_args()
    from lightgaussian_b200 import parallel
    if args.impl != "ours":
        # the reference is single-GPU (utils/general_utils.py:151 pins cuda:0): under torchrun rank 0 alone runs it, the other
        # ranks exit without joining any process group
        if int(os.environ.get("RANK", "0")) != 0:
            return 0
        rank, world, local = 0, 1, int(os.environ.get("LOCAL_RANK", "0"))
    else:
        rank, world, local = parallel.init_from_env()
    assert torch.cuda.is_available(), "bench.py needs a GPU (there is no CPU path in the product)"
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if args.mode == "distill":
        return main_distill(args, rank, world, dev)

    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.synth import make_scene, make_cameras
    from lightgaussian_b200.trainstep import train_view
    P, W, H = args.P, args.width, args.height
    scene = make_scene(P, sh_degree=3, seed=0)
    cams_np = make_cameras(args.cams, W, H)
    pc = GaussianParams(scene["raw"], 3, dev)
    stock = None
    if args.impl == "reference":
        stock = make_stock_reference(scene["raw"], dev)
        if stock is not None:
            pc = stock[1]           # the reference's own GaussianModel holds the parameters
    cams = [TorchCamera(c, dev) for c in cams_np]
    bg = torch.zeros(3, device=dev)
    pipe = pipeline_params()
    params = pc.parameters()
    grad_bytes = sum(p.numel() for p in params) * 4

    def zero_grads():  # optimizer.zero_grad(set_to_none=True), as the reference loop does (prune_finetune.py:287-289)
        for p in params:
            p.grad = None

    fused_exchange = (args.impl == "ours" and world > 1 and os.environ.get("LGR_FUSED", "1") != "0" and not args.dense_allreduce
                      and not args.no_exchange)
    if fused_exchange:
        parallel.enable_gradient_exchange(world)   # gradients come out of backward() already summed over the ranks

    def allreduce_grads():  # the path's one exchange step: sum of the per-Gaussian gradients over the ranks (NCCL)
        if world > 1 and not fused_exchange and not args.no_exchange:
            hs = [torch.distributed.all_reduce(p.grad, op=torch.distributed.ReduceOp.SUM, async_op=True) for p in params]
            for h in hs:
                h.wait()

    gen = torch.Generator().manual_seed(1234)
    targets_host = [torch.rand(3, H, W, generator=gen).pin_memory() for _ in range(min(args.cams, 8))]
    targets_dev = [t.to(dev) for t in targets_host]
    cam_host = [(torch.from_numpy(c.world_view_transform).pin_memory(), torch.from_numpy(c.full_proj_transform).pin_memory(),
                 torch.from_numpy(c.camera_center).pin_memory()) for c in cams_np]

    if args.impl == "ours":
        from lightgaussian_b200 import capi, rasterizer
        from lightgaussian_b200.renderer import render as render_fn
        capi.load()
        capi.set_blend_mode(args.blend_mode)
        capi.set_binning_mode(args.bin_mode)
        capi.set_kback_mode(args.kback_mode)
        kind = None
    elif stock is not None:
        render_fn, kind = stock[0], "reference"
    else:
        render_fn = make_reference_render()
        kind = "reference-kernels"
        if render_fn is None:
            kind = "port"

    # the step's L1: each arm uses ITS OWN stack's l1_loss -- ours the fused kernel pair (lightgaussian_b200.loss, what
    # dropin/utils/loss_utils.py exports), the reference arm the torch composition of utils/loss_utils.py:18-19
    step_loss = None
    if args.impl == "ours" and os.environ.get("LGR_BENCH_TORCH_L1", "0") != "1":
        from lightgaussian_b200.loss import l1_loss as step_loss
    elif stock is not None:
        step_loss = stock[2]        # utils/loss_utils.py:18-19, the reference's own

    # which view a rank renders in a step.  N > 1: a step lasts as long as its slowest rank, so the views of one step are chosen with
    # similar cost (parallel.balanced_view_schedule on each camera's instance count, measured here by every rank for all cameras ->
    # the same schedule everywhere without communication); every camera is still used equally often.
    schedule = None
    if world > 1 and args.impl == "ours" and os.environ.get("LGR_BALANCED_VIEWS", "1") != "0":
        costs = []
        with torch.no_grad():
            for c in cams:
                render_fn(c, pc, pipe, bg)
                costs.append(rasterizer.last_num_rendered())
        schedule = parallel.balanced_view_schedule(costs, world)

    def view_index(step):
        if schedule is not None:
            return schedule[step % len(schedule)][rank]
        return (step * world + rank) % len(cams)

    def step_resident(step):
        i = view_index(step)
        zero_grads()
        loss = train_view(render_fn, cams[i], pc, pipe, bg, targets_dev[i % len(targets_dev)], step_loss)
        allreduce_grads()
        return loss

    # e2e: every step's camera and target image start in pinned HOST memory.  The copies are issued one step ahead on a
    # separate stream (copy engine) into a 2-deep device ring, so they overlap the previous step's kernels; the
    # compute stream waits on the copy's event before it touches the data.
    copy_stream = torch.cuda.Stream(device=dev)
    ring = [dict(wv=torch.empty(4, 4, device=dev), fp=torch.empty(4, 4, device=dev), cc=torch.empty(3, device=dev),
                 tgt=torch.empty(3, H, W, device=dev), ev=torch.cuda.Event(), used=torch.cuda.Event()) for _ in range(2)]
    e2e_cam = TorchCamera(cams_np[0], dev)

    def prefetch(step):
        slot = ring[step % 2]
        i = view_index(step)
        wv, fp, cc = cam_host[i]
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(slot["used"])          # the slot's previous consumer has finished
            slot["wv"].copy_(wv, non_blocking=True)        # H2D: this step's camera
            slot["fp"].copy_(fp, non_blocking=True)
            slot["cc"].copy_(cc, non_blocking=True)
            slot["tgt"].copy_(targets_host[i % len(targets_host)], non_blocking=True)  # H2D: this step's target image
            slot["ev"].record(copy_stream)

    e2e_state = {"primed": -1, "losses": []}
    loss_ring = [dict(host=torch.empty(1).pin_memory(), ev=torch.cuda.Event(), pending=False) for _ in range(2)]

    def step_e2e(step):
        if e2e_state["primed"] != step:
            prefetch(step)
        slot = ring[step % 2]
        prefetch(step + 1)
        e2e_state["primed"] = step + 1
        torch.cuda.current_stream().wait_event(slot["ev"])
        e2e_cam.world_view_transform, e2e_cam.full_proj_transform, e2e_cam.camera_center = slot["wv"], slot["fp"], slot["cc"]
        zero_grads()
        loss = train_view(render_fn, e2e_cam, pc, pipe, bg, slot["tgt"], step_loss)
        allreduce_grads()
        slot["used"].record()
        # D2H: the step's result goes to pinned host memory asynchronously and is READ one step later (the host never stalls the
        # launch of the next step; every step's value is read inside the timed region, the last one at its closing synchronise)
        res = loss_ring[step % 2]
        res["host"].copy_(loss.detach().reshape(1), non_blocking=True)
        res["ev"].record()
        prev = loss_ring[(step + 1) % 2]
        if prev["pending"]:
            prev["ev"].synchronize()
            e2e_state["losses"].append(float(prev["host"][0]))
        res["pending"] = True
        prev["pending"] = False
        return None

    def barrier():
        if world > 1:
            torch.distributed.barrier()

    def exchange_self_check():
        """N > 1, outside every timed region: on a 20k-Gaussian scene each rank renders ITS view and runs the exchanging backward; the
        summed leaf gradients must be (a) bit-identical on every rank -- replicas cannot drift -- and (b) within 1e-3 of the serial
        sum of the per-view gradients, which every rank recomputes locally with the exchange switched off.  Raises on failure, so a
        driver-run SCALE step cannot report a number for a broken exchange."""
        from lightgaussian_b200.synth import make_scene as mk_scene, make_cameras as mk_cams
        Ws, Hs = 320, 240
        sc = mk_scene(20000, sh_degree=3, seed=3, scale_mult=1.5)
        cs = [TorchCamera(c, dev) for c in mk_cams(world, Ws, Hs)]
        tg = [torch.rand(3, Hs, Ws, generator=torch.Generator().manual_seed(100 + r)).to(dev) for r in range(world)]
        ps = GaussianParams(sc["raw"], 3, dev)

        def grads_of(view):
            for q in ps.parameters():
                q.grad = None
            train_view(render_fn, cs[view], ps, pipe, bg, tg[view], step_loss)
            return [q.grad.detach().clone() for q in ps.parameters()]
        gx = grads_of(rank)                                   # exchanged: already the sum over all ranks' views
        parallel.enable_gradient_exchange(1)                  # serial reference on this rank
        try:
            serial = None
            for v_ in range(world):
                gv = grads_of(v_)
                serial = gv if serial is None else [a + b for a, b in zip(serial, gv)]
        finally:
            parallel.enable_gradient_exchange(world)
        worst, equal = 0.0, True
        for a, b in zip(gx, serial):
            worst = max(worst, float((a - b).abs().max() / b.abs().max().clamp_min(1e-20)))
            ref0 = a.clone()
            torch.distributed.broadcast(ref0, src=0)
            equal = equal and bool(torch.equal(ref0, a))
        flags = torch.tensor([1.0 if equal else 0.0, -worst], device=dev)
        torch.distributed.all_reduce(flags, op=torch.distributed.ReduceOp.MIN)
        res = {"bit_equal_across_ranks": bool(flags[0].item() == 1.0), "max_rel_err_vs_serial_sum": float(-flags[1].item()),
               "scene": "20000 Gaussians, 320x240, one view per rank", "unfused_exchange_calls": rasterizer.unfused_exchange_calls()}
        if not res["bit_equal_across_ranks"] or not res["max_rel_err_vs_serial_sum"] <= 1e-3:
            raise RuntimeError(f"gradient exchange self-check FAILED: {res}")
        return res

    def timed(fn, steps, sampler=None, after=None):
        barrier()
        torch.cuda.synchronize()
        if sampler:
            sampler.begin()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(steps):
            fn(args.warmup + s)
        e1.record()
        torch.cuda.synchronize()
        if after:
            after()
        clocks = None
        if sampler:
            sampler.end()
            if len(sampler.in_window()) < 2 and world == 1:
                # the timed region was shorter than two polls: keep the GPU under the SAME load (untimed) until 0.4 s have been sampled
                sampler.window = "timed region + untimed continuation of the same steps (region shorter than two 50 ms polls)"
                k = 0
                while time.perf_counter() - sampler.t0 < 0.4:
                    fn(args.warmup + steps + k)
                    k += 1
                torch.cuda.synchronize()
                sampler.end()
            clocks = sampler.stop()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
        return float(ms.item()), clocks

    # ---------------- the reference arm when its kernels could not be built: CPU port ----------------
    if args.impl != "ours" and kind == "port":
        v, dt = cpu_oracle_sample(scene, cams_np[0], W, H)
        line = {"impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": 1, "steps": 1, "warmup": 0,
                "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
                "data": "synthetic", "config": {"workload": f"{P} Gaussians SH3 {W}x{H} fwd+bwd, 1 view (CPU port of the reference algorithm)"},
                "cpu_baseline": {"value": v, "unit": UNIT, "cores": 1, "kind": "port", "sample": "1 view forward+backward, oracle/lgo.c single thread"},
                "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        print(json.dumps(line))
        return 0

    # ---------------- warm-up, then the timed regions ----------------
    sampler = ClockSampler(local) if rank == 0 else None      # starts polling now: nvidia-smi needs ~0.2 s to come up
    for s in range(args.warmup):
        step_resident(s)
    torch.cuda.synchronize()
    n0 = capi.launch_count() if args.impl == "ours" else 0
    dump = {}

    def capture_outputs():
        """what the last timed step computed: its loss and its leaf gradients, the latter as a fixed, seeded sample of rows"""
        if not args.dump_outputs:
            return
        rows = torch.randperm(P, generator=torch.Generator().manual_seed(2024))[:min(P, 65536)].sort().values.to(dev)
        dump["loss"] = last_loss[0].detach().double().reshape(1)
        dump["sample_rows"] = rows.double()
        for name, p_ in zip(("xyz", "features_dc", "features_rest", "scaling", "rotation", "opacity"), params):
            dump["grad_" + name] = p_.grad.detach().reshape(P, -1).index_select(0, rows).float()
        for k in dump:
            dump[k] = dump[k].cpu().numpy()

    last_loss = [None]

    def step_resident_kept(step):
        last_loss[0] = step_resident(step)

    ms, clocks = timed(step_resident_kept, args.steps, sampler, after=capture_outputs)
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, a in dump.items():
            np.save(os.path.join(args.dump_outputs, f"{k}.npy"), a)
    launches = (capi.launch_count() - n0) if args.impl == "ours" else 0
    views = args.steps * world
    value = views / (ms * 1e-3)

    e2e = None
    if not args.no_e2e:
        for s in range(2):
            step_e2e(s)
        e2e_state["losses"].clear()
        ms_e, _ = timed(step_e2e, args.steps)
        for r in loss_ring:                                          # the last step's value (its copy completed before timed() returned)
            if r["pending"]:
                e2e_state["losses"].append(float(r["host"][0]))
                r["pending"] = False
        assert len(e2e_state["losses"]) >= args.steps and all(math.isfinite(v) for v in e2e_state["losses"])
        h2d = 3 * H * W * 4 + (16 + 16 + 3) * 4
        e2e = {"value": views / (ms_e * 1e-3), "unit": UNIT, "ms_per_step": ms_e / args.steps, "h2d_bytes_per_step": h2d,
               "d2h_bytes_per_step": 4}

    exchange_check = exchange_self_check() if fused_exchange else None

    # ---------------- roofline of the dominant kernel (rank 0, our arm) ----------------
    roofline, stages = None, None
    if args.impl == "ours" and not args.no_roofline:   # every rank takes part (the backward contains collectives when N > 1)
        peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
        if os.path.exists(peaks_path):
            peak, peak_src = float(json.load(open(peaks_path))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, burst copy)"
        else:
            peak, peak_src = 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)"
        capi.profile_collect()
        capi.profile_enable(True)
        nprof = min(args.steps, 10)
        vis, Rs = [], []
        for s in range(nprof):
            i = view_index(args.warmup + s)
            zero_grads()
            pkg = render_fn(cams[i], pc, pipe, bg)
            (pkg["render"] - targets_dev[i % len(targets_dev)]).abs().mean().backward()
            vis.append(int((pkg["radii"] > 0).sum().item()))
            Rs.append(int(rasterizer.last_num_rendered()))
        prof = capi.profile_collect()
        capi.profile_enable(False)
        barrier()
        Pv, R, N, M = float(np.mean(vis)), float(np.mean(Rs)), W * H, 16
        nnz_est = 0.13 * P    # Gaussians with a non-zero gradient per view (measured 12-13 % on this scene, scripts/exp_grad_density.py)
        # ALGORITHMIC bytes per launch (SURVEY.md section 8d, split per kernel in DESIGN.md section 4)
        alg = {
            "preprocess_kernel": 12 * P + Pv * (32 + 12 * M) + 4 * P + 40 * Pv,
            "depth_sort(cub)": 16 * P, "scan(cub)": 8 * P, "emit_kernel": 12 * Pv + 6 * R, "tile_sort(cub)": 12 * R,
            "ranges_kernel": 2 * R,
            # hand-written binning (csrc/lgr_bin.cuh): keys+ids read and written once; 16-byte bin record + id per Gaussian read by the
            # count and by the scatter, 4 bytes per listed instance written (R here = the reference's num_rendered >= instances listed)
            "depth_sort(dsort_count+bin_scan+dsort_scatter x3)": 16 * P, "tile_count_kernel+bin_scan_kernel": 20 * P,
            "tile_scatter_kernel": 20 * P + 4 * R,
            "blend_forward_kernel": 40 * R + 20 * N,
            # the P*(56+12M) bytes of dense gradient rows are written (cleared) by the blend backward's producer thread in kback mode 0,
            # by the K7+K8 kernels otherwise: the bytes follow the kernel that moves them
            "blend_backward_kernel": 20 * N + 40 * R + 44 * Pv + (P * (56 + 12 * M) if (args.kback_mode == 0 and world == 1) else 0),
            "preprocess_backward_kernel": 44 * Pv + 12 * P + Pv * (32 + 12 * M) + (0 if args.kback_mode == 0 else P * (56 + 12 * M)),
            # view-parallel exchange (N > 1): pack = accumulator records in, per listed Gaussian its parameters in and one 64-byte row out to
            # every rank; accumulate = every rank's bitmap + prefix + rows in, xyz in, the dense summed gradient rows out
            "sparse_pack(flag+scan+index+K8)": 48 * P + nnz_est * (44 + 12 * M + 64 * world),
            "sparse_accumulate_kernel": P * (56 + 12 * M) + 12 * P + world * (P // 4 + nnz_est * 64),
            "memset": 48 * P,
            "sh_grad_from_views_kernel": 12 * P + 12 * P * world + 12 * M * P,
            "peer_allreduce_kernel": 2 * 44 * P * (world - 1) / max(world, 1),
        }
        stages = {k: {"ms_per_launch": ms_k / n, "launches": n, "alg_bytes": alg.get(k),
                      "gbs": (alg[k] / (ms_k / n * 1e-3) / 1e9) if k in alg else None}
                  for k, (ms_k, n) in prof.items() if n > 0}
        # the dominant stage among those with an algorithmic-byte figure (every kernel of the path has one; guards against a new stage name)
        rated = [k for k in stages if stages[k]["gbs"] is not None] or list(stages)
        top = max(rated, key=lambda k: stages[k]["ms_per_launch"] * stages[k]["launches"])
        ach = stages[top]["gbs"] or 0.0
        tot_ms = sum(v["ms_per_launch"] * v["launches"] for v in stages.values()) / nprof
        Bf = 12 * P + Pv * (32 + 12 * M) + 4 * P + 40 * Pv + 28 * R + 40 * R + 20 * N
        Bb = 20 * N + 40 * R + 88 * Pv + 12 * P + Pv * (32 + 12 * M) + P * (56 + 12 * M)
        roofline = {"bound": "hbm", "kernel": top, "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak,
                    "peak_source": peak_src,
                    "share_of_native_time": stages[top]["ms_per_launch"] * stages[top]["launches"] / nprof / tot_ms,
                    "whole_view": {"alg_bytes": Bf + Bb, "native_ms_per_view": tot_ms,
                                   "achieved": (Bf + Bb) / (tot_ms * 1e-3) / 1e9, "frac": (Bf + Bb) / (tot_ms * 1e-3) / 1e9 / peak},
                    "measured": {"P_visible": Pv, "num_rendered": R}}

    # ---------------- significance pass (prune.prune_list): count_render over this rank's cameras ----------------
    signif = None
    if args.impl == "ours" and not args.no_roofline:
        from lightgaussian_b200.renderer import count_render
        with torch.no_grad():
            for i in range(3):
                count_render(cams[i], pc, pipe, bg)
            nsig = min(len(cams), 16)
            t_sig, _ = timed(lambda s: count_render(cams[(s * world + rank) % len(cams)], pc, pipe, bg), nsig)
        signif = {"value": nsig * world / (t_sig * 1e-3), "unit": "views/s", "views": nsig * world,
                  "what": "count_render() (forward + exact Global Significance counts), cameras sharded over ranks"}

    # ---------------- image-loss pass (row N2): (1-l)*L1 + l*(1-SSIM) forward+backward on one HxW image ----------------
    loss_pass = None
    if args.impl == "ours" and not args.no_roofline and world == 1:
        from lightgaussian_b200 import loss as fused_loss
        gimg = torch.rand(3, H, W, device=dev)
        gtgt = torch.rand(3, H, W, device=dev)
        torch_loss = make_torch_reference_loss(dev)

        def run(fn):
            def step(_s):
                x = gimg.detach().requires_grad_(True)
                fn(x, gtgt).backward()
            for _ in range(3):
                step(0)
            t, _ = timed(step, 20)
            return t / 20
        t_f = run(lambda x, y: fused_loss.l1_ssim_loss(x, y, 0.2))
        t_t = run(torch_loss)
        loss_pass = {"fused_ms": t_f, "torch_composed_ms": t_t, "image": [3, H, W],
                     "alg_bytes": 3 * H * W * 4 * (2 + 3 + 2 + 3 + 1),
                     "what": "l1_ssim_loss forward+backward (lgr_image_loss_forward/backward) vs the reference's torch op sequence"}

    # ---------------- whole training iteration (rows N2 + N3 included): render -> L1+DSSIM -> backward -> AdamW -> zero_grad ------
    # prune_finetune.py:144-166,287-289.  Reported beside the headline (whose step definition stays render+L1+backward).
    iteration_pass = None
    if not args.no_roofline and (world == 1 or args.impl == "ours"):
        names = ["_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"]
        lrs = [1.6e-4, 2.5e-3, 2.5e-3 / 20, 0.05, 0.005, 0.001]                       # arguments/__init__.py OptimizationParams
        groups = lambda: [{"params": [getattr(pc, n)], "lr": lr, "name": n} for n, lr in zip(names, lrs)]  # noqa: E731
        torch_loss = make_torch_reference_loss(dev)

        def make_iter(loss_fn, opt):
            def it(step):
                i = view_index(step)
                img = render_fn(cams[i], pc, pipe, bg)["render"]
                loss_fn(img, targets_dev[i % len(targets_dev)]).backward()
                opt.step()
                opt.zero_grad(set_to_none=True)
            return it
        zero_grads()
        arms = {}
        if world == 1:
            arms["torch_loss_and_adamw"] = (torch_loss, torch.optim.AdamW(groups(), lr=0.0, eps=1e-15))
        if args.impl == "ours":
            from lightgaussian_b200 import loss as fused_loss, optim as fused_optim
            arms["fused_loss_and_adamw"] = (lambda x, y: fused_loss.l1_ssim_loss(x, y, 0.2), fused_optim.FusedAdamW(groups(), lr=0.0, eps=1e-15))
        iteration_pass = {"what": "render + (0.8 L1 + 0.2 DSSIM) + backward (+ gradient exchange when N > 1) + AdamW.step + zero_grad; views/s over all ranks",
                          "unit": "views/s"}
        nit = min(args.steps, 10)
        for name, (lf, opt) in arms.items():
            fn = make_iter(lf, opt)
            for s_ in range(3):
                fn(s_)
            t_it, _ = timed(fn, nit)
            iteration_pass[name] = nit * world / (t_it * 1e-3)
            if name == "fused_loss_and_adamw":
                # device time of the N2/N3 kernels inside this iteration (library CUDA events), against the HBM peak
                peak_rows = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]) \
                    if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
                capi.profile_collect()
                capi.profile_enable(True)
                for s_ in range(5):
                    fn(s_)
                prof_rows = capi.profile_collect()
                capi.profile_enable(False)
                n_el = sum(getattr(pc, n).numel() for n in names)
                alg_rows = {"adamw_multi_kernel": 28 * n_el, "image_loss_forward_kernel": 3 * H * W * 20,
                            "image_loss_backward_kernel": 3 * H * W * 24}
                rows = {}
                for kname, (ms_tot, nl) in prof_rows.items():
                    if kname in alg_rows and nl:
                        ms1 = ms_tot / nl
                        rows[kname] = {"ms_per_launch": ms1, "alg_bytes": alg_rows[kname], "gbs": alg_rows[kname] / (ms1 * 1e-3) / 1e9,
                                       "frac_of_hbm_peak": alg_rows[kname] / (ms1 * 1e-3) / 1e9 / peak_rows}
                iteration_pass["kernels"] = rows
                # every native stage of one iteration (ms per iteration, this rank): where a view-parallel iteration spends its time
                iteration_pass["stages_ms_per_iteration"] = {k: ms_tot / 5 for k, (ms_tot, nl) in prof_rows.items() if nl}
                t_h0 = time.perf_counter()
                for s_ in range(5):
                    fn(100 + s_)
                t_h1 = time.perf_counter()           # host time to ENQUEUE an iteration (no synchronisation inside)
                torch.cuda.synchronize()
                iteration_pass["host_enqueue_ms_per_iteration"] = (t_h1 - t_h0) * 1e3 / 5
            del opt
        zero_grads()

    # ---------------- VecTree k-means iteration (row N4): 80 000 samples x 8192 codes x 27 dims, importance weighted ----------------
    vq_pass = None
    if args.impl == "ours" and world == 1 and not args.no_roofline:
        try:
            from lightgaussian_b200 import vectree as fused_vq
            nv, dv, Kv = 80000, 27, 8192
            gv = torch.Generator(device=dev).manual_seed(3)
            xv = torch.randn(nv, dv, device=dev, generator=gv) * 0.5
            wv = torch.rand(nv, device=dev, generator=gv) ** 2
            model_vq = fused_vq.VectorQuantize(dim=dv, codebook_size=Kv).to(dev).train()
            embed_t = model_vq._codebook.embed[0].clone()
            cs_t = torch.zeros(Kv, device=dev)

            def ours_iter(_s):
                model_vq(xv.unsqueeze(0), weight=wv.reshape(1, -1, 1))

            def torch_iter(_s):                        # vq.py:262-300 op for op: cdist, argmax, one_hot, broadcast multiply, einsum, EMA
                wn = (wv * wv.numel() / wv.sum()).reshape(1, -1, 1)
                flat = xv[None]
                ind = (-torch.cdist(flat, embed_t[None], p=2)).argmax(dim=-1)
                onehot = torch.nn.functional.one_hot(ind, Kv).type(xv.dtype)
                cs = cs_t * 0.8 + 0.2 * (onehot * wn).sum(dim=1)[0]
                esum = torch.einsum("hnd,hnc->hcd", flat * wn, onehot)[0]
                sm = (cs + 1e-5) / (cs.sum() + Kv * 1e-5) * cs.sum()
                return embed_t * 0.8 + 0.2 * esum / sm[:, None]
            for fn in (ours_iter, torch_iter):
                for _ in range(2):
                    fn(0)
            capi.profile_collect()
            capi.profile_enable(True)
            t_o, _ = timed(ours_iter, 10)
            prof_vq = capi.profile_collect()
            capi.profile_enable(False)
            t_t, _ = timed(torch_iter, 5)
            ms_assign = prof_vq["vq_assign_kernel"][0] / max(prof_vq["vq_assign_kernel"][1], 1)
            flops = 2.0 * nv * Kv * dv
            # the same iteration with the nearest-code search forced onto the FP32 FFMA kernel (round 1's path), for comparison
            fp32_only = None
            try:
                capi.set_vq_mode(1)
                for _ in range(2):
                    ours_iter(0)
                capi.profile_collect()
                capi.profile_enable(True)
                t_f, _ = timed(ours_iter, 10)
                prof_f = capi.profile_collect()
                capi.profile_enable(False)
                ms_assign_f = prof_f["vq_assign_kernel"][0] / max(prof_f["vq_assign_kernel"][1], 1)
                fp32_only = {"fused_ms": t_f / 10, "assign_ms": ms_assign_f, "assign_tflops_fp32": flops / (ms_assign_f * 1e-3) / 1e12}
            except Exception as ex:  # noqa: BLE001  (an auxiliary comparison must never take the bench line down)
                fp32_only = {"error": f"{type(ex).__name__}: {ex}"}
            finally:
                capi.profile_enable(False)
                capi.set_vq_mode(0)
            vq_pass = {"fused_ms": t_o / 10, "torch_formulation_ms": t_t / 5, "assign_ms": ms_assign, "samples": nv, "codes": Kv, "dim": dv,
                       "fp32_kernel_only": fp32_only,
                       "what": "one importance-weighted EMA k-means iteration (VectorQuantize.forward in training mode); assign = operand split + "
                               "wgmma coarse pass (bf16 hi/lo, K = 96, FP32 accumulators in registers) + exact FP32 rescore of the undecided rows; "
                               "fp32_kernel_only = the FFMA kernel alone (2*n*K*d flops)"}
            del model_vq, xv, wv
        except Exception as ex:  # noqa: BLE001  (an auxiliary pass must never take the bench line down)
            vq_pass = {"error": f"{type(ex).__name__}: {ex}"}

    cpu_baseline = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        if args.impl == "ours":
            v_cpu, dt = cpu_oracle_sample(scene, cams_np[0], W, H)
            cpu_baseline = {"value": v_cpu, "unit": UNIT, "cores": 1, "kind": "port",
                            "sample": f"1 view forward+backward of the same workload ({dt:.1f} s), oracle/lgo.c single thread; host has {os.cpu_count()} cores"}
        else:
            how = ("its stock public path: gaussian_renderer.render + GaussianModel + the pybind extension built from RAST/setup.py (oracle/_ref/stock)"
                   if kind == "reference" else
                   "its kernels behind our harness (oracle/_ref: forward.cu/backward.cu/rasterizer_impl.cu compiled unmodified for sm_90a)")
            cpu_baseline = {"value": value, "unit": UNIT, "cores": 0, "kind": "reference",
                            "sample": f"the reference has NO CPU implementation of this path: this arm times {how} on the same GPU, "
                                      f"same steps; host has {os.cpu_count()} cores"}

    if args.impl == "ours" and os.environ.get("LGR_EXCHANGE_TIMING", "0") == "1":
        print(f"[rank {rank}] exchange timing: {rasterizer.exchange_timing_report()}", file=sys.stderr)
    xdesc, xbytes = None, None
    if fused_exchange:
        mode, rows = rasterizer.exchange_info(world)
        if mode.startswith("sparse-p2p"):
            how = ("WRITES them into every peer's buffer from inside its pack kernel (posted stores over NVLink); after one barrier each rank "
                   "accumulates from local memory") if mode.endswith("push") else "and reads every peer's rows in its accumulate kernel"
            xdesc = (f"sparse over NVLink peer memory ({mode}): each rank packs bitmap + 64-byte rows of the Gaussians with a non-zero gradient "
                     f"({rows} of {P} in rank 0's last view) {how}; no NCCL call")
            xbytes = (world - 1) * (rows * 64 + P // 4)
        else:
            xdesc = "dense (NCCL): all-reduce 44 B/Gaussian + all-gather dRGB 12 B/Gaussian/rank, SH gradient rebuilt locally"
            xbytes = P * 44 + P * 12 * world
    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            # `config` identifies the WORKLOAD only, so that both arms (and every N) print the same object; how this run executed it
            # (ranks, exchange, which code path) is under "run"
            "config": {"workload": f"{P} Gaussians SH degree 3, {W}x{H}, {len(cams)} synthetic cameras (Fibonacci sphere r=3), "
                                   "step = one training view per GPU: render() + L1 + backward to the six raw leaves",
                       "gaussians": P, "resolution": [W, H], "cameras": len(cams),
                       "l2_policy": "inputs larger than L2 (>=0.7 GB of parameters streamed per step)"},
            "run": {"views_per_step": world, "parallelism": f"view-parallel x{world}", "l1": "each stack's own l1_loss",
                    "grad_exchange": ("none" if world == 1 else "DISABLED (diagnostic run, not a valid measurement)" if args.no_exchange else
                                      (xdesc if fused_exchange else "dense all-reduce")),
                    "grad_exchange_bytes_per_rank": 0 if world == 1 else (xbytes if fused_exchange else grad_bytes),
                    "path": ("fused activations + raw-leaf kernels" if (args.impl == "ours" and os.environ.get("LGR_FUSED", "1") != "0") else
                             "reference-compatible API path" if args.impl == "ours" else kind)},
            "clocks": clocks, "gpu_launches": launches,
        }
        if args.impl == "ours":
            line["run"]["binning"] = {"mode": args.bin_mode, "repeats_for_capacity": capi.binning_overflows(),
                                      "what": "views whose binning blob estimate was too small (scatter + blend repeated), whole run"}
        if args.impl != "ours":
            line["impl"] = args.impl
            line["e2e"] = {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
            if e2e:
                line["e2e_host_buffers"] = e2e
        else:
            line["e2e"] = e2e
        if exchange_check:
            line["exchange_check"] = exchange_check
        if roofline:
            line["roofline"] = roofline
            line["stages"] = stages
        if signif:
            line["significance_pass"] = signif
        if loss_pass:
            line["loss_pass"] = loss_pass
        if iteration_pass:
            line["iteration_pass"] = iteration_pass
        if vq_pass:
            line["vq_pass"] = vq_pass
        if cpu_baseline:
            line["cpu_baseline"] = cpu_baseline
        print(json.dumps(line))
    if world > 1:
        torch.distributed.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
