"""SelectiveAdamW (lgr_adamw_step_selective): AdamW on the Gaussians whose gradient row is not all zero.

The reference is torch.optim.AdamW stepped on copies, with the rows the mask calls inactive restored afterwards from a pre-step
copy of the parameter and both moments.  Every parameter and moment must equal it bit for bit (NaN rows: NaN in the same places)."""
import copy
import math
import types

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi, optim
from lightgaussian_b200.optim import FusedAdamW, SelectiveAdamW

pytestmark = pytest.mark.gpu
NAMES = ["xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"]
SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
LRS = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 2.5e-3 / 20, "opacity": 0.05, "scaling": 0.005, "rotation": 0.001}
KINDS = ["none", "all", "rand13", "single", "negzero", "nan", "scale1e-18", "scale1e-21", "scale1e30"]


def _same(a, b):
    """bit-identical, except that a NaN only has to meet a NaN (its payload is not specified)"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.detach()[~na].view(torch.int32), b.detach()[~nb].view(torch.int32))


def _active(grads, P):
    act = torch.zeros(P, dtype=torch.bool, device="cuda")
    for g in grads:
        if g.numel():
            act |= (g.reshape(P, -1) != 0).any(dim=1)
    return act


def _masked_grads(shapes, P, kind, gen):
    """gradients [P, *shape] whose non-zero rows follow `kind`"""
    base = []
    for s in shapes:
        x = torch.randn((P,) + s, generator=gen) * (10.0 ** float(torch.randint(-6, 1, (1,), generator=gen)))
        x[torch.rand((P,) + s, generator=gen) < 0.1] = 0.0              # zeros inside active rows too
        base.append(x)
    rows = torch.rand(P, generator=gen)
    if kind == "none":
        keep = torch.zeros(P, dtype=torch.bool)
    elif kind == "all":
        keep = torch.ones(P, dtype=torch.bool)
        for x in base:                                                  # no row of any group all zero
            x[x == 0] = 1e-3
    elif kind.startswith("scale"):
        keep = rows < 0.5
        base = [x * float(kind[5:]) for x in base]
    else:
        keep = rows < 0.13
    out = [torch.where(keep.view((P,) + (1,) * len(s)), x, torch.zeros(())) for x, s in zip(base, shapes)]
    if kind == "single":                                                # rows active through ONE element of ONE group
        out = [torch.zeros_like(x) for x in out]
        for r in torch.nonzero(keep).flatten().tolist():
            k = int(torch.randint(0, len(shapes), (1,), generator=gen))
            if out[k][r].numel():
                out[k][r].view(-1)[int(torch.randint(0, out[k][r].numel(), (1,), generator=gen))] = 0.5
    elif kind == "negzero":                                             # -0.0 everywhere outside the active rows
        out = [torch.where(keep.view((P,) + (1,) * len(s)), x, torch.full((), -0.0)) for x, s in zip(out, shapes)]
    elif kind == "nan" and P > 1:                                       # a row with one NaN, not otherwise active
        r = int(torch.nonzero(~keep).flatten()[0]) if (~keep).any() else 0
        out[0][r].view(-1)[0] = float("nan")
    return [x.cuda() for x in out]


class _MaskedTorch:
    """torch.optim.AdamW with the inactive rows restored after each step"""

    def __init__(self, params, groups_kw, **kw):
        self.params = params
        self.opt = torch.optim.AdamW([dict(g, params=[p]) for g, p in zip(groups_kw, params)], **kw)

    def step(self, P):
        grads = [p.grad for p in self.params if p.grad is not None]
        act = _active(grads, P)
        pre = []
        for p in self.params:
            st = self.opt.state.get(p, {})
            pre.append((p.detach().clone(), st["exp_avg"].clone() if st else torch.zeros_like(p), st["exp_avg_sq"].clone() if st else torch.zeros_like(p)))
        self.opt.step()
        with torch.no_grad():
            for p, (p0, m0, v0) in zip(self.params, pre):
                if p.grad is None or p.numel() == 0:
                    continue
                st = self.opt.state[p]
                for now, before in ((p, p0), (st["exp_avg"], m0), (st["exp_avg_sq"], v0)):
                    now[~act] = before[~act]
        return act


def _setup(P, seed, shapes=SHAPES, names=NAMES):
    g = torch.Generator().manual_seed(seed)
    init = [torch.randn((P,) + shapes[k], generator=g) for k in names]
    groups = [{"lr": LRS[k], "name": k} for k in names]
    ours = [torch.nn.Parameter(x.clone().cuda()) for x in init]
    ref = [torch.nn.Parameter(x.clone().cuda()) for x in init]
    opt = SelectiveAdamW([dict(gk, params=[p]) for gk, p in zip(groups, ours)], lr=0.0, eps=1e-15, weight_decay=0.01)
    return ours, opt, ref, _MaskedTorch(ref, groups, lr=0.0, eps=1e-15, weight_decay=0.01)


def _check(ours, opt, ref, mref):
    for a, b in zip(ours, ref):
        assert _same(a, b)
        sa, sb = opt.state.get(a), mref.opt.state.get(b)
        assert (sa is None) == (sb is None)
        if sa is not None:
            assert _same(sa["exp_avg"], sb["exp_avg"]) and _same(sa["exp_avg_sq"], sb["exp_avg_sq"])
            assert float(sa["step"]) == float(sb["step"])


@pytest.mark.parametrize("P", [1, 31, 32, 33, 4097, 100_003])
def test_bit_exact_against_masked_torch_adamw(P):
    ours, opt, ref, mref = _setup(P, 1)
    gen = torch.Generator().manual_seed(P)
    for it in range(25):
        grads = _masked_grads([SHAPES[k] for k in NAMES], P, KINDS[it % len(KINDS)], gen)
        for a, b, gr in zip(ours, ref, grads):
            a.grad, b.grad = gr.clone(), gr.clone()
        if it == 10:
            opt.param_groups[0]["lr"] = mref.opt.param_groups[0]["lr"] = 1.0e-4
        opt.step()
        act = mref.step(P)
        _check(ours, opt, ref, mref)
        if KINDS[it % len(KINDS)] == "none":
            assert not act.any()
    for a in ours:
        assert float(opt.state[a]["step"]) == 25.0


def test_full_size_3m_step():
    P = 3_000_000
    ours, opt, ref, mref = _setup(P, 2)
    gen = torch.Generator().manual_seed(0)
    for kind in ("all", "rand13"):
        grads = _masked_grads([SHAPES[k] for k in NAMES], P, kind, gen)
        for a, b, gr in zip(ours, ref, grads):
            a.grad, b.grad = gr, gr.clone()
        opt.step()
        mref.step(P)
        del grads
    _check(ours, opt, ref, mref)


def test_layouts_permuted_row_strided_zero_width_and_missing_grad():
    P = 5003
    gen = torch.Generator().manual_seed(4)
    xyz0 = torch.randn(3, P, generator=gen).cuda().t()                  # create_from_pcd: strides (1, P)
    full0 = torch.randn(P, 15, 3, generator=gen).cuda()
    full = full0.clone()
    student = full[:, :8, :]                                            # distill_train.py: the row-strided student
    student.requires_grad_(True)
    xyz = torch.nn.Parameter(xyz0.clone())
    assert xyz.stride() == (1, P) and not student.is_contiguous()
    empty = torch.nn.Parameter(torch.zeros(P, 0, 3, device="cuda"))    # _features_rest at degree 0
    opac = torch.nn.Parameter(torch.randn(P, 1, generator=gen).cuda())
    frozen = torch.nn.Parameter(torch.randn(P, 4, generator=gen).cuda())  # never gets a gradient
    frozen0 = frozen.detach().clone()
    ours = [xyz, student, empty, opac]
    ref = [torch.nn.Parameter(t.detach().clone().contiguous()) for t in ours]
    groups = [{"lr": 1e-3, "name": n} for n in ("xyz", "f_rest", "f_rest0", "opacity")]
    opt = SelectiveAdamW([dict(g, params=[p]) for g, p in zip(groups, ours)] + [{"params": [frozen], "lr": 1e-3, "name": "frozen"}],
                         lr=0.0, eps=1e-15)
    mref = _MaskedTorch(ref, groups, lr=0.0, eps=1e-15)
    for it in range(12):
        grads = _masked_grads([(3,), (8, 3), (0, 3), (1,)], P, KINDS[it % len(KINDS)], gen)
        for a, b, gr in zip(ours, ref, grads):
            a.grad, b.grad = gr.clone(), gr.clone()
        opt.step()
        mref.step(P)
        for a, b in zip(ours, ref):
            assert _same(a, b)
            assert _same(opt.state[a]["exp_avg"], mref.opt.state[b]["exp_avg"])
            assert _same(opt.state[a]["exp_avg_sq"], mref.opt.state[b]["exp_avg_sq"])
    assert xyz.stride() == (1, P) and student.data_ptr() == full.data_ptr()
    assert torch.equal(full[:, 8:, :], full0[:, 8:, :])                # coefficients outside the view untouched
    assert frozen not in opt.state and torch.equal(frozen, frozen0)    # no gradient: skipped, no step
    assert float(opt.state[empty]["step"]) == 12.0


def test_mismatched_rows_raise_before_any_launch():
    a = torch.nn.Parameter(torch.randn(100, 3, device="cuda"))
    b = torch.nn.Parameter(torch.randn(101, 1, device="cuda"))
    opt = SelectiveAdamW([{"params": [a], "lr": 1e-2}, {"params": [b], "lr": 1e-2}], lr=0.0, eps=1e-15)
    a.grad, b.grad = torch.ones_like(a), torch.ones_like(b)
    opt.param_groups[1]["params"][0].grad = None
    opt.step()                                                          # a alone: fine
    a0, m0 = a.detach().clone(), opt.state[a]["exp_avg"].clone()
    b.grad = torch.ones_like(b)
    torch.cuda.synchronize()
    n0 = capi.launch_count()
    with pytest.raises(RuntimeError, match="rows"):
        opt.step()
    torch.cuda.synchronize()
    assert capi.launch_count() == n0
    assert float(opt.state[a]["step"]) == 1.0 and b not in opt.state
    assert torch.equal(a, a0) and torch.equal(opt.state[a]["exp_avg"], m0)


def test_real_gradients_touch_exactly_the_nonzero_rows():
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.synth import make_scene, make_cameras
    scene = make_scene(6000, sh_degree=3, seed=41, scale_mult=1.6)
    cams = [TorchCamera(c, "cuda") for c in make_cameras(8, 192, 144)]
    pcs = [GaussianParams(scene["raw"], 3, "cuda") for _ in range(2)]
    opts = [cls([{"params": [p], "lr": lr} for p, lr in zip(pc.parameters(), (1.6e-4, 2.5e-3, 1.25e-4, 5e-3, 1e-3, 5e-2))], lr=0.0, eps=1e-15)
            for cls, pc in zip((SelectiveAdamW, FusedAdamW), pcs)]
    target = torch.rand(3, 144, 192, generator=torch.Generator().manual_seed(0)).cuda()
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    for step in range(3):
        img = render(cams[step], pcs[0], pipe, bg)["render"]
        (img - target).abs().mean().backward()
        for p, q in zip(pcs[0].parameters(), pcs[1].parameters()):
            q.grad = p.grad.clone()
        before = [p.detach().clone() for p in pcs[0].parameters()]
        mom = [(opts[0].state[p]["exp_avg"].clone(), opts[0].state[p]["exp_avg_sq"].clone()) if p in opts[0].state else None
               for p in pcs[0].parameters()]
        act = _active([p.grad for p in pcs[0].parameters()], 6000)
        assert 0 < int(act.sum()) < 6000
        for o in opts:
            o.step()
            o.zero_grad(set_to_none=True)
        for p, q, p0, mv in zip(pcs[0].parameters(), pcs[1].parameters(), before, mom):
            assert torch.equal(p[~act], p0[~act])
            assert torch.equal(p[act], q[act])                          # the first step of a row is FusedAdamW's first step
            if mv is not None:
                assert torch.equal(opts[0].state[p]["exp_avg"][~act], mv[0][~act])
                assert torch.equal(opts[0].state[p]["exp_avg_sq"][~act], mv[1][~act])
        if step == 0:                                                   # later steps: moments of rows frozen earlier differ
            for p, q in zip(pcs[0].parameters(), pcs[1].parameters()):
                assert torch.equal(opts[0].state[p]["exp_avg"][act], opts[1].state[q]["exp_avg"][act])
        for p, q in zip(pcs[0].parameters(), pcs[1].parameters()):     # keep both on the same parameters for the next step
            with torch.no_grad():
                q.copy_(p)
                opts[1].state[q]["exp_avg"].copy_(opts[0].state[p]["exp_avg"])
                opts[1].state[q]["exp_avg_sq"].copy_(opts[0].state[p]["exp_avg_sq"])


def _holder(params, opt, P):
    h = types.SimpleNamespace(optimizer=opt, percent_dense=0.01)
    for k, p in zip(NAMES, params):
        setattr(h, optim._GROUP_ATTR[k], p)
    gen = torch.Generator().manual_seed(17)
    h.xyz_gradient_accum = torch.rand(P, 1, generator=gen).cuda() * 4e-4
    h.denom = torch.ones(P, 1).cuda()
    h.max_radii2D = torch.rand(P, generator=gen).cuda()
    return h


def test_state_dict_checkpoints_prune_and_densify():
    from lightgaussian_b200 import densify
    P = 20011
    ours, opt, ref, mref = _setup(P, 3)
    gen = torch.Generator().manual_seed(5)
    for it in range(3):
        grads = _masked_grads([SHAPES[k] for k in NAMES], P, "rand13", gen)
        for a, b, gr in zip(ours, ref, grads):
            a.grad, b.grad = gr.clone(), gr.clone()
        opt.step()
        mref.step(P)
    sa, sb = opt.state_dict(), mref.opt.state_dict()
    for ga, gb in zip(sa["param_groups"], sb["param_groups"]):
        assert all(ga[k] == gb[k] for k in ("lr", "betas", "eps", "weight_decay", "name", "params"))
    for i in sb["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa["state"][i][k], sb["state"][i][k]), (i, k)
    # a torch AdamW checkpoint loaded into a fresh SelectiveAdamW (GaussianModel.restore), then prune, densify, step
    params = [torch.nn.Parameter(p.detach().clone()) for p in ref]
    sel = SelectiveAdamW([{"params": [p], "lr": LRS[k], "name": k} for p, k in zip(params, NAMES)], lr=0.0, eps=1e-15, weight_decay=0.01)
    sel.load_state_dict(copy.deepcopy(sb))
    h_ours = _holder(params, sel, P)
    h_ref = _holder(ref, mref.opt, P)
    mask = (torch.rand(P, generator=torch.Generator().manual_seed(2)) < 0.3).cuda()
    for h in (h_ours, h_ref):
        optim.prune_points(h, mask)
        torch.manual_seed(11)
        densify.densify_and_prune(h, 2e-4, 0.005, 3.0, 20)
    P2 = h_ours._xyz.shape[0]
    assert P2 == h_ref._xyz.shape[0] and P2 != P - int(mask.sum())
    new_ours = [getattr(h_ours, optim._GROUP_ATTR[k]) for k in NAMES]
    new_ref = [getattr(h_ref, optim._GROUP_ATTR[k]) for k in NAMES]
    mref.params = new_ref
    grads = _masked_grads([SHAPES[k] for k in NAMES], P2, "rand13", gen)
    for a, b, gr in zip(new_ours, new_ref, grads):
        a.grad, b.grad = gr.clone(), gr.clone()
    sel.step()
    mref.step(P2)
    _check(new_ours, sel, new_ref, mref)


def _psnr(a, b):
    mse = float(((a - b) ** 2).mean())
    return 99.0 if mse == 0 else 10.0 * math.log10(1.0 / mse)


def test_finetune_quality_within_3_percent_of_dense():
    """the finetune loop of test_gpu_loops.py from a perturbed start, same views and learning rates: SelectiveAdamW must learn
    (> 3 dB over the start) and land within 3 % of the dense optimizer's PSNR"""
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.synth import make_scene, make_cameras
    scene = make_scene(5000, sh_degree=3, seed=53, scale_mult=1.6)
    cams = [TorchCamera(c, "cuda") for c in make_cameras(8, 192, 144)]
    pipe, bg = pipeline_params(), torch.zeros(3, device="cuda")
    with torch.no_grad():
        gt = GaussianParams(scene["raw"], 3, "cuda", requires_grad=False)
        targets = [render(c, gt, pipe, bg)["render"].clone() for c in cams]
    rng = np.random.default_rng(1)
    raw = {k: v.copy() for k, v in scene["raw"].items()}
    raw["features_dc"] += 0.5 * rng.standard_normal(raw["features_dc"].shape).astype(np.float32)
    raw["opacity"] += 1.0 * rng.standard_normal(raw["opacity"].shape).astype(np.float32)

    def run(cls, steps):
        pc = GaussianParams(raw, 3, "cuda", requires_grad=steps > 0)
        if steps:
            opt = cls([{"params": [pc._xyz], "lr": 1e-4}, {"params": [pc._features_dc], "lr": 1e-2}, {"params": [pc._features_rest], "lr": 5e-4},
                       {"params": [pc._opacity], "lr": 5e-2}, {"params": [pc._scaling], "lr": 5e-3}, {"params": [pc._rotation], "lr": 1e-3}],
                      lr=0.0, eps=1e-15)
            for it in range(steps):
                i = it % len(cams)
                (render(cams[i], pc, pipe, bg)["render"] - targets[i]).abs().mean().backward()
                opt.step()
                opt.zero_grad(set_to_none=True)
        with torch.no_grad():
            return float(np.mean([_psnr(render(c, pc, pipe, bg)["render"], t) for c, t in zip(cams, targets)]))

    p0 = run(None, 0)
    dense = run(FusedAdamW, 480)
    sel = run(SelectiveAdamW, 480)
    print(f"finetune PSNR: start {p0:.3f} dB, dense {dense:.3f} dB, selective {sel:.3f} dB")
    assert sel > p0 + 3.0, (p0, dense, sel)
    assert sel > dense - 0.03 * dense, (p0, dense, sel)


def test_prune_finetune_script_opts_in_unmodified(tmp_path):
    """prune_finetune.py through the drop-ins with LGR_SELECTIVE_ADAM=1: the trace shows the selective steps and the held-out PSNR is
    within 3 % of the dense run's"""
    import os
    from tests import scripts_harness as sh
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)
    it0, steps = 30000, 200
    w = sh.build_workdir(str(tmp_path), iteration=it0)
    gt_q = [np.rint(np.clip(g, 0, 1) * 255.0).astype(np.float32) / 255.0 for g in w["gt"]]
    test_idx = [k for k in range(len(w["cams"])) if k % 8 == 0]
    last = it0 + steps
    out = {}
    saved = os.environ.get("LGR_SELECTIVE_ADAM")
    try:
        for port, sel in ((6120, "0"), (6121, "1")):
            os.environ["LGR_SELECTIVE_ADAM"] = sel
            model = os.path.join(str(tmp_path), f"pf_{sel}")
            trace = model + ".trace.json"
            sh.run("ours", ["prune_finetune.py", "-s", w["data"], "-m", model, "--eval", "-r", "1", "--port", str(port),
                            "--start_checkpoint", w["ckpt"], "--iterations", str(last), "--prune_percent", "0.66", "--prune_type",
                            "v_important_score", "--prune_decay", "1", "--v_pow", "0.1", "--position_lr_max_steps", str(last),
                            "--prune_iterations", str(it0 + 1), "--test_iterations", "999999", "--save_iterations", str(last),
                            "--checkpoint_iterations", str(last)], trace=trace)
            ck = sh.load_checkpoint_leaves(os.path.join(model, f"chkpnt{last}.pth"))
            out[sel] = (sh.read_trace(trace), sh.psnr_of_leaves(ck["leaves"], 3, [w["cams"][k] for k in test_idx], [gt_q[k] for k in test_idx]))
    finally:
        if saved is None:
            os.environ.pop("LGR_SELECTIVE_ADAM", None)
        else:
            os.environ["LGR_SELECTIVE_ADAM"] = saved
    (t_dense, p_dense), (t_sel, p_sel) = out["0"], out["1"]
    print(f"prune_finetune held-out PSNR: dense {p_dense:.3f} dB, selective {p_sel:.3f} dB")
    assert t_dense.get("adamw_selective_steps", 0) == 0 and t_dense["adamw_steps"] == steps - 1, t_dense
    assert t_sel.get("adamw_selective_steps", 0) > 0 and t_sel.get("adamw_steps", 0) == 0, t_sel
    assert p_sel >= 0.97 * p_dense, (p_dense, p_sel)
