"""Blending-weight significance without a GPU: the reference weights derived from the CPU oracle's own blend, the exactness of the
fixed-point sums, the view-parallel reduction under gloo, the overflow bound, the LGR_SIGNIFICANCE switch and the kernel's resources.

Reference weights.  The oracle's blend accumulates C += fl(T * fl(alpha * colour)) per blended pair.  With the background black and
colour 1 on one channel of ONE Gaussian (0 everywhere else), a pixel's channel is exactly fl(alpha * T) of that Gaussian's pair, or 0
when the pixel does not blend it; the colours change no decision of the blend.  So each oracle call yields the per-pixel weights of
three Gaussians, straight from the oracle's own per-pixel lists, alpha and transmittance."""
import os
import re
import socket
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lightgaussian_b200 import build, parallel, renderer
from oracle.lgo import Oracle
from tests.test_deterministic_sass import CUOBJDUMP, _find, sass  # noqa: F401  (module fixture: the library's SASS by kernel name)
from tests.util import CONFIGS, make_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWO32 = 2.0 ** 32


# ---------------------------------------------------------------------------------------------------------------------------------
# reference weights from the oracle
# ---------------------------------------------------------------------------------------------------------------------------------
def oracle_pair_weights(o: Oracle, view, geom, point_list, ranges, ids):
    """{Gaussian id: [H*W] per-pixel alpha*T in the oracle's dtype (0 where the pixel does not blend it)} for `ids`."""
    dt = o.dt
    P = geom["radii"].shape[0]
    bg0 = view.bg
    view.bg = np.zeros(3, np.float32)
    out = {}
    try:
        for k in range(0, len(ids), 3):
            grp = ids[k:k + 3]
            col = np.zeros((P, 3), dt)
            for c, g in enumerate(grp):
                col[g, c] = 1
            img = o.blend_forward(view, ranges, point_list, geom["means2D"], col, geom["conic_opacity"])
            for c, g in enumerate(grp):
                out[int(g)] = img["color"][c].reshape(-1).copy()
    finally:
        view.bg = bg0
    return out


def fixed_point(w32: np.ndarray) -> np.ndarray:
    """q = rint(w * 2^32), round half to even, per element (the kernel's __float2uint_rn on the exactly scaled value)."""
    return np.rint(w32.astype(np.float64) * TWO32).astype(np.int64)


def reference(name, want_double=False):
    """float32 oracle geometry, lists and blend of config `name`, with every visible Gaussian's per-pixel weights."""
    act, view, _ = make_config(name)
    o = Oracle()
    geom = o.preprocess(view, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
    point_list, ranges = o.bin(view, geom["means2D"], geom["depths"], geom["radii"], geom["tiles_touched"])
    P = geom["radii"].shape[0]
    cnt = np.zeros(P, np.int64)
    img = o.blend_forward(view, ranges, point_list, geom["means2D"], geom["rgb"], geom["conic_opacity"], cnt, want_fragile=True)
    ids = np.unique(point_list)
    w = oracle_pair_weights(o, view, geom, point_list, ranges, ids)
    res = dict(act=act, view=view, geom=geom, point_list=point_list, ranges=ranges, img=img, count=cnt, ids=ids, w=w, P=P)
    if want_double:
        od = Oracle(double=True)
        gd = {k: (v.astype(np.float64) if v.dtype == np.float32 else v) for k, v in geom.items()}
        res["w64"] = oracle_pair_weights(od, view, gd, point_list, ranges, ids)
    return res


def weight_fx(ref) -> np.ndarray:
    fx = np.zeros(ref["P"], np.int64)
    for g, w in ref["w"].items():
        fx[g] = fixed_point(w).sum()
    return fx


def touches_fragile(ref) -> np.ndarray:
    """Gaussians listed in a tile that holds a fragile pixel (a threshold test within rounding noise): their pairs may differ
    between implementations whose exp() differs."""
    view, frag = ref["view"], ref["img"]["fragile"]
    gx = (view.W + 15) // 16
    out = np.zeros(ref["P"], bool)
    for t, (a, b) in enumerate(ref["ranges"]):
        ty, tx = divmod(t, gx)
        if b > a and frag[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16].any():
            out[ref["point_list"][a:b]] = True
    return out


@pytest.fixture(scope="module", params=list(CONFIGS))
def ref(request):
    return reference(request.param, want_double=True)


def test_weights_match_a_plain_loop_and_the_blend(ref):
    """The pairs with a weight are exactly the pairs gaussians_count counts; the fixed-point sums equal a plain Python loop over
    each Gaussian's pixels with integer arithmetic."""
    fx = weight_fx(ref)
    for g, w in ref["w"].items():
        assert int((w > 0).sum()) == ref["count"][g], g
        assert (w <= np.float32(0.99)).all() and (w[w > 0] > np.float32(3.9e-7)).all(), g
    rng = np.random.default_rng(0)
    for g in rng.choice(ref["ids"], size=min(40, len(ref["ids"])), replace=False):
        total = 0
        for v in ref["w"][int(g)].tolist():
            if v:
                total += round(v * 2 ** 32)      # exact: v is a float32, v * 2^32 a float64 with the same mantissa
        assert total == int(fx[g]), g
    assert fx.sum() > 0 and (fx[ref["count"] == 0] == 0).all()


def test_float32_against_float64(ref):
    """float32 fixed-point weights within the quantisation bound plus float32 rounding of the float64 oracle's real-valued sums,
    on the same per-pixel lists; exact agreement is not expected (T accumulates rounding pair by pair)."""
    fx = weight_fx(ref)
    frag = touches_fragile(ref)
    worst = 0.0
    for g, w64 in ref["w64"].items():
        exact = float(w64.sum())
        n = int(ref["count"][g])
        err = abs(fx[g] / TWO32 - exact)
        if not frag[g]:
            assert err <= n * 2.0 ** -33 + 1e-4 * exact + n * 1e-6, (g, fx[g] / TWO32, exact)
            worst = max(worst, err / max(exact, 1e-12))
        else:
            assert err <= 0.02 * exact + n * 2e-3, (g, fx[g] / TWO32, exact)
    print(f"worst relative float32/float64 weight difference off fragile tiles: {worst:.2e}")


def test_weights_sum_to_one_minus_final_T_on_every_pixel(ref):
    """On every pixel the blended weights add up to the coverage 1 - final_T (telescoping sum), within n_contrib float32 ulps."""
    N = ref["view"].W * ref["view"].H
    acc = np.zeros(N, np.float64)
    for w in ref["w"].values():
        acc += w.astype(np.float64)
    cover = 1.0 - ref["img"]["final_T"].astype(np.float64)
    n = ref["img"]["n_contrib"].astype(np.float64)
    assert (np.abs(acc - cover) <= 2 * (n + 1) * 2.0 ** -24).all(), np.abs(acc - cover).max()


# ---------------------------------------------------------------------------------------------------------------------------------
# view-parallel reduction, overflow bound, switch
# ---------------------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _cams(n, W=64, H=48):
    return [SimpleNamespace(idx=i, image_width=W, image_height=H) for i in range(n)]


def _fake_count_render(cam, gaussians, pipe, bg):
    """fixed per-camera int64 weights up to 0.99 * 2^32 * (W*H) / P, as a real view could produce"""
    g = torch.Generator().manual_seed(5000 + cam.idx)
    P = gaussians.get_xyz.shape[0]
    fx = torch.randint(0, 2 ** 40, (P,), generator=g, dtype=torch.int64)
    return {"gaussians_count": torch.randint(0, 500, (P,), generator=g, dtype=torch.int32), "blend_weight_fx": fx,
            "important_score": renderer.weight_score(fx)}


def _model(P=301):
    g = torch.Generator().manual_seed(9)
    return SimpleNamespace(get_xyz=torch.rand(P, 3, generator=g), get_opacity=torch.rand(P, 1, generator=g))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      LGR_SIGNIFICANCE="blend_weight")
    parallel.init_from_env("gloo")
    cnt, imp = parallel.sharded_prune_list(_model(), _cams(13), None, None, _fake_count_render, rank, world)
    torch.save(dict(cnt=cnt, imp=imp), os.path.join(out, f"w{world}_r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_weights_identical_on_every_rank_and_world_size(tmp_path, monkeypatch):
    monkeypatch.setenv("LGR_SIGNIFICANCE", "blend_weight")
    cams, model = _cams(13), _model()
    cnt1, imp1 = parallel.sharded_prune_list(model, cams, None, None, _fake_count_render, 0, 1)
    fx = sum(_fake_count_render(c, model, None, None)["blend_weight_fx"] for c in cams)
    assert torch.equal(imp1, (fx.double() * 2.0 ** -32).float())
    assert torch.equal(cnt1, sum(_fake_count_render(c, model, None, None)["gaussians_count"].long() for c in cams))
    for world in (2, 3, 4):
        mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
        for r in range(world):
            d = torch.load(os.path.join(tmp_path, f"w{world}_r{r}.pt"))
            assert torch.equal(d["cnt"], cnt1), (world, r)
            assert torch.equal(d["imp"], imp1), (world, r)


def test_overflow_bound_raises_before_any_view(monkeypatch):
    monkeypatch.setenv("LGR_SIGNIFICANCE", "blend_weight")
    calls = []

    def fn(*a):
        calls.append(a)
        return _fake_count_render(*a)
    big = [SimpleNamespace(idx=i, image_width=1920, image_height=1080) for i in range(1036)]   # 2 148 291 200 >= 2^31 pixel-views
    with pytest.raises(RuntimeError, match="2\\^31 pixel-views"):
        parallel.sharded_prune_list(_model(), big, None, None, fn, 0, 1)
    assert calls == []
    assert parallel.check_weight_bound(big[:1035]) == 1035 * 1920 * 1080     # just below
    monkeypatch.setenv("LGR_SIGNIFICANCE", "count")                            # the bound is the weight's only
    parallel.sharded_prune_list(_model(), big[:2], None, None, fn, 0, 1)


def test_unknown_significance_mode_raises(monkeypatch):
    monkeypatch.delenv("LGR_SIGNIFICANCE", raising=False)
    assert renderer.significance_mode() == "count"
    monkeypatch.setenv("LGR_SIGNIFICANCE", "blend_weight")
    assert renderer.significance_mode() == "blend_weight"
    monkeypatch.setenv("LGR_SIGNIFICANCE", "weight")
    with pytest.raises(RuntimeError, match="LGR_SIGNIFICANCE"):
        renderer.count_render(None, None, None, None)        # before anything is read from the camera or the model
    with pytest.raises(RuntimeError, match="LGR_SIGNIFICANCE"):
        parallel.sharded_prune_list(_model(), _cams(2), None, None, _fake_count_render)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]), LGR_SIGNIFICANCE="weight")
    r = subprocess.run([sys.executable, "-c", "import gaussian_renderer"], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "LGR_SIGNIFICANCE" in r.stderr, r.stderr[-2000:]
    env["LGR_SIGNIFICANCE"] = "blend_weight"
    r = subprocess.run([sys.executable, "-c", "import gaussian_renderer"], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]


def test_weight_kernel_does_not_spill(sass):  # noqa: F811
    """The WEIGHT instantiation of the count blend: no spills and no more stack than the default count kernel (whose 8 bytes are the
    ring-timeout printf), two REDUX per pair and one 64-bit integer reduction."""
    out = subprocess.run([CUOBJDUMP, "--dump-resource-usage", build.build_library()], check=True, capture_output=True, text=True).stdout
    usage = dict((n, (int(r), int(s), int(loc))) for n, r, s, loc in
                 re.findall(r"Function (\S*blend_forward_ring_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out))
    weight = [n for n in usage if "ILb1ELb0ELb0ELb1E" in n]
    count = [n for n in usage if "ILb1ELb0ELb0ELb0E" in n]
    assert len(weight) == 1 and len(count) == 1, sorted(usage)
    reg, stack, local = usage[weight[0]]
    assert local == 0 and stack <= usage[count[0]][1], usage[weight[0]]
    assert reg * 288 <= 65536, reg
    body = sass[_find(sass, "blend_forward_ring_kernelILb1ELb0ELb0ELb1E")[0]]
    assert "REDUX" in body and re.search(r"\bRED[G]?\.E\.ADD\.64\b", body), "expected warp REDUX and a 64-bit integer reduction"
    assert "REDUX" not in sass[_find(sass, "blend_forward_ring_kernelILb1ELb0ELb0ELb0E")[0]]
